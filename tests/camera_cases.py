"""The cases of tests/golden/camera_fit.npz (made by tests/golden/make_golden_camera.py) and the parity bound derived
from them, shared by test_camera_cpu.py and test_gpu_camera.py."""
import numpy as np

from helpers import load_npz

N_CASES = 65
DEMO, ZERO = 0, 64
COCO = range(32, 64)
CAM_FLOOR = 1e-3   # the bound never goes below this (a case whose 1-ulp rerun lands on the same bits has spread 0)
LOSS_FLOOR = 2e-3  # relative; measured: the kernel-order float32 loop ends 1.35e-3 from the reference's loss on case 58
# Cases whose L1 minimum is not unique: the reference's loop in float32 and the same loop in float64 end 0.40 (case 58)
# and 4.9e-3 (case 52) apart in the camera, while their losses agree within 7e-4 (relative).  The 1-ulp rerun does not
# reveal this (its spread there is 0 and 8e-5), so on these two cases only the loss is held to the bound.
AMBIGUOUS = (52, 58)


def fixture():
    return load_npz("camera_fit.npz")


def joint_inputs(z):
    """The 65 image poses in case order, each with the dtype the reference saw."""
    it_int, it_f64 = iter(z["joints_h36m_int"]), iter(z["joints_h36m_f64"])
    out = [z["joints_demo"]]
    for k in z["kind"][1:32]:
        out.append(next(it_int) if k == 1 else next(it_f64))
    out += list(z["joints_coco"])
    out.append(z["joints_zero"])
    return out


def targets(z):
    """Per-case crop targets [Jin, 2] (17 rows, 19 for the coco cases)."""
    t = [z["target_17"][i] for i in range(N_CASES)]
    for k, i in enumerate(COCO):
        t[i] = z["target_coco"][k]
    return t


def cam_bound(z):
    """Per case: 2 x the spread of the reference's 1-ulp-perturbed rerun, floored at CAM_FLOOR."""
    spread = np.abs(z["cam"].astype(np.float64) - z["cam_pert"]).max(1)
    return np.maximum(2 * spread, CAM_FLOOR)


def loss_bound(z):
    """Per case, relative to the reference's loss: 2 x the rerun's relative spread, floored at LOSS_FLOOR."""
    loss = z["loss"].astype(np.float64)
    rel = np.abs(loss - z["loss_pert"]) / np.maximum(loss, 1e-30)
    return np.maximum(2 * rel, LOSS_FLOOR)


def violations(z, cam, loss, cases=None):
    """Indices of cases whose camera or loss falls outside the bound."""
    cases = np.arange(N_CASES) if cases is None else np.asarray(cases)
    dc = np.abs(np.asarray(cam, np.float64) - z["cam"][cases]).max(1)
    ref = z["loss"][cases].astype(np.float64)
    dl = np.abs(np.asarray(loss, np.float64) - ref) / np.maximum(ref, 1e-30)
    cam_ok = (dc <= cam_bound(z)[cases]) | np.isin(cases, AMBIGUOUS)
    bad = ~cam_ok | (dl > loss_bound(z)[cases]) | ~np.isfinite(dc)
    return cases[bad].tolist()
