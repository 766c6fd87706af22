"""The camera-fit oracle (oracle/camera_oracle.py) against the outputs of the unmodified reference
(tests/golden/camera_fit.npz, made by tests/golden/make_golden_camera.py).

The fit is chaotic at the scale of the learning rate: a one-ulp change of the target moves the reference's final
camera by up to ~1e-3.  The parity bound is therefore per case, 2 x the spread of the reference's own one-ulp rerun,
floored at 1e-3 (tests/camera_cases.py); test_bound_teeth records which mutations of the loop it rejects."""
import numpy as np
import pytest

import camera_cases as cc
from oracle import camera_oracle as co

MUTATION_OUTCOME = {
    # mutation of the float64 oracle: does the reference bound reject it (on at least one fixture case)?  Measured.
    "lr_switch_one_step_early": True,    # cases 0, 19, 29
    "no_bias_correction": True,          # cases 0, 1, 10, 58, 62
    "eps_inside_sqrt": False,            # eps = 1e-8 against sqrt(v) ~ 1e-2 .. 1e2: invisible at this bound
    "sign_of_zero_plus_one": False,      # case 64's residuals are exactly zero in float32 only; in float64 they are
                                         # ~1e-14 and never zero, so this restatement cannot show the switch
    "bbox_scale_1": True,                # every case
    "aspect_ratio_0_75": True,           # 32 of 65 cases
    "all_19_coco_rows_in_loss": True,    # every coco case
}


def _all_targets(z, **kw):
    return [co.crop_target(j, **kw)[1] for j in cc.joint_inputs(z)]


def test_oracle_target_and_bbox_match_reference_bitwise():
    z = cc.fixture()
    for i, j in enumerate(cc.joint_inputs(z)):
        bbox, tgt = co.crop_target(j)
        assert bbox.dtype == np.float32 and np.array_equal(bbox, z["bbox"][i]), i
        assert np.array_equal(tgt, cc.targets(z)[i]), i


def test_orig_cam_matches_reference_bitwise():
    z = cc.fixture()
    got = co.orig_cam_f32(z["cam"], z["bbox"], z["img_wh"][:, 0], z["img_wh"][:, 1])
    assert np.array_equal(got, z["orig_cam"])


def _fit(z, fit, targets=None, p3d=None, cases=None, **kw):
    cases = np.arange(cc.N_CASES) if cases is None else np.asarray(cases)
    targets = cc.targets(z) if targets is None else targets
    p3d = z["pred_joints3d"] if p3d is None else p3d
    tg = np.stack([targets[i][:p3d.shape[1]] for i in cases])
    return fit(p3d[cases], tg, z["init"][cases], **kw)


def test_float64_fit_within_reference_spread():
    z = cc.fixture()
    cam, loss = _fit(z, co.fit_f64)
    assert cc.violations(z, cam, loss) == []


def test_kernel_order_fit_within_reference_spread():
    z = cc.fixture()
    cam, loss = _fit(z, co.fit_f32_kernel_order)
    assert cc.violations(z, cam, loss) == []
    assert np.array_equal(cam[cc.ZERO], np.array([1, 0, 0], np.float32)) and loss[cc.ZERO] == 0   # sign(0) = 0
    assert np.array_equal(z["cam"][cc.ZERO], np.array([1, 0, 0], np.float32))                      # as the reference


def _mutated(z, name):
    """(cam, loss, cases) of the float64 oracle under one mutation."""
    if name == "lr_switch_one_step_early":
        return (*_fit(z, co.fit_f64, schedule=((0, 0.1), (500, 0.05), (1000, 0.001))), None)
    if name == "no_bias_correction":
        return (*_fit(z, co.fit_f64, bias_correction=False), None)
    if name == "eps_inside_sqrt":
        return (*_fit(z, co.fit_f64, eps_inside_sqrt=True), None)
    if name == "sign_of_zero_plus_one":
        return (*_fit(z, co.fit_f64, cases=[cc.ZERO], sign_of_zero=1.0), [cc.ZERO])
    if name == "bbox_scale_1":
        return (*_fit(z, co.fit_f64, targets=_all_targets(z, scale=1.0)), None)
    if name == "aspect_ratio_0_75":
        return (*_fit(z, co.fit_f64, targets=_all_targets(z, aspect=0.75)), None)
    if name == "all_19_coco_rows_in_loss":
        # 19 predicted joints: the 17 regressed ones with pelvis and neck appended as the inputs' are (run.py:127-146)
        p = z["pred_joints3d"].astype(np.float64)
        p19 = np.concatenate([p, (p[:, 11:12] + p[:, 12:13]) * 0.5, (p[:, 5:6] + p[:, 6:7]) * 0.5], 1)
        return (*_fit(z, co.fit_f64, p3d=p19, cases=list(cc.COCO)), list(cc.COCO))
    raise KeyError(name)


@pytest.mark.parametrize("name", sorted(MUTATION_OUTCOME))
def test_bound_teeth(name):
    z = cc.fixture()
    cam, loss, cases = _mutated(z, name)
    bad = cc.violations(z, cam, loss, cases)
    print(name, "cases outside the bound:", bad)
    assert bool(bad) == MUTATION_OUTCOME[name], (name, bad)
