#!/usr/bin/env python
"""Golden vectors of the body-model forwards, produced by the UNMODIFIED reference layers: smplpytorch's
SMPL_Layer.forward and manopth's ManoLayer.forward, run on CPU in float32.  The layers are built on the seeded synthetic
models of tests/body_models.py with __new__ + Module.__init__ + register_buffer (tests/body_models.py:_layer), which
bypasses only the chumpy pkl loader; both modules import and run this way without chumpy.

    P2M_REFERENCE_ROOT=/path/to/Pose2Mesh_RELEASE python tests/golden/make_golden_body_model.py -> body_model.npz

Models: "smpl" and "mano_{right,left}{,_flat}" (flat = flat_hand_mean, zero hands_mean); digest_{model} is
body_models.digest of each.  Case c: c__model, c__pose, c__betas (absent = the layer's default argument), c__trans
(absent = default), c__center (-1 = None), c__joints [B, J, 3] and c__verts on the rows c__rows (a seeded 512 of
SMPL's 6890 rows; all of MANO's 778).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import body_models as bm  # noqa: E402
import body_model_oracle as bo  # noqa: E402

REF = os.environ.get("P2M_REFERENCE_ROOT", "")


def models():
    out = {"smpl": bm.smpl_model()}
    for side in ("right", "left"):
        for flat in (False, True):
            out[f"mano_{side}" + ("_flat" if flat else "")] = bm.mano_model(side, flat)
    return out


def cases(rng):
    """(name, model, pose, betas, trans, center_idx); betas / trans None = the layer's default argument."""
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    n = lambda *s, sd=1.0: f(rng.normal(0.0, sd, s))  # noqa: E731
    angles = bm.random_axisang(rng, 4 * 24, 1e-7, 3 * np.pi)
    angles[:3] = [[1e-7, 0, 0], [0, 0, 3 * np.pi], [np.pi, 0, 0]]
    mano_angles = bm.random_axisang(rng, 3 * 16, 1e-7, 3 * np.pi)
    mano_angles[:2] = [[0, 1e-7, 0], [0, 3 * np.pi, 0]]
    out = [
        ("smpl_random", "smpl", n(4, 72, sd=0.6), n(4, 10, sd=1.5), n(4, 3, sd=0.5), None),
        ("smpl_zero_pose", "smpl", f(np.zeros((2, 72))), n(2, 10, sd=1.5), None, None),
        ("smpl_zero_betas", "smpl", n(3, 72, sd=0.6), f(np.zeros((3, 10))), n(3, 3, sd=0.5), None),
        ("smpl_no_betas", "smpl", n(2, 72, sd=0.6), None, None, None),
        ("smpl_center", "smpl", n(3, 72, sd=0.6), n(3, 10, sd=1.5), f(np.zeros((3, 3))), 0),
        ("smpl_center_no_trans", "smpl", n(2, 72, sd=0.6), n(2, 10, sd=1.5), None, 3),
        ("smpl_angles", "smpl", f(angles.reshape(4, 72)), n(4, 10, sd=1.5), n(4, 3, sd=0.5), None),
    ]
    for m in ("mano_right", "mano_left", "mano_right_flat", "mano_left_flat"):
        out.append((f"{m}_random", m, n(3, 48, sd=0.8), n(3, 10, sd=1.5), n(3, 3, sd=0.1), None))
    out += [
        ("mano_zero_betas", "mano_right", n(2, 48, sd=0.8), f(np.zeros((2, 10))), n(2, 3, sd=0.1), None),
        ("mano_no_betas", "mano_left", n(2, 48, sd=0.8), None, None, None),
        ("mano_zero_pose", "mano_right", f(np.zeros((2, 48))), n(2, 10, sd=1.5), None, None),
        ("mano_center", "mano_right", n(2, 48, sd=0.8), n(2, 10, sd=1.5), f(np.zeros((2, 3))), 9),
        ("mano_center_tip", "mano_left_flat", n(2, 48, sd=0.8), n(2, 10, sd=1.5), None, 4),
        ("mano_angles", "mano_right", f(mano_angles.reshape(3, 48)), n(3, 10, sd=1.5), n(3, 3, sd=0.1), None),
    ]
    return out


def oracle(model, pose, betas, trans, center):
    fwd = bo.smpl_forward if "parents" in model and len(model["parents"]) == 24 else bo.mano_forward
    return fwd(model, pose, betas, trans, center)


def main():
    if not os.path.isdir(os.path.join(REF, "smplpytorch")):
        raise SystemExit("set P2M_REFERENCE_ROOT to a Pose2Mesh_RELEASE checkout")
    sys.path[:0] = [os.path.join(REF, "smplpytorch"), os.path.join(REF, "manopth")]
    from manopth.manolayer import ManoLayer
    from smplpytorch.pytorch.smpl_layer import SMPL_Layer

    torch.set_num_threads(1)
    ms = models()
    rng = np.random.RandomState(2024)
    smpl_rows = np.sort(rng.choice(6890, 512, replace=False)).astype(np.int32)
    Z = {f"digest_{k}": np.array(bm.digest(m)) for k, m in ms.items()}
    names = []
    for name, mk, pose, betas, trans, center in cases(rng):
        m = ms[mk]
        if mk == "smpl":
            layer = bm.smpl_reference_layer(SMPL_Layer, m, center_idx=center)
            rows = smpl_rows
        else:
            layer = bm.mano_reference_layer(ManoLayer, m, center_idx=center, flat_hand_mean=mk.endswith("_flat"))
            rows = np.arange(778, dtype=np.int32)
        args = {}
        if betas is not None:
            args["th_betas"] = torch.from_numpy(betas)
        if trans is not None:
            args["th_trans"] = torch.from_numpy(trans)
        with torch.no_grad():
            v, j = layer(torch.from_numpy(pose), **args)
        v, j = v.numpy(), j.numpy()
        ov, oj = oracle(m, pose, betas, trans, center)
        scale = np.maximum(np.abs(ov).max(axis=(1, 2)), np.abs(oj).max(axis=(1, 2)))
        err = max(np.abs(v - ov).max(axis=(1, 2)).max() / scale.min(), np.abs(j - oj).max() / scale.min())
        print(f"{name:24s} B={pose.shape[0]}  reference fp32 vs oracle: {err:.2e} of the sample max")
        Z[f"{name}__model"] = np.array(mk)
        Z[f"{name}__pose"] = pose
        if betas is not None:
            Z[f"{name}__betas"] = betas
        if trans is not None:
            Z[f"{name}__trans"] = trans
        Z[f"{name}__center"] = np.array(-1 if center is None else center, np.int32)
        Z[f"{name}__rows"] = rows
        Z[f"{name}__verts"] = np.ascontiguousarray(v[:, rows])
        Z[f"{name}__joints"] = j
        names.append(name)
    Z["cases"] = np.array(names)
    path = os.path.join(HERE, "body_model.npz")
    np.savez_compressed(path, **Z)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
