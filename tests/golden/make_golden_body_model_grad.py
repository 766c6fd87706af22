#!/usr/bin/env python
"""Golden vector-Jacobian products of the body-model forwards, produced by the UNMODIFIED reference layers:
smplpytorch's SMPL_Layer and manopth's ManoLayer, moved to float64 with .double() and differentiated by autograd on
CPU.  The layers are built on the seeded synthetic models of tests/body_models.py, as make_golden_body_model.py builds
them.

    P2M_REFERENCE_ROOT=/path/to/Pose2Mesh_RELEASE python tests/golden/make_golden_body_model_grad.py
        -> body_model_grad.npz

Models and digest_{model} as in body_model.npz.  Case c: c__model, c__pose, c__betas / c__trans (absent = the layer's
default argument), c__center (-1 = None), c__seed.  The cotangents are regenerated from the seed
(`cotangents`, float32 values).  For each mode m in ("verts", "joints", "both") -- the cotangent on the vertices, on
the joints, on both -- c__m__pose and, when the input was given, c__m__betas / c__m__trans: the reference's float64
gradients, with zeros where autograd reports none (an input the forward did not use).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import body_models as bm  # noqa: E402

REF = os.environ.get("P2M_REFERENCE_ROOT", "")
MODES = ("verts", "joints", "both")


def models():
    out = {"smpl": bm.smpl_model()}
    for side in ("right", "left"):
        for flat in (False, True):
            out[f"mano_{side}" + ("_flat" if flat else "")] = bm.mano_model(side, flat)
    return out


def cotangents(seed, B, n_vertex, n_joint, mode):
    """(grad_verts, grad_joints) of one mode; None = zero."""
    rng = np.random.RandomState(seed)
    gv = rng.normal(0.0, 1.0, (B, n_vertex, 3)).astype(np.float32)
    gj = rng.normal(0.0, 1.0, (B, n_joint, 3)).astype(np.float32)
    return (None if mode == "joints" else gv), (None if mode == "verts" else gj)


def cases(rng):
    """(name, model, pose, betas, trans, center_idx); betas / trans None = the layer's default argument."""
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    n = lambda *s, sd=1.0: f(rng.normal(0.0, sd, s))  # noqa: E731
    angles = bm.random_axisang(rng, 3 * 24, 1e-7, 3 * np.pi)
    angles[:6] = [[1e-7, 0, 0], [0, 2e-7, -1e-7], [np.pi, 0, 0], [0, np.pi - 1e-3, 0], [0, 0, 3 * np.pi],
                  [3 * np.pi - 1e-2, 0, 0]]
    mano_angles = bm.random_axisang(rng, 2 * 16, 1e-7, 3 * np.pi)
    mano_angles[:3] = [[0, 1e-7, 0], [0, 0, np.pi], [0, 3 * np.pi, 0]]
    out = [
        ("smpl_random", "smpl", n(3, 72, sd=0.6), n(3, 10, sd=1.5), n(3, 3, sd=0.5), None),
        ("smpl_zero_pose", "smpl", f(np.zeros((2, 72))), n(2, 10, sd=1.5), None, None),
        ("smpl_angles", "smpl", f(angles.reshape(3, 72)), n(3, 10, sd=1.5), n(3, 3, sd=0.5), None),
        ("smpl_zero_betas", "smpl", n(2, 72, sd=0.6), f(np.zeros((2, 10))), n(2, 3, sd=0.5), None),
        ("smpl_no_betas", "smpl", n(2, 72, sd=0.6), None, n(2, 3, sd=0.5), None),
        ("smpl_center_zero_trans", "smpl", n(2, 72, sd=0.6), n(2, 10, sd=1.5), f(np.zeros((2, 3))), 0),
        ("smpl_center_no_trans", "smpl", n(2, 72, sd=0.6), n(2, 10, sd=1.5), None, 3),
    ]
    for m in ("mano_right", "mano_left", "mano_right_flat", "mano_left_flat"):
        out.append((f"{m}_random", m, n(2, 48, sd=0.8), n(2, 10, sd=1.5), n(2, 3, sd=0.1), None))
    out += [
        ("mano_zero_pose", "mano_right_flat", f(np.zeros((2, 48))), n(2, 10, sd=1.5), None, None),
        ("mano_angles", "mano_right", f(mano_angles.reshape(2, 48)), n(2, 10, sd=1.5), n(2, 3, sd=0.1), None),
        ("mano_zero_betas", "mano_right", n(2, 48, sd=0.8), f(np.zeros((2, 10))), n(2, 3, sd=0.1), None),
        ("mano_no_betas", "mano_left", n(2, 48, sd=0.8), None, n(2, 3, sd=0.1), None),
        ("mano_center_zero_trans", "mano_right", n(2, 48, sd=0.8), n(2, 10, sd=1.5), f(np.zeros((2, 3))), 9),
        ("mano_center_tip", "mano_left_flat", n(2, 48, sd=0.8), n(2, 10, sd=1.5), None, 4),
        ("mano_center_tip_zero_trans", "mano_right", n(2, 48, sd=0.8), n(2, 10, sd=1.5), f(np.zeros((2, 3))), 8),
    ]
    return out


def main():
    if not os.path.isdir(os.path.join(REF, "smplpytorch")):
        raise SystemExit("set P2M_REFERENCE_ROOT to a Pose2Mesh_RELEASE checkout")
    sys.path[:0] = [os.path.join(REF, "smplpytorch"), os.path.join(REF, "manopth")]
    from manopth.manolayer import ManoLayer
    from smplpytorch.pytorch.smpl_layer import SMPL_Layer

    torch.set_num_threads(1)
    ms = models()
    rng = np.random.RandomState(2025)
    Z = {f"digest_{k}": np.array(bm.digest(m)) for k, m in ms.items()}
    names = []
    for i, (name, mk, pose, betas, trans, center) in enumerate(cases(rng)):
        m = ms[mk]
        if mk == "smpl":
            layer = bm.smpl_reference_layer(SMPL_Layer, m, center_idx=center)
            n_joint = 24
        else:
            layer = bm.mano_reference_layer(ManoLayer, m, center_idx=center, flat_hand_mean=mk.endswith("_flat"))
            n_joint = 21
        layer = layer.double()
        seed = 1000 + i
        Z[f"{name}__model"] = np.array(mk)
        Z[f"{name}__pose"] = pose
        if betas is not None:
            Z[f"{name}__betas"] = betas
        if trans is not None:
            Z[f"{name}__trans"] = trans
        Z[f"{name}__center"] = np.array(-1 if center is None else center, np.int32)
        Z[f"{name}__seed"] = np.array(seed, np.int32)
        for mode in MODES:
            p = torch.from_numpy(pose).double().requires_grad_(True)
            args, inputs = {}, [("pose", p)]
            if betas is not None:
                args["th_betas"] = torch.from_numpy(betas).double().requires_grad_(True)
                inputs.append(("betas", args["th_betas"]))
            if trans is not None:
                args["th_trans"] = torch.from_numpy(trans).double().requires_grad_(True)
                inputs.append(("trans", args["th_trans"]))
            v, j = layer(p, **args)
            gv, gj = cotangents(seed, pose.shape[0], v.shape[1], n_joint, mode)
            loss = 0.0
            if gv is not None:
                loss = loss + (v * torch.from_numpy(gv).double()).sum()
            if gj is not None:
                loss = loss + (j * torch.from_numpy(gj).double()).sum()
            grads = torch.autograd.grad(loss, [t for _, t in inputs], allow_unused=True)
            for (k, t), g in zip(inputs, grads):
                g = np.zeros(tuple(t.shape)) if g is None else g.numpy()
                assert np.isfinite(g).all(), (name, mode, k)
                Z[f"{name}__{mode}__{k}"] = g
        names.append(name)
        print(f"{name:28s} B={pose.shape[0]}  |grad_pose| max {np.abs(Z[f'{name}__both__pose']).max():.3e}")
    Z["cases"] = np.array(names)
    path = os.path.join(HERE, "body_model_grad.npz")
    np.savez_compressed(path, **Z)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
