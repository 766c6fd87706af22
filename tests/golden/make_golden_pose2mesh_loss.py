#!/usr/bin/env python
"""Golden vectors of the Trainer's objective (lib/core/base.py:129-143): the UNMODIFIED reference loss classes
(lib/core/loss.py) on CPU in float64, composed as base.py:130-143 does, with autograd gradients with respect to the
padded model output and lift_pose.   python tests/golden/make_golden_pose2mesh_loss.py -> pose2mesh_loss.npz

Cases: a 6890-vertex sphere in 7168 padded rows (B = 1, 17 regressor joints) and a 778-vertex one in 1088 rows
(B = 3, 21 joints, whole zero samples in every mask), each with the edge term on and off."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden_loss import load_ref_loss  # noqa: E402
from oracle import ref_shim  # noqa: E402
from pose2mesh_loss_cases import INPUTS, make_case  # noqa: E402

CASES = {"smpl": (6890, 7168, 1, 17, 17, 31), "mano": (778, 1088, 3, 21, 21, 32)}
WEIGHTS = (0.1, 20.0, 1e-3)   # normal, edge, joint: every released yml


def reference_objective(ref_loss, c, edge):
    """base.py:130-143 line for line (graph_perm_reverse, mesh_model.face, J_regressor, the loss list of get_loss)."""
    loss_list = ref_loss.get_loss(c["face"])
    normal_weight, edge_weight, joint_weight = WEIGHTS
    model_out = c["cam_mesh"].double().requires_grad_(True)
    lift_pose = c["lift_pose"].double().requires_grad_(True)
    gt_mesh, gt_reg3dpose, gt_lift3dpose = (c[k].double() for k in ("gt_mesh", "gt_reg3dpose", "gt_lift3dpose"))
    val_mesh, val_reg3dpose, val_lift3dpose = (c[k].double() for k in ("mesh_valid", "reg3dpose_valid",
                                                                       "lift3dpose_valid"))
    J_regressor = c["joint_regressor"].double()
    pred_mesh = model_out[:, c["perm_reverse"][:c["face"].max() + 1], :]
    pred_pose = torch.matmul(J_regressor[None, :, :], pred_mesh * 1000)
    loss1, loss2, loss4, loss5 = loss_list[0](pred_mesh, gt_mesh, val_mesh), \
        normal_weight * loss_list[1](pred_mesh, gt_mesh), \
        joint_weight * loss_list[3](pred_pose, gt_reg3dpose, val_reg3dpose), \
        joint_weight * loss_list[4](lift_pose, gt_lift3dpose, val_lift3dpose)
    loss3 = 0
    loss = loss1 + loss2 + loss3 + loss4 + loss5
    if edge:
        loss3 = edge_weight * loss_list[2](pred_mesh, gt_mesh)
        loss += loss3
    loss.backward()
    terms = [float(torch.as_tensor(t).detach()) for t in (loss1, loss2, loss3, loss4, loss5)]
    return float(loss.detach()), np.array(terms), model_out.grad.numpy(), lift_pose.grad.numpy()


if __name__ == "__main__":
    ref_loss = load_ref_loss()
    out = {"weights": np.array(WEIGHTS)}
    for name, size in CASES.items():
        c = make_case(*size)
        for k in INPUTS + ("joint_regressor",):
            out[f"{name}/{k}"] = c[k].numpy()
        out[f"{name}/face"] = c["face"].astype(np.int32)
        out[f"{name}/perm_reverse"] = c["perm_reverse"].astype(np.int32)
        nv = int(c["face"].max()) + 1
        for edge in (False, True):
            with ref_shim.cpu_cuda_noop():
                loss, terms, g_mesh, g_lift = reference_objective(ref_loss, c, edge)
            pad = np.ones(g_mesh.shape[1], bool)
            pad[c["perm_reverse"][:nv]] = False
            assert not g_mesh[:, pad].any()
            tag = f"{name}/edge{int(edge)}"
            out[f"{tag}/loss"], out[f"{tag}/terms"] = np.float64(loss), terms
            # the gradient's real rows in vertex order (its padding rows are zero), rounded to float32
            out[f"{tag}/grad_mesh"] = g_mesh[:, c["perm_reverse"][:nv]].astype(np.float32)
            out[f"{tag}/grad_lift"] = g_lift.astype(np.float32)
    path = os.path.join(HERE, "pose2mesh_loss.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))
