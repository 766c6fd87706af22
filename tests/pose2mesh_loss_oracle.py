"""TEST INFRASTRUCTURE ONLY — the Trainer's objective, lib/core/base.py:129-143, restated in torch on the mesh losses of
oracle/loss_oracle.py.  Parity status: PINNED against the unmodified reference classes composed as base.py:130-143
(tests/golden/pose2mesh_loss.npz, made by tests/golden/make_golden_pose2mesh_loss.py; tests/test_pose2mesh_loss_cpu.py).
"""
import numpy as np
import torch

from oracle.loss_oracle import coord_loss, edge_length_loss, normal_vector_loss


def pose2mesh_loss(cam_mesh, lift_pose, gt_mesh, gt_reg3dpose, gt_lift3dpose, mesh_valid, reg3dpose_valid,
                   lift3dpose_valid, face, joint_regressor, perm_reverse, weights=(0.1, 20.0, 1e-3), edge=True):
    """base.py:129-143 in the dtype of the inputs (float64 for a reference): the real rows of the padded output, the
    regressed joints (mm) and the five weighted terms.  Returns (loss, terms [5]); loss3 = 0 when edge is off."""
    n_vertex = int(np.max(face)) + 1
    pred_mesh = cam_mesh[:, torch.as_tensor(np.asarray(perm_reverse)[:n_vertex], dtype=torch.long)]
    pred_pose = torch.matmul(joint_regressor[None], pred_mesh * 1000)
    w_normal, w_edge, w_joint = weights
    l1 = coord_loss(pred_mesh, gt_mesh, mesh_valid)
    l2 = w_normal * normal_vector_loss(pred_mesh, gt_mesh, face)
    l3 = w_edge * edge_length_loss(pred_mesh, gt_mesh, face) if edge else cam_mesh.new_zeros(())
    l4 = w_joint * coord_loss(pred_pose, gt_reg3dpose, reg3dpose_valid)
    l5 = w_joint * coord_loss(lift_pose, gt_lift3dpose, lift3dpose_valid)
    return l1 + l2 + l3 + l4 + l5, torch.stack([l1, l2, l3, l4, l5])
