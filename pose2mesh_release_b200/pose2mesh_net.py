"""FlatPose2Mesh: drop-in for the reference's ``models.pose2mesh_net`` (lib/models/pose2mesh_net.py:8-29).

    pose3d       = PoseNet(pose2d)                      posenet.LinearModel      (SURVEY.md §8 row f1)
    pose_combine = cat(pose2d, pose3d.detach() / 1000)  fused into the native PoseNet call (eval and training)
    cam_mesh     = MeshNet(pose_combine)                meshnet.Pose2Mesh        (rows a1-a9)

``forward`` returns ``(cam_mesh, pose3d)`` like the reference; ``predict_vertices_and_joints`` additionally fuses the
callers' vertex gather and joint regression (lib/core/base.py:130-131; demo/run.py:170-171 — row f2).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import meshnet, posenet, postprocess


class FlatPose2Mesh(nn.Module):
    def __init__(self, num_joint, graph_L, posenet_pretrained: bool = False):
        super().__init__()
        self.num_joint = num_joint
        # attribute names = the reference's (state_dict prefixes `pose_lifter.` / `pose2mesh.`), constructed in its order
        self.pose_lifter = posenet.LinearModel(num_joint, linear_size=4096, num_stage=2, p_dropout=0.5,
                                               pretrained=posenet_pretrained)
        self.pose2mesh = meshnet.Pose2Mesh(2 + 3, 3, graph_L)

    def _lift(self, pose2d):
        """(pose3d [B, J, 3], pose_combine [B, J, 5]): one native call in eval mode and, for contiguous float32 CUDA
        tensors, in training mode; the reference's torch ops otherwise."""
        lifter, flat = self.pose_lifter, pose2d.reshape(len(pose2d), -1)
        if lifter.training and lifter.native_train_ok(flat):
            pose3d, combine = lifter.forward_train_native(flat, with_combine=True)
            return pose3d.reshape(-1, self.num_joint, 3), combine
        if not lifter.training and pose2d.is_cuda and not (torch.is_grad_enabled() and pose2d.requires_grad):
            pose3d, combine = lifter.forward_native(flat, with_combine=True)
            return pose3d.reshape(-1, self.num_joint, 3), combine
        pose3d = lifter(flat).reshape(-1, self.num_joint, 3)
        return pose3d, torch.cat((pose2d, pose3d.detach() / 1000), dim=2)

    def forward(self, pose2d):
        pose3d, combine = self._lift(pose2d)
        return self.pose2mesh(combine), pose3d

    @torch.no_grad()
    def predict_vertices_and_joints(self, pose2d, perm_reverse, n_vertex, joint_regressor):
        """Inference: real vertices [B, n_vertex, 3] (gather fused into MeshNet's head) and regressed joints
        [B, n_joint_out, 3] = joint_regressor @ vertices, plus pose3d."""
        lifter = self.pose_lifter
        pose3d, pose_combine = lifter.forward_native(pose2d.reshape(len(pose2d), -1), with_combine=True)
        verts = self.pose2mesh.forward_vertices(pose_combine, perm_reverse, n_vertex)
        joints = postprocess.regress_joints(verts, joint_regressor)
        return verts, joints, pose3d.reshape(-1, self.num_joint, 3)


def get_model(num_joint, graph_L):
    """lib/models/pose2mesh_net.py:25-28."""
    return FlatPose2Mesh(num_joint, graph_L)
