"""pose2mesh_release_b200 — the MeshNet hot path of hongsukchoi/Pose2Mesh_RELEASE, H100-native.

Public surface (mirrors the reference's modules for this path, SURVEY.md §8b):

    meshnet.Pose2Mesh / meshnet.get_model            <- lib/models/meshnet.py
    cheby_graph_conv.graph_conv_cheby                <- lib/models/backbones/cheby_graph_conv.py
    graph.build_coarse_graphs (+ coarsening helpers) <- lib/graph_utils.py, lib/coarsening.py
    install.install()                                 rebinding overlay for an unmodified reference checkout
    dist.DataParallelStep                             one-process-per-GPU data parallel, single NCCL all-reduce
    body_model.SMPLLayer / body_model.ManoLayer       <- smplpytorch SMPL_Layer, manopth ManoLayer (batched, forward)
    camera.fit_cameras                                <- demo/run.py optimize_cam_param (batched camera fit)
    temporal.smooth_pose / temporal.evaluate_video    <- lib/smooth_utils.py, compute_error_accel, the 3DPW video block
    freihand.FreiHANDEvaluator / freihand.f_scores    <- the FreiHAND evaluation script (F-scores, align_w_scale, PCK)
    render.render_meshes                              <- demo/renderer.py Renderer.render (batched mesh overlay)
    targets.Human36MTargets                           <- Human36M.__getitem__'s targets (batched, on the device)
    inputs.training_pose2d / inputs.synthesize_pose   <- the datasets' replace_joint_img, lib/noise_utils.py

All device work is in libp2m_b200.so (csrc/, C ABI in include/p2m_b200.h); there is no CPU fallback.
"""
from . import _lib  # noqa: F401
from .graph import build_coarse_graphs  # noqa: F401
from .meshnet import Pose2Mesh, get_model  # noqa: F401
from .cheby_graph_conv import graph_conv_cheby  # noqa: F401
from .body_model import ManoLayer, SMPLLayer  # noqa: F401
from .camera import convert_crop_cam_to_orig_img, fit_cameras  # noqa: F401
from .temporal import accel_errors, compute_error_accel, evaluate_video, smooth_pose, smooth_sequences  # noqa: F401
from .freihand import (FreiHANDEvaluator, align_w_scale, f_scores, mano_eval_regressor,  # noqa: F401
                       nearest_distances)
from . import render  # noqa: F401
from .render import render_meshes  # noqa: F401
from . import inputs  # noqa: F401

__version__ = "0.1.0"
