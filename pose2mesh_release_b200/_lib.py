"""ctypes binding of libp2m_b200.so (C ABI declared in include/p2m_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails, a
RuntimeError is raised (the product has no CPU / eager path — north_star, SURVEY.md §7).
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libp2m_b200.so")

P2M_PREC_FP32_SIMT = 0
P2M_PREC_FP16X3_TC = 1
P2M_PREC_FP16_TC = 2  # inference only: single-pass fp16 operands in the Chebyshev convs (include/p2m_b200.h)
P2M_PREC_FP16_MIXED_TC = 3  # training too: single-pass fp16 in the forward, backward-data and weight-gradient convs
PRECISIONS = {"fp32": P2M_PREC_FP32_SIMT, "fp16x3": P2M_PREC_FP16X3_TC, "fp16": P2M_PREC_FP16_TC,
              "fp16_mixed": P2M_PREC_FP16_MIXED_TC}


def default_precision() -> int:
    """Precision of new modules / graph handles: the tensor-core path (fp16x3: error-compensated split, fp32
    accumulate, 1e-4 parity like the fp32 path) unless the environment says ``P2M_PRECISION=fp32`` (the CUDA-core
    escape hatch for activations beyond fp16's range), ``P2M_PRECISION=fp16`` (single-pass fp16 Chebyshev convs,
    inference only) or ``P2M_PRECISION=fp16_mixed`` (single-pass fp16 in the training forward and backward as well:
    fp16 operands, fp32 accumulation, fp32 weights and BatchNorm).  A drop-in user (install.py) therefore gets the
    fast path without touching the module; ``Pose2Mesh.set_precision`` / ``set_default_precision`` still override
    it."""
    name = os.environ.get("P2M_PRECISION", "fp16x3").strip().lower()
    if name not in PRECISIONS:
        raise RuntimeError(f"P2M_PRECISION={name!r}: expected one of {sorted(PRECISIONS)}")
    return PRECISIONS[name]

c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)
c_int64_p = C.POINTER(C.c_int64)


class ModelDesc(C.Structure):
    _fields_ = [
        ("n_levels", C.c_int32),
        ("level_size", c_int32_p),
        ("rowptr", C.POINTER(c_int32_p)),
        ("colidx", C.POINTER(c_int32_p)),
        ("values", C.POINTER(c_float_p)),
        ("n_blocks", C.c_int32),
        ("block_len", c_int32_p),
        ("block_chans", c_int32_p),
        ("device", C.c_int32),
    ]


class Params(C.Structure):
    _fields_ = [
        ("fc_w", C.c_void_p),
        ("fc_b", C.c_void_p),
        ("cl_w", C.POINTER(C.c_void_p)),
        ("cl_b", C.POINTER(C.c_void_p)),
        ("bn_w", C.POINTER(C.c_void_p)),
        ("bn_b", C.POINTER(C.c_void_p)),
        ("bn_rm", C.POINTER(C.c_void_p)),
        ("bn_rv", C.POINTER(C.c_void_p)),
        ("bn_nbt", C.POINTER(C.c_void_p)),
    ]


P2M_BN_BATCH_UPDATE = 0
P2M_BN_BATCH = 1
P2M_BN_RUNNING = 2


class BnOpts(C.Structure):
    """p2m_bn_opts_t: what one BatchNorm's forward reads (statistics mode, momentum None, momentum, eps)."""
    _fields_ = [("stats", C.c_int32), ("cumulative", C.c_int32), ("momentum", C.c_double), ("eps", C.c_double)]


class ConvFwdArgs(C.Structure):
    _fields_ = [
        ("level", C.c_int32), ("batch", C.c_int32), ("fin", C.c_int32), ("fout", C.c_int32),
        ("x", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p),
        ("bn_mode", C.c_int32),
        ("bn_weight", C.c_void_p), ("bn_bias", C.c_void_p),
        ("bn_running_mean", C.c_void_p), ("bn_running_var", C.c_void_p),
        ("bn_num_batches_tracked", C.c_void_p),
        ("save_mean", C.c_void_p), ("save_invstd", C.c_void_p),
        ("relu", C.c_int32),
        ("y", C.c_void_p),
    ]


class ConvBwdArgs(C.Structure):
    _fields_ = [
        ("level", C.c_int32), ("batch", C.c_int32), ("fin", C.c_int32), ("fout", C.c_int32),
        ("x", C.c_void_p), ("weight", C.c_void_p), ("dz", C.c_void_p),
        ("dx", C.c_void_p), ("dweight", C.c_void_p), ("dbias", C.c_void_p),
    ]


class Capture(C.Structure):
    """p2m_capture_t: per-layer device buffers the network schedules copy their tensors into (p2m_debug_set_capture)."""
    _fields_ = [
        ("z", C.POINTER(C.c_void_p)), ("a", C.POINTER(C.c_void_p)), ("y", C.POINTER(C.c_void_p)),
        ("fc_out", C.c_void_p),
        ("g_a", C.POINTER(C.c_void_p)), ("g_z", C.POINTER(C.c_void_p)), ("dx", C.POINTER(C.c_void_p)),
        ("fc_dx", C.c_void_p),
    ]


class Pose2MeshLossArgs(C.Structure):
    """p2m_pose2mesh_loss_args_t: the Trainer's objective (sizes, then device pointers)."""
    _fields_ = [(n, C.c_int32) for n in ("batch", "n_padded", "n_vertex", "n_face", "n_reg_joint", "n_lift_joint")] + [
        (n, C.c_void_p) for n in ("cam_mesh", "lift_pose", "gt_mesh", "gt_reg3dpose", "gt_lift3dpose", "mesh_valid",
                                  "reg3dpose_valid", "lift3dpose_valid", "faces", "joint_regressor", "perm_reverse",
                                  "weights", "edge", "pred_pose", "scratch", "loss", "terms", "grad_loss",
                                  "d_cam_mesh", "d_lift_pose")]


P2M_POSE2MESH_MAX_REG_JOINT = 24


class PoseNetStage(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1_w", "w1_b", "w2_w", "w2_b", "bn1_w", "bn1_b", "bn1_rm", "bn1_rv",
                                          "bn2_w", "bn2_b", "bn2_rm", "bn2_rv")]


class PoseNetParams(C.Structure):
    _fields_ = [("num_joint", C.c_int32), ("hidden", C.c_int32), ("num_stage", C.c_int32),
                ("w1_w", C.c_void_p), ("w1_b", C.c_void_p), ("w2_w", C.c_void_p), ("w2_b", C.c_void_p),
                ("stages", C.POINTER(PoseNetStage))]


class PoseNetTrainStage(C.Structure):
    _fields_ = [("bn1_nbt", C.c_void_p), ("bn2_nbt", C.c_void_p)]


class PoseNetTrain(C.Structure):
    _fields_ = [("stages", C.POINTER(PoseNetTrainStage))]


class PoseNetStageGrads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1_w", "w1_b", "w2_w", "w2_b", "bn1_w", "bn1_b", "bn2_w", "bn2_b")]


class PoseNetGrads(C.Structure):
    _fields_ = [("w1_w", C.c_void_p), ("w1_b", C.c_void_p), ("w2_w", C.c_void_p), ("w2_b", C.c_void_p),
                ("stages", C.POINTER(PoseNetStageGrads))]


class PoseNetCapture(C.Structure):
    """p2m_posenet_capture_t: device buffers the PoseNet backward copies its intermediates into
    (p2m_debug_posenet_backward_capture); the per-stage fields are [num_stage] arrays, scale[s] a float[4]."""
    _fields_ = [(n, C.POINTER(C.c_void_p)) for n in ("g_y", "a2", "g_a2", "g_z2", "a1", "g_a1", "g_bn1", "scale")] + [
        ("g_y0", C.c_void_p)]


class BodyModelDesc(C.Structure):
    _fields_ = [
        ("n_vertex", C.c_int32), ("n_joint", C.c_int32), ("n_betas", C.c_int32), ("n_out_joints", C.c_int32),
        ("v_template", c_float_p), ("shapedirs", c_float_p), ("posedirs", c_float_p), ("J_regressor", c_float_p),
        ("weights", c_float_p), ("parents", c_int32_p), ("model_betas", c_float_p), ("pose_mean", c_float_p),
        ("joint_map", c_int32_p), ("scale", C.c_float), ("device", C.c_int32),
    ]


P2M_BETAS_ZERO_MEANS_MODEL = 0
P2M_BETAS_AS_GIVEN = 1

P2M_FRAME_ROTATE_ROOT = 1
P2M_FRAME_CLAMP_BETAS = 2
P2M_FRAME_ZERO_BETAS_MODEL = 4
P2M_FRAME_LAYER_TRANS_T = 8
P2M_FRAME_LAYER_TRANS = 16
P2M_FRAME_H36M_COMPENSATE = 32
P2M_FRAME_ADD_T = 64
P2M_FRAME_TO_MM = 128

P2M_JOINTS_HUMAN36 = 0
P2M_JOINTS_COCO = 1
P2M_JOINTS_SMPL = 2
P2M_JOINTS_MANO = 3
P2M_DATASET_HUMAN36M = 0
P2M_DATASET_COCO = 1
P2M_DATASET_MUCO = 2
P2M_DATASET_AMASS = 3
P2M_DATASET_PW3D = 4
P2M_DATASET_SURREAL = 5
P2M_DATASET_FREIHAND = 6

P2M_CAM_INPUT_F64 = 0
P2M_CAM_INPUT_INT = 1
P2M_CAM_INPUT_F32 = 2

P2M_DTYPE_F32 = 0
P2M_DTYPE_F64 = 1

P2M_NOISE_NONE = 0
P2M_NOISE_COCO = 1
P2M_NOISE_H36M = 2
P2M_AREA_TIGHT = 0
P2M_AREA_CROP = 1


class RmspropSegment(C.Structure):
    """p2m_rmsprop_segment_t: one parameter tensor of an RMSprop step (device pointers, element count, group)."""
    _fields_ = [(n, C.c_void_p) for n in ("param", "grad", "square_avg", "momentum_buffer", "grad_avg", "step")] + [
        ("numel", C.c_int64), ("group", C.c_int32)]


class RmspropGroup(C.Structure):
    """p2m_rmsprop_group_t: one param group's hyperparameters (lr_device: a device float32 lr, or None for lr)."""
    _fields_ = [("lr", C.c_double), ("lr_device", C.c_void_p), ("alpha", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double), ("momentum", C.c_double), ("centered", C.c_int32)]


class H36MError(C.Structure):
    _fields_ = [("mean", C.c_double * 2), ("std", C.c_double * 2), ("weight", C.c_double)]


EXPORTS = [
    "p2m_model_create", "p2m_model_destroy", "p2m_model_num_layers", "p2m_model_layer_info",
    "p2m_model_set_precision", "p2m_debug_kernel_status", "p2m_debug_set_trace", "p2m_debug_set_fuse_head", "p2m_debug_set_elide_padding", "p2m_debug_set_dedup_padding", "p2m_debug_conv_path", "p2m_debug_conv_tiling", "p2m_debug_tile_families", "p2m_debug_set_sm_count", "p2m_debug_layer_route", "p2m_debug_set_capture", "p2m_model_set_profiling", "p2m_model_layer_times_ms", "p2m_meshnet_workspace_bytes", "p2m_meshnet_backward_scratch_bytes",
    "p2m_meshnet_forward", "p2m_meshnet_backward", "p2m_meshnet_workspace_bytes_opts", "p2m_meshnet_forward_opts",
    "p2m_meshnet_backward_opts", "p2m_model_set_output_gather", "p2m_meshnet_forward_vertices", "p2m_meshnet_host_io_bytes", "p2m_meshnet_forward_host", "p2m_meshnet_forward_vertices_host",
    "p2m_cheb_conv_workspace_bytes", "p2m_cheb_conv_fwd", "p2m_cheb_conv_bwd", "p2m_graph_match_level", "p2m_posenet_workspace_bytes", "p2m_posenet_forward",
    "p2m_posenet_train_workspace_bytes", "p2m_posenet_train_saved_bytes", "p2m_posenet_train_forward", "p2m_posenet_backward",
    "p2m_posenet_forward_opts", "p2m_posenet_train_forward_opts", "p2m_posenet_backward_opts",
    "p2m_debug_posenet_backward_capture",
    "p2m_regress_joints", "p2m_regress_joints_backward", "p2m_normalize_pose2d", "p2m_mesh_losses", "p2m_coord_loss",
    "p2m_pose2mesh_loss", "p2m_pose2mesh_loss_backward",
    "p2m_rigid_align", "p2m_point_errors", "p2m_fit_camera", "p2m_crop_cam_to_orig",
    "p2m_one_euro_smooth", "p2m_accel_error", "p2m_segment_mean",
    "p2m_nearest_distances", "p2m_align_w_scale", "p2m_pck_accumulate",
    "p2m_render_workspace_bytes", "p2m_render_meshes",
    "p2m_body_model_create", "p2m_body_model_destroy", "p2m_body_model_workspace_bytes", "p2m_body_model_forward",
    "p2m_body_model_backward_workspace_bytes", "p2m_body_model_backward",
    "p2m_camera_frame_workspace_bytes", "p2m_camera_frame_coords", "p2m_h36m_regressors_create",
    "p2m_h36m_regressors_destroy", "p2m_h36m_targets", "p2m_synthesize_pose", "p2m_h36m_syn_error",
    "p2m_training_pose2d", "p2m_augm_params", "p2m_training_pose2d_augmented", "p2m_sample_targets",
    "p2m_layer_joint_targets", "p2m_rmsprop_step",
    "p2m_last_error", "p2m_version", "p2m_launch_count", "p2m_launch_count_reset",
    "p2m_debug_conv_log", "p2m_debug_conv_log_reset",
]

_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """Load (once) and type the shared library.  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m pose2mesh_release_b200.build` "
                "(or __graft_entry__.build()).  pose2mesh_release_b200 has no CPU / eager fallback.")
        lib = C.CDLL(LIB_PATH)
        vp, i32, i64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
        lib.p2m_model_create.argtypes = [C.POINTER(ModelDesc), C.POINTER(vp)]
        lib.p2m_model_create.restype = C.c_int
        lib.p2m_model_destroy.argtypes = [vp]
        lib.p2m_model_destroy.restype = None
        lib.p2m_model_num_layers.argtypes = [vp]
        lib.p2m_model_num_layers.restype = C.c_int
        lib.p2m_model_layer_info.argtypes = [vp, C.c_int, c_int32_p]
        lib.p2m_model_layer_info.restype = C.c_int
        lib.p2m_model_set_precision.argtypes = [vp, C.c_int]
        lib.p2m_model_set_precision.restype = C.c_int
        lib.p2m_model_set_profiling.argtypes = [vp, C.c_int]
        lib.p2m_model_set_profiling.restype = C.c_int
        lib.p2m_model_layer_times_ms.argtypes = [vp, c_float_p, C.c_int]
        lib.p2m_model_layer_times_ms.restype = C.c_int
        lib.p2m_debug_set_fuse_head.argtypes = [vp, C.c_int]
        lib.p2m_debug_set_fuse_head.restype = C.c_int
        lib.p2m_debug_set_elide_padding.argtypes = [vp, C.c_int]
        lib.p2m_debug_set_elide_padding.restype = C.c_int
        lib.p2m_debug_set_dedup_padding.argtypes = [vp, C.c_int]
        lib.p2m_debug_set_dedup_padding.restype = C.c_int
        lib.p2m_debug_set_trace.argtypes = [vp, vp]
        lib.p2m_debug_set_trace.restype = C.c_int
        lib.p2m_debug_conv_path.argtypes = [vp, C.c_int, C.c_int, C.c_int, c_int32_p]
        lib.p2m_debug_conv_path.restype = C.c_int
        lib.p2m_debug_conv_tiling.argtypes = [vp, C.c_int, C.c_int, C.c_int, c_int32_p]
        lib.p2m_debug_conv_tiling.restype = C.c_int
        lib.p2m_debug_tile_families.argtypes = [vp, C.c_int, C.c_int, C.c_int, c_int32_p]
        lib.p2m_debug_tile_families.restype = C.c_int
        lib.p2m_debug_set_sm_count.argtypes = [vp, C.c_int]
        lib.p2m_debug_set_sm_count.restype = C.c_int
        lib.p2m_debug_layer_route.argtypes = [vp, C.c_int, C.c_int, C.c_int, c_int32_p]
        lib.p2m_debug_layer_route.restype = C.c_int
        lib.p2m_debug_set_capture.argtypes = [vp, C.POINTER(Capture)]
        lib.p2m_debug_set_capture.restype = C.c_int
        lib.p2m_debug_kernel_status.argtypes = [vp, c_int32_p]
        lib.p2m_debug_kernel_status.restype = C.c_int
        lib.p2m_meshnet_workspace_bytes.argtypes = [vp, C.c_int, C.c_int]
        lib.p2m_meshnet_workspace_bytes.restype = sz
        lib.p2m_meshnet_backward_scratch_bytes.argtypes = [vp, C.c_int]
        lib.p2m_meshnet_backward_scratch_bytes.restype = sz
        lib.p2m_meshnet_host_io_bytes.argtypes = [vp, C.c_int]
        lib.p2m_meshnet_host_io_bytes.restype = sz
        lib.p2m_meshnet_forward.argtypes = [vp, C.POINTER(Params), vp, vp, C.c_int, C.c_int, vp, sz, vp]
        lib.p2m_meshnet_forward.restype = C.c_int
        lib.p2m_model_set_output_gather.argtypes = [vp, c_int32_p, C.c_int]
        lib.p2m_model_set_output_gather.restype = C.c_int
        lib.p2m_meshnet_forward_vertices.argtypes = [vp, C.POINTER(Params), vp, vp, C.c_int, vp, sz, vp]
        lib.p2m_meshnet_forward_vertices.restype = C.c_int
        lib.p2m_meshnet_forward_host.argtypes = [vp, C.POINTER(Params), vp, vp, C.c_int, vp, sz, vp]
        lib.p2m_meshnet_forward_host.restype = C.c_int
        lib.p2m_meshnet_forward_vertices_host.argtypes = [vp, C.POINTER(Params), vp, vp, C.c_int, vp, sz, vp]
        lib.p2m_meshnet_forward_vertices_host.restype = C.c_int
        lib.p2m_meshnet_backward.argtypes = [vp, C.POINTER(Params), C.POINTER(Params), vp, vp, vp, C.c_int, vp, sz,
                                             vp, sz, vp]
        lib.p2m_meshnet_backward.restype = C.c_int
        bn_p = C.POINTER(BnOpts)
        lib.p2m_meshnet_workspace_bytes_opts.argtypes = [vp, C.c_int, C.c_int, bn_p]
        lib.p2m_meshnet_workspace_bytes_opts.restype = sz
        lib.p2m_meshnet_forward_opts.argtypes = [vp, C.POINTER(Params), bn_p, vp, vp, C.c_int, C.c_int, vp, sz, vp]
        lib.p2m_meshnet_forward_opts.restype = C.c_int
        lib.p2m_meshnet_backward_opts.argtypes = [vp, C.POINTER(Params), C.POINTER(Params), bn_p, vp, vp, vp, C.c_int,
                                                  vp, sz, vp, sz, vp]
        lib.p2m_meshnet_backward_opts.restype = C.c_int
        lib.p2m_cheb_conv_workspace_bytes.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.p2m_cheb_conv_workspace_bytes.restype = sz
        lib.p2m_cheb_conv_fwd.argtypes = [vp, C.POINTER(ConvFwdArgs), vp, sz, vp]
        lib.p2m_cheb_conv_fwd.restype = C.c_int
        lib.p2m_cheb_conv_bwd.argtypes = [vp, C.POINTER(ConvBwdArgs), vp, sz, vp]
        lib.p2m_cheb_conv_bwd.restype = C.c_int
        lib.p2m_posenet_workspace_bytes.argtypes = [C.c_int, C.c_int]
        lib.p2m_posenet_workspace_bytes.restype = sz
        lib.p2m_posenet_forward.argtypes = [C.POINTER(PoseNetParams), vp, vp, vp, C.c_int, vp, sz, vp]
        lib.p2m_posenet_forward.restype = C.c_int
        for fn in (lib.p2m_posenet_train_workspace_bytes, lib.p2m_posenet_train_saved_bytes):
            fn.argtypes = [C.c_int] * 4
            fn.restype = sz
        lib.p2m_posenet_train_forward.argtypes = [C.POINTER(PoseNetParams), C.POINTER(PoseNetTrain), vp, C.c_int,
                                                  C.c_float, vp, vp, vp, vp, sz, vp, sz, vp]
        lib.p2m_posenet_train_forward.restype = C.c_int
        lib.p2m_posenet_backward.argtypes = [C.POINTER(PoseNetParams), vp, C.c_int, C.c_float, vp, vp, sz, vp,
                                             C.POINTER(PoseNetGrads), vp, vp, sz, vp]
        lib.p2m_posenet_backward.restype = C.c_int
        lib.p2m_posenet_forward_opts.argtypes = [C.POINTER(PoseNetParams), bn_p, vp, vp, vp, C.c_int, vp, sz, vp]
        lib.p2m_posenet_forward_opts.restype = C.c_int
        lib.p2m_posenet_train_forward_opts.argtypes = [C.POINTER(PoseNetParams), C.POINTER(PoseNetTrain), bn_p,
                                                       c_float_p, vp, C.c_int, vp, vp, vp, vp, sz, vp, sz, vp]
        lib.p2m_posenet_train_forward_opts.restype = C.c_int
        lib.p2m_posenet_backward_opts.argtypes = [C.POINTER(PoseNetParams), bn_p, c_float_p, vp, C.c_int, vp, vp, sz,
                                                  vp, C.POINTER(PoseNetGrads), vp, vp, sz, vp]
        lib.p2m_posenet_backward_opts.restype = C.c_int
        lib.p2m_debug_posenet_backward_capture.argtypes = (lib.p2m_posenet_backward_opts.argtypes[:-1]
                                                           + [C.POINTER(PoseNetCapture), vp])
        lib.p2m_debug_posenet_backward_capture.restype = C.c_int
        lib.p2m_regress_joints.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        lib.p2m_regress_joints.restype = C.c_int
        lib.p2m_regress_joints_backward.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        lib.p2m_regress_joints_backward.restype = C.c_int
        lib.p2m_normalize_pose2d.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        lib.p2m_normalize_pose2d.restype = C.c_int
        lib.p2m_mesh_losses.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
        lib.p2m_mesh_losses.restype = C.c_int
        lib.p2m_coord_loss.argtypes = [vp, vp, vp, i64, vp, vp, vp, vp]
        lib.p2m_coord_loss.restype = C.c_int
        for fn in (lib.p2m_pose2mesh_loss, lib.p2m_pose2mesh_loss_backward):
            fn.argtypes = [C.POINTER(Pose2MeshLossArgs), vp]
            fn.restype = C.c_int
        lib.p2m_rigid_align.argtypes = [vp, vp, C.c_int, C.c_int, c_int32_p, C.c_int, vp, vp, vp, vp, vp]
        lib.p2m_rigid_align.restype = C.c_int
        lib.p2m_point_errors.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, c_int32_p, C.c_int, C.c_int, vp, vp, vp]
        lib.p2m_point_errors.restype = C.c_int
        lib.p2m_fit_camera.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int,
                                       c_int32_p, C.POINTER(C.c_double), C.c_int, vp, vp, vp, vp, vp, vp, vp]
        lib.p2m_fit_camera.restype = C.c_int
        lib.p2m_crop_cam_to_orig.argtypes = [vp, vp, vp, C.c_int, vp, vp]
        lib.p2m_crop_cam_to_orig.restype = C.c_int
        lib.p2m_one_euro_smooth.argtypes = [C.c_int, vp, vp, i64, c_int64_p, C.c_int, i64, C.c_double, C.c_double,
                                            C.c_double, vp]
        lib.p2m_one_euro_smooth.restype = C.c_int
        lib.p2m_accel_error.argtypes = [C.c_int, vp, vp, C.c_int, c_int64_p, C.c_int, i64, vp, vp, vp, vp, vp]
        lib.p2m_accel_error.restype = C.c_int
        lib.p2m_segment_mean.argtypes = [C.c_int, vp, i64, c_int64_p, C.c_int, i64, vp, vp, vp]
        lib.p2m_segment_mean.restype = C.c_int
        c_double_p = C.POINTER(C.c_double)
        lib.p2m_nearest_distances.argtypes = [C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, c_double_p, C.c_int, vp, vp,
                                              vp, vp, vp, vp]
        lib.p2m_nearest_distances.restype = C.c_int
        lib.p2m_align_w_scale.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
        lib.p2m_align_w_scale.restype = C.c_int
        lib.p2m_pck_accumulate.argtypes = [vp, vp, vp, i64, c_double_p, C.c_int, vp, vp, vp]
        lib.p2m_pck_accumulate.restype = C.c_int
        lib.p2m_render_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.p2m_render_workspace_bytes.restype = sz
        lib.p2m_render_meshes.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int,
                                          vp, vp, vp, vp, vp, sz, vp]
        lib.p2m_render_meshes.restype = C.c_int
        lib.p2m_body_model_create.argtypes = [C.POINTER(BodyModelDesc), C.POINTER(vp)]
        lib.p2m_body_model_create.restype = C.c_int
        lib.p2m_body_model_destroy.argtypes = [vp]
        lib.p2m_body_model_destroy.restype = None
        lib.p2m_body_model_workspace_bytes.argtypes = [vp, C.c_int]
        lib.p2m_body_model_workspace_bytes.restype = sz
        lib.p2m_body_model_forward.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, C.c_int, vp, sz, vp]
        lib.p2m_body_model_forward.restype = C.c_int
        lib.p2m_body_model_backward_workspace_bytes.argtypes = [vp, C.c_int]
        lib.p2m_body_model_backward_workspace_bytes.restype = sz
        lib.p2m_body_model_backward.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp, sz,
                                                vp]
        lib.p2m_body_model_backward.restype = C.c_int
        lib.p2m_camera_frame_workspace_bytes.argtypes = [vp, C.c_int]
        lib.p2m_camera_frame_workspace_bytes.restype = sz
        lib.p2m_camera_frame_coords.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, c_int32_p, C.c_int, vp, vp, C.c_int,
                                                vp, sz, vp]
        lib.p2m_camera_frame_coords.restype = C.c_int
        lib.p2m_h36m_regressors_create.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_int,
                                                   C.POINTER(vp)]
        lib.p2m_h36m_regressors_create.restype = C.c_int
        lib.p2m_h36m_regressors_destroy.argtypes = [vp]
        lib.p2m_h36m_regressors_destroy.restype = None
        lib.p2m_h36m_targets.argtypes = [vp, C.c_int, C.c_float, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp,
                                         vp, vp]
        lib.p2m_h36m_targets.restype = C.c_int
        lib.p2m_synthesize_pose.argtypes = [vp, vp, vp, C.c_int, vp, vp]
        lib.p2m_synthesize_pose.restype = C.c_int
        lib.p2m_h36m_syn_error.argtypes = [C.POINTER(H36MError), vp, C.c_int, vp, vp]
        lib.p2m_h36m_syn_error.restype = C.c_int
        lib.p2m_training_pose2d.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.POINTER(H36MError),
                                            vp, C.c_int, C.c_int, vp, vp]
        lib.p2m_training_pose2d.restype = C.c_int
        lib.p2m_augm_params.argtypes = [C.c_int, C.c_int, C.c_double, vp, vp, vp, vp]
        lib.p2m_augm_params.restype = C.c_int
        lib.p2m_training_pose2d_augmented.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int,
                                                      C.POINTER(H36MError), vp, C.c_int, C.c_int, vp, vp, C.c_int,
                                                      C.c_int, vp, vp]
        lib.p2m_training_pose2d_augmented.restype = C.c_int
        lib.p2m_sample_targets.argtypes = [vp, C.c_int, C.c_int, C.c_float, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp,
                                           vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.p2m_sample_targets.restype = C.c_int
        lib.p2m_layer_joint_targets.argtypes = [C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, vp, vp,
                                                vp, vp, vp, vp, vp, vp, vp, vp]
        lib.p2m_layer_joint_targets.restype = C.c_int
        lib.p2m_rmsprop_step.argtypes = [C.POINTER(RmspropSegment), C.c_int, C.POINTER(RmspropGroup), C.c_int, vp]
        lib.p2m_rmsprop_step.restype = C.c_int
        lib.p2m_graph_match_level.argtypes = [i64, c_int32_p, c_int32_p, C.POINTER(C.c_double), c_int64_p,
                                              C.POINTER(C.c_double), c_int32_p]
        lib.p2m_graph_match_level.restype = i32
        lib.p2m_last_error.argtypes = []
        lib.p2m_last_error.restype = C.c_char_p
        lib.p2m_version.argtypes = []
        lib.p2m_version.restype = C.c_char_p
        lib.p2m_launch_count.argtypes = []
        lib.p2m_launch_count.restype = i64
        lib.p2m_launch_count_reset.argtypes = []
        lib.p2m_launch_count_reset.restype = None
        lib.p2m_debug_conv_log.argtypes = [c_int32_p, C.c_int]
        lib.p2m_debug_conv_log.restype = i64
        lib.p2m_debug_conv_log_reset.argtypes = []
        lib.p2m_debug_conv_log_reset.restype = None
        _lib = lib
    return _lib


CONV_LOG_FIELDS = ("kind", "nc", "ns", "xs", "mode", "f16", "grid_x", "grid_y", "n_tiles")
TC_KINDS = ("conv", "dw", "gemm")


def conv_log(reset: bool = False) -> list:
    """Debug: the tensor-core launches logged since the last reset (p2m_debug_conv_log), one dict per launch with
    the fields of CONV_LOG_FIELDS (kind as a TC_KINDS name) and tiles_per_cta = ceil(n_tiles / grid_x).  Raises if the
    log overflowed.  reset: clear the log after reading it."""
    lib = load()
    n = lib.p2m_debug_conv_log(None, 0)
    buf = (C.c_int32 * (9 * max(n, 1)))()
    if lib.p2m_debug_conv_log(buf, n) != n:
        raise RuntimeError("conv log: launches were logged while it was read")
    if n > 32768:
        raise RuntimeError(f"conv log overflowed: {n} launches, 32768 stored")
    if reset:
        lib.p2m_debug_conv_log_reset()
    out = []
    for i in range(n):
        e = dict(zip(CONV_LOG_FIELDS, buf[9 * i:9 * i + 9]))
        e["kind"] = TC_KINDS[e["kind"]]
        e["tiles_per_cta"] = -(-e["n_tiles"] // e["grid_x"])
        out.append(e)
    return out


TILE_FAMILIES = ("consecutive", "real", "iso", "rep")
TILE_CONFIGS = ("t1_fp16x3", "plain_fp16x3", "t1_fp16", "plain_fp16")


def tile_families(handle, level: int, fin: int, fout: int) -> dict:
    """Debug: a model handle's tile families on `level` (p2m_debug_tile_families, host only).  Returns
    {family: {128: d, 64: d}} for the TILE_FAMILIES, d = {"n_pattern", "max_h1", "stride"} plus, per TILE_CONFIGS
    name, the (output columns per CTA, ring slots, X stages) a conv fin -> fout would launch with on those tiles
    ((0, 0, 0): does not fit, or not the tile size the conv runs on)."""
    out = (C.c_int32 * 120)()
    check(load().p2m_debug_tile_families(handle, level, fin, fout, out), "tile_families")
    res = {}
    for f, fam in enumerate(TILE_FAMILIES):
        res[fam] = {}
        for k, tm in enumerate((128, 64)):
            o = out[(2 * f + k) * 15:(2 * f + k + 1) * 15]
            d = dict(n_pattern=o[0], max_h1=o[1], stride=o[2])
            d.update({name: tuple(o[3 + 3 * c:6 + 3 * c]) for c, name in enumerate(TILE_CONFIGS)})
            res[fam][tm] = d
    return res


def check(status: int, what: str = "p2m call"):
    if status != 0:
        msg = load().p2m_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (status {status}): {msg}")


def call(name: str, device, *args):
    """Run entry point `name` on `args` (a tensor is passed as its data pointer) with the current stream of `device`
    as the last argument, which every stream-taking entry point has; raise RuntimeError if it fails.  The library
    picks the device to run on itself (the handle's, or the data arrays'), so no device context is needed here."""
    fn = getattr(load(), name)
    ptrs = (a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args)
    check(fn(*ptrs, torch.cuda.current_stream(device).cuda_stream), name)


def bn_opts(bn) -> BnOpts:
    """The p2m_bn_opts_t of an nn.BatchNorm1d in its current state, by torch's _BatchNorm.forward: batch statistics when
    it is in training mode or has no running buffers, an update of the buffers only in training mode with
    track_running_stats, momentum None as the cumulative average.  ValueError for what the native kernels do not
    implement: another module type in a BatchNorm's place, or affine=False."""
    if not isinstance(bn, torch.nn.BatchNorm1d):
        raise ValueError(f"pose2mesh_release_b200: expected an nn.BatchNorm1d, got {type(bn).__name__}")
    if not bn.affine:
        raise ValueError("pose2mesh_release_b200: BatchNorm1d(affine=False) is not supported by the native kernels")
    batch = bn.training or (bn.running_mean is None and bn.running_var is None)
    update = bn.training and bn.track_running_stats
    o = BnOpts()
    o.stats = P2M_BN_RUNNING if not batch else (P2M_BN_BATCH_UPDATE if update else P2M_BN_BATCH)
    o.cumulative = int(bn.momentum is None)
    o.momentum = 0.0 if bn.momentum is None else float(bn.momentum)
    o.eps = float(bn.eps)
    return o


def dropout_p(drop) -> float:
    """The p an nn.Dropout applies in its current state (0 in eval mode); ValueError for another module type."""
    if not isinstance(drop, torch.nn.Dropout):
        raise ValueError(f"pose2mesh_release_b200: expected an nn.Dropout, got {type(drop).__name__}")
    return float(drop.p) if drop.training else 0.0


def cuda_tensor(x, what: str) -> torch.Tensor:
    """x, if it is a CUDA tensor: there is no CPU path."""
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError(f"pose2mesh_release_b200 runs on CUDA (sm_90a) only; {what} is not a CUDA tensor")
    return x
