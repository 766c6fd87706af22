"""PoseNet, the 2-D -> 3-D pose lifter in front of MeshNet: drop-in for the reference's ``models.posenet``
(lib/models/posenet.py:13-87) — SURVEY.md §8 row f1.

``LinearModel`` keeps the reference's constructor, attribute names and ``state_dict`` keys (``w1``, ``batch_norm1``
(constructed but unused by the reference's forward), ``linear_stages.<i>.{w1,batch_norm1,w2,batch_norm2}``, ``w2``)
so PoseNet checkpoints load unchanged.  In eval mode (what FlatPose2Mesh uses for inference, demo/run.py:168) the
forward runs in libp2m_b200.so (``p2m_posenet_forward``: fp32 GEMMs with the BatchNorm / ReLU / residual fused into
their epilogues).  In training mode (dropout + batch statistics: lib/core/base.py:116, and the PoseNet pre-training of
:246-265) forward and backward run there too (``p2m_posenet_train_forward_opts`` / ``p2m_posenet_backward_opts``) for
contiguous float32 CUDA tensors; the dropout mask follows the rule stated in include/p2m_b200.h, not torch's generator
stream.  Every BatchNorm and each stage's Dropout act by their own state (frozen statistics, momentum, eps, p).
Anything else (CPU tensors, other dtypes, gradients through an eval-mode forward) runs the reference's torch ops.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib


def weight_init(module):
    """lib/models/posenet.py:6-8 (kaiming-normal Linear weights; not applied by the reference's constructor either)."""
    if isinstance(module, nn.Linear):
        nn.init.kaiming_normal_(module.weight)


def _register(owner: nn.Module, spec):
    """Create the sub-modules of `spec` (name -> factory) in order: registration order fixes both the state_dict key
    order and the order in which the default initialisers draw from the global RNG (identical to the reference's)."""
    for name, factory in spec:
        setattr(owner, name, factory())


class Linear(nn.Module):
    """One residual stage (lib/models/posenet.py:13-39): x + w2(drop(relu(bn2(w1(drop(relu(bn1(x)))))))."""

    def __init__(self, linear_size, p_dropout=0.5):
        super().__init__()
        h = self.l_size = linear_size
        _register(self, (("relu", lambda: nn.ReLU(inplace=True)), ("dropout", lambda: nn.Dropout(p_dropout)),
                         ("w1", lambda: nn.Linear(h, h)), ("batch_norm1", lambda: nn.BatchNorm1d(h)),
                         ("w2", lambda: nn.Linear(h, h)), ("batch_norm2", lambda: nn.BatchNorm1d(h))))

    def forward(self, x):
        y = x
        for bn, lin in ((self.batch_norm1, self.w1), (self.batch_norm2, self.w2)):
            y = lin(self.dropout(self.relu(bn(y))))
        return x + y


def _train_forward(module, x, seed, with_combine, modes):
    """p2m_posenet_train_forward_opts: (pose3d, pose_combine or None, saved).  modes = (BnOpts [2 S], float [S])."""
    lib = _lib.load()
    dev, B = x.device, x.shape[0]
    dims = (B, module.num_joint, module.linear_size, module.num_stage)
    out = torch.empty((B, module.output_size), device=dev, dtype=torch.float32)
    comb = torch.empty((B, module.num_joint, 5), device=dev, dtype=torch.float32) if with_combine else None
    n_saved, n_ws = lib.p2m_posenet_train_saved_bytes(*dims), lib.p2m_posenet_train_workspace_bytes(*dims)
    saved = torch.empty(n_saved, device=dev, dtype=torch.uint8)
    ws = torch.empty(n_ws, device=dev, dtype=torch.uint8)
    native = module._native_params()
    extra = module._native_train_extra()
    _lib.call("p2m_posenet_train_forward_opts", dev, C.byref(native), C.byref(extra), modes[0], modes[1], x, B, seed,
              out, comb, saved, n_saved, ws, n_ws)
    return out, comb, saved


class _PoseNetTrainFunction(torch.autograd.Function):
    """LinearModel's train-mode forward / backward through p2m_posenet_train_forward_opts / p2m_posenet_backward_opts.
    modes: LinearModel._native_modes() of the forward, which the backward takes too.  params: w1.weight, w1.bias,
    w2.weight, w2.bias, then per stage w1.weight, w1.bias, w2.weight, w2.bias, batch_norm1.weight, batch_norm1.bias,
    batch_norm2.weight, batch_norm2.bias."""

    @staticmethod
    def forward(ctx, module, x, seed, with_combine, modes, *params):
        dims = (x.shape[0], module.num_joint, module.linear_size, module.num_stage)
        out, comb, saved = _train_forward(module, x, seed, with_combine, modes)
        ctx.module, ctx.saved, ctx.dims, ctx.modes = module, saved, dims, modes
        ctx.save_for_backward(x, seed, *params)
        if comb is None:
            return out
        ctx.mark_non_differentiable(comb)                 # the reference detaches pose3d before the concat
        return out, comb

    @staticmethod
    def backward(ctx, d_out, *_):
        if ctx.saved is None:
            raise RuntimeError("pose2mesh_release_b200: the saved activations of this forward were already released "
                               "by an earlier backward (retain_graph is not supported: run the forward again)")
        lib = _lib.load()
        x, seed, *params = ctx.saved_tensors
        module, dev = ctx.module, x.device
        grads = [torch.empty_like(p) for p in params]
        g = _lib.PoseNetGrads()
        g.w1_w, g.w1_b, g.w2_w, g.w2_b = (t.data_ptr() for t in grads[:4])
        stages = (_lib.PoseNetStageGrads * module.num_stage)()
        for i in range(module.num_stage):
            for (name, _), t in zip(_lib.PoseNetStageGrads._fields_, grads[4 + 8 * i:12 + 8 * i]):
                setattr(stages[i], name, t.data_ptr())
        g.stages = stages
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        n_ws = lib.p2m_posenet_train_workspace_bytes(*ctx.dims)
        ws = torch.empty(n_ws, device=dev, dtype=torch.uint8)
        native = module._native_params()
        _lib.call("p2m_posenet_backward_opts", dev, C.byref(native), ctx.modes[0], ctx.modes[1], x, ctx.dims[0], seed,
                  ctx.saved, ctx.saved.numel(), d_out.contiguous().float(), C.byref(g), dx, ws, n_ws)
        ctx.saved = None
        return (None, dx, None, None, None, *grads)


class LinearModel(nn.Module):
    """lib/models/posenet.py:41-87: Linear(2J, H) -> `num_stage` residual stages -> Linear(H, 3J)."""

    def __init__(self, num_joint, linear_size=4096, num_stage=2, p_dropout=0.5, pretrained=False):
        super().__init__()
        self.num_joint, self.linear_size, self.num_stage, self.p_dropout = num_joint, linear_size, num_stage, p_dropout
        self.input_size, self.output_size = 2 * num_joint, 3 * num_joint          # 2-D joints in, 3-D joints out
        h = linear_size
        _register(self, (("w1", lambda: nn.Linear(self.input_size, h)),
                         ("batch_norm1", lambda: nn.BatchNorm1d(h)),               # constructed, never applied (reference :63 vs :74-87)
                         ("linear_stages", lambda: nn.ModuleList(Linear(h, p_dropout) for _ in range(num_stage))),
                         ("w2", lambda: nn.Linear(h, self.output_size)),
                         ("relu", lambda: nn.ReLU(inplace=True)), ("dropout", lambda: nn.Dropout(p_dropout))))
        if pretrained:
            raise RuntimeError("pretrained PoseNet weights are loaded by the reference's own checkpoint code "
                               "(funcs_utils.load_checkpoint); load_state_dict() them into this module")

    def _native_params(self):
        stages = (_lib.PoseNetStage * self.num_stage)()
        keep = []
        for i, st in enumerate(self.linear_stages):
            vals = [st.w1.weight, st.w1.bias, st.w2.weight, st.w2.bias,
                    st.batch_norm1.weight, st.batch_norm1.bias, st.batch_norm1.running_mean, st.batch_norm1.running_var,
                    st.batch_norm2.weight, st.batch_norm2.bias, st.batch_norm2.running_mean, st.batch_norm2.running_var]
            for (name, _), t in zip(_lib.PoseNetStage._fields_, vals):
                if t is None:  # the running statistics of a BatchNorm without them (track_running_stats=False)
                    continue
                if t.dtype != torch.float32 or not t.is_contiguous():
                    raise RuntimeError("PoseNet parameters must be contiguous float32")
                setattr(stages[i], name, t.data_ptr())
            keep.append(vals)
        p = _lib.PoseNetParams()
        p.num_joint, p.hidden, p.num_stage = self.num_joint, self.linear_size, self.num_stage
        p.w1_w, p.w1_b = self.w1.weight.data_ptr(), self.w1.bias.data_ptr()
        p.w2_w, p.w2_b = self.w2.weight.data_ptr(), self.w2.bias.data_ptr()
        p.stages = stages
        p._keep = (stages, keep)
        return p

    def _native_modes(self):
        """(BnOpts [2 num_stage], float [num_stage]): each stage's bn1 / bn2 options and its Dropout's p (0 in eval
        mode) from the submodules' current state.  ValueError for a submodule the native kernels do not implement."""
        bn = (_lib.BnOpts * (2 * self.num_stage))()
        p = (C.c_float * self.num_stage)()
        for i, st in enumerate(self.linear_stages):
            bn[2 * i], bn[2 * i + 1] = _lib.bn_opts(st.batch_norm1), _lib.bn_opts(st.batch_norm2)
            p[i] = _lib.dropout_p(st.dropout)
        return bn, p

    @staticmethod
    def _batch_stats(modes) -> bool:
        return any(o.stats != _lib.P2M_BN_RUNNING for o in modes[0])

    def forward_native(self, x: torch.Tensor, with_combine: bool = False):
        """Eval forward in libp2m_b200.so.  x [B, 2J] (or [B, J, 2]) on the module's CUDA device -> pose3d [B, 3J];
        with_combine additionally returns pose_combine = cat(pose2d, pose3d / 1000) [B, J, 5]
        (lib/models/pose2mesh_net.py:18-19).  Each BatchNorm and Dropout acts by its own state: when one uses batch
        statistics or drops (e.g. a BatchNorm without running buffers), the training forward's kernels run instead,
        without a backward."""
        modes = self._native_modes()
        lib = _lib.load()
        _lib.cuda_tensor(x, "x")
        x = x.reshape(len(x), -1).contiguous().float()
        if x.shape[1] != self.input_size:
            raise ValueError(f"PoseNet expects {self.input_size} inputs per pose, got {x.shape[1]}")
        dev, B = x.device, x.shape[0]
        if self.w1.weight.device != dev:
            raise RuntimeError("parameters and input live on different devices")
        if self._batch_stats(modes) or any(p > 0 for p in modes[1]):
            seed = torch.empty(2, dtype=torch.int64, device=dev).random_()
            out, comb, _ = _train_forward(self, x, seed, with_combine, modes)
            return (out, comb) if with_combine else out
        out = torch.empty((B, self.output_size), device=dev, dtype=torch.float32)
        comb = torch.empty((B, self.num_joint, 5), device=dev, dtype=torch.float32) if with_combine else None
        nbytes = lib.p2m_posenet_workspace_bytes(B, self.linear_size)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        params = self._native_params()
        _lib.call("p2m_posenet_forward_opts", dev, C.byref(params), modes[0], x, out, comb, B, ws, nbytes)
        return (out, comb) if with_combine else out

    def _native_train_extra(self):
        stages = (_lib.PoseNetTrainStage * self.num_stage)()
        keep = []
        for i, st in enumerate(self.linear_stages):
            nbt = (st.batch_norm1.num_batches_tracked, st.batch_norm2.num_batches_tracked)
            stages[i].bn1_nbt, stages[i].bn2_nbt = (None if t is None else t.data_ptr() for t in nbt)
            keep.append(nbt)
        e = _lib.PoseNetTrain()
        e.stages = stages
        e._keep = (stages, keep)
        return e

    def _trained_tensors(self):
        """The 4 + 8 num_stage tensors the backward produces gradients for, in _PoseNetTrainFunction's order."""
        out = [self.w1.weight, self.w1.bias, self.w2.weight, self.w2.bias]
        for st in self.linear_stages:
            out += [st.w1.weight, st.w1.bias, st.w2.weight, st.w2.bias, st.batch_norm1.weight, st.batch_norm1.bias,
                    st.batch_norm2.weight, st.batch_norm2.bias]
        return out

    def native_train_ok(self, x: torch.Tensor) -> bool:
        """Whether the train-mode forward of x runs in libp2m_b200.so: x, the trained tensors and the BatchNorm running
        statistics (where a BatchNorm has them) are contiguous float32 CUDA tensors on one device."""
        if not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()):
            return False
        tensors = self._trained_tensors()
        for st in self.linear_stages:
            for bn in (st.batch_norm1, st.batch_norm2):
                tensors += [t for t in (bn.running_mean, bn.running_var) if t is not None]
        return all(t.device == x.device and t.dtype == torch.float32 and t.is_contiguous() for t in tensors)

    def forward_train_native(self, x: torch.Tensor, seed: torch.Tensor = None, with_combine: bool = False):
        """Train-mode forward in libp2m_b200.so, differentiable (the backward runs there too).  x [B, 2J] (or
        [B, J, 2]) -> pose3d [B, 3J]; with_combine additionally returns the detached pose_combine [B, J, 5].  seed:
        two int64 on x's device that define the dropout masks (include/p2m_b200.h); drawn from torch's generator when
        not given, so torch.manual_seed reproduces a run.  Each BatchNorm and each stage's Dropout acts by its own state
        (train / eval, track_running_stats, momentum, eps, p): an eval-mode BatchNorm keeps its running statistics
        (frozen), a train-mode one with track_running_stats updates them."""
        modes = self._native_modes()
        x = x.reshape(len(x), -1)
        if not self.native_train_ok(x):
            raise RuntimeError("the native train-mode PoseNet needs contiguous float32 CUDA tensors on one device")
        if x.shape[1] != self.input_size:
            raise ValueError(f"PoseNet expects {self.input_size} inputs per pose, got {x.shape[1]}")
        if x.shape[0] < 2 and self._batch_stats(modes):
            raise ValueError(f"Expected more than 1 value per channel when training, got input size {tuple(x.shape)}")
        if seed is None:
            seed = torch.empty(2, dtype=torch.int64, device=x.device).random_()
        return _PoseNetTrainFunction.apply(self, x, seed, with_combine, modes, *self._trained_tensors())

    def _forward_torch(self, x):
        """The reference's own op sequence (lib/models/posenet.py:77-87)."""
        y = self.w1(x)
        for stage in self.linear_stages:
            y = stage(y)
        return self.w2(y)

    def forward(self, x):
        if self.training:
            return self.forward_train_native(x) if self.native_train_ok(x) else self._forward_torch(x)
        if x.is_cuda and not (torch.is_grad_enabled() and x.requires_grad):
            return self.forward_native(x)
        return self._forward_torch(x)


CAPTURE_FIELDS = ("g_y", "a2", "g_a2", "g_z2", "a1", "g_a1", "g_bn1", "scale", "g_y0")


def debug_train_step_capture(module, x, seed, d_out, capture=CAPTURE_FIELDS):
    """One native train step of `module` with the backward's intermediates captured
    (p2m_debug_posenet_backward_capture): p2m_posenet_train_forward_opts, then the capture backward with the same
    LinearModel._native_modes().  Running statistics are updated as by the module's own forward.  capture: the
    p2m_posenet_capture_t fields to fill (the others stay null); None runs p2m_posenet_backward_opts instead, without
    a capture.  Returns a dict with out [B, 3J], combine [B, J, 5], saved (uint8), grads (in the order of
    LinearModel._trained_tensors()), dx [B, 2J], and per captured field a list of num_stage [B, H] tensors
    (scale: [S, 4], g_y0: one [B, H] tensor)."""
    lib = _lib.load()
    x = x.reshape(len(x), -1).contiguous().float()
    dev, B, S, H = x.device, x.shape[0], module.num_stage, module.linear_size
    modes = module._native_modes()
    out, comb, saved = _train_forward(module, x, seed, True, modes)
    params = module._trained_tensors()
    grads = [torch.empty_like(p) for p in params]
    g = _lib.PoseNetGrads()
    g.w1_w, g.w1_b, g.w2_w, g.w2_b = (t.data_ptr() for t in grads[:4])
    stages = (_lib.PoseNetStageGrads * S)()
    for i in range(S):
        for (name, _), t in zip(_lib.PoseNetStageGrads._fields_, grads[4 + 8 * i:12 + 8 * i]):
            setattr(stages[i], name, t.data_ptr())
    g.stages = stages
    dx = torch.empty_like(x)
    res = dict(out=out, combine=comb, saved=saved, grads=grads, dx=dx)
    n_ws = lib.p2m_posenet_train_workspace_bytes(B, module.num_joint, H, S)
    ws = torch.empty(n_ws, device=dev, dtype=torch.uint8)
    native = module._native_params()
    args = (C.byref(native), modes[0], modes[1], x, B, seed, saved, saved.numel(), d_out.contiguous().float(),
            C.byref(g), dx, ws, n_ws)
    if capture is None:
        _lib.call("p2m_posenet_backward_opts", dev, *args)
        return res
    cap = _lib.PoseNetCapture()
    keep = []
    for name in CAPTURE_FIELDS[:-1]:
        if name not in capture:
            continue
        shape = (4,) if name == "scale" else (B, H)
        fill = float("nan") if name == "scale" else 0.0      # an unwritten scale stays NaN
        ts = [torch.full(shape, fill, device=dev, dtype=torch.float32) for _ in range(S)]
        arr = (C.c_void_p * max(S, 1))(*[t.data_ptr() for t in ts])
        keep.append(arr)
        setattr(cap, name, C.cast(arr, C.POINTER(C.c_void_p)))
        res[name] = ts
    if "g_y0" in capture:
        res["g_y0"] = torch.zeros((B, H), device=dev, dtype=torch.float32)
        cap.g_y0 = res["g_y0"].data_ptr()
    _lib.call("p2m_debug_posenet_backward_capture", dev, *args, C.byref(cap))
    if "scale" in res:
        res["scale"] = torch.stack(res["scale"]) if S else torch.empty((0, 4), device=dev)
    return res


def get_model(num_joint, hid_dim, num_layer, p_dropout, pretrained=False):
    """lib/models/posenet.py:89-92."""
    return LinearModel(num_joint, hid_dim, num_layer, p_dropout, pretrained)
