"""MeshNet on H100: drop-in for the reference's ``models.meshnet`` (lib/models/meshnet.py).

``Pose2Mesh`` keeps the reference's constructor, ``forward(x)`` and ``state_dict`` surface
(SURVEY.md §8b) — ``fc.*``, ``cl.<i>.*``, ``bn.<i>.*`` with a ``None`` hole for the last BatchNorm —
so checkpoints load unchanged and ``main/train.py`` / ``demo/run.py`` can use it as is.  All
device work of ``forward`` and ``backward`` runs in libp2m_b200.so (hand-written sm_90a CUDA,
C ABI in include/p2m_b200.h); PyTorch only owns the memory, the stream and autograd bookkeeping.
There is no CPU / eager fallback: inputs must live on a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _lib

CHEB_K = 3  # lib/models/meshnet.py:23,29: every layer uses Chebyshev order 3


def channel_plan(num_joint_input_chan: int, num_mesh_output_chan: int, mano: bool):
    """Per-block channel chains (lib/models/meshnet.py:21-33)."""
    if mano:
        return [(num_joint_input_chan, 32, 64, 64), (64, 128, 256), (256, 256, 256), (256, 256, 256),
                (256, 256, 256), (256, 128, 128), (128, 64, num_mesh_output_chan)]
    return [(num_joint_input_chan, 32, 64, 64), (64, 128, 256), (256, 256, 256), (256, 256, 256),
            (256, 256, 256), (256, 256, 256), (256, 128, 128), (128, 128, 128), (128, 128, 128),
            (128, 64, num_mesh_output_chan)]


def _is_mano(graph_L) -> bool:
    """lib/models/meshnet.py:21 reads cfg.DATASET.target_joint_set; honour it when the reference's
    config module is importable, otherwise infer the plan from the hierarchy depth (levels=6 -> 7
    Laplacians for MANO, levels=9 -> 10 for SMPL; demo/run.py:79-114)."""
    try:
        from core.config import cfg  # type: ignore

        return cfg.DATASET.target_joint_set == "mano"
    except Exception:
        return len(graph_L) == 7


class BakedHierarchy:
    """Host copy of the Laplacian list in the layout the C ABI wants (CSR, int32 indices, float32
    values = graph_utils.sparse_python_to_torch's f64->f32 cast, lib/graph_utils.py:98-109), plus
    lazily created per-device native handles."""

    def __init__(self, laplacians: Sequence, plan):
        self.level_size = np.array([m.shape[0] for m in laplacians], dtype=np.int32)
        self.rowptr, self.colidx, self.values = [], [], []
        for i, m in enumerate(laplacians):
            c = m.tocsr().astype(np.float32)  # noqa: keeps explicit entries
            c.sort_indices()
            if (c != c.T).nnz:  # the backward passes apply L~ where the gradient needs L~^T
                raise ValueError(f"Laplacian {i} is not symmetric: MeshNet's kernels need L~ == L~^T")
            self.rowptr.append(np.ascontiguousarray(c.indptr, dtype=np.int32))
            self.colidx.append(np.ascontiguousarray(c.indices, dtype=np.int32))
            self.values.append(np.ascontiguousarray(c.data, dtype=np.float32))
        self.block_len = np.array([len(p) for p in plan], dtype=np.int32)
        self.block_chans = np.array([c for p in plan for c in p], dtype=np.int32)
        self._handles = {}
        self._lock = threading.Lock()
        self.precision = _lib.default_precision()

    def handle(self, device_index: int) -> int:
        with self._lock:
            h = self._handles.get(device_index)
            if h is None:
                lib = _lib.load()
                n = len(self.level_size)
                desc = _lib.ModelDesc()
                desc.n_levels = n
                desc.level_size = self.level_size.ctypes.data_as(_lib.c_int32_p)
                rp = (_lib.c_int32_p * n)(*[a.ctypes.data_as(_lib.c_int32_p) for a in self.rowptr])
                ci = (_lib.c_int32_p * n)(*[a.ctypes.data_as(_lib.c_int32_p) for a in self.colidx])
                va = (_lib.c_float_p * n)(*[a.ctypes.data_as(_lib.c_float_p) for a in self.values])
                desc.rowptr, desc.colidx, desc.values = rp, ci, va
                desc.n_blocks = len(self.block_len)
                desc.block_len = self.block_len.ctypes.data_as(_lib.c_int32_p)
                desc.block_chans = self.block_chans.ctypes.data_as(_lib.c_int32_p)
                desc.device = device_index
                out = C.c_void_p()
                _lib.check(lib.p2m_model_create(C.byref(desc), C.byref(out)), "p2m_model_create")
                _lib.check(lib.p2m_model_set_precision(out, self.precision), "p2m_model_set_precision")
                h = out.value
                self._handles[device_index] = h
            return h

    def set_precision(self, precision: int):
        with self._lock:
            self.precision = precision
            for h in self._handles.values():
                _lib.check(_lib.load().p2m_model_set_precision(h, precision), "p2m_model_set_precision")

    def set_profiling(self, device_index: int, enable: bool):
        _lib.check(_lib.load().p2m_model_set_profiling(self.handle(device_index), int(enable)), "set_profiling")

    def set_debug(self, device_index: int, fuse_head: Optional[bool] = None, elide_padding: Optional[int] = None,
                  dedup_padding: Optional[bool] = None, sm_count: Optional[int] = None):
        """Ablation switches of the tensor-core path: fused 64->3 head in eval (default on), isolated padding vertices
        through a plain GEMM with combined weights (0 off, 1 = default: levels with >= 40 % isolated rows, 2 = every
        level that has the tile families), the SM count the persistent tensor-core grids are sized for (0 = the
        device's own; a smaller count gives each CTA more tiles, as on a part with fewer SMs)."""
        lib, h = _lib.load(), self.handle(device_index)
        if sm_count is not None:
            _lib.check(lib.p2m_debug_set_sm_count(h, int(sm_count)), "set_sm_count")
        if fuse_head is not None:
            _lib.check(lib.p2m_debug_set_fuse_head(h, int(fuse_head)), "set_fuse_head")
        if elide_padding is not None:
            _lib.check(lib.p2m_debug_set_elide_padding(h, int(elide_padding)), "set_elide_padding")
        if dedup_padding is not None:  # eval: one representative per class of identical isolated rows (default on)
            _lib.check(lib.p2m_debug_set_dedup_padding(h, int(dedup_padding)), "set_dedup_padding")

    def set_capture(self, device_index: int, capture: Optional[dict] = None):
        """Debug: copy the network schedules' intermediate tensors into device tensors (p2m_debug_set_capture).
        ``capture`` maps the p2m_capture_t field names to a list with one tensor (or None) per layer for z, a, y, g_a,
        g_z and dx, or to one tensor for fc_out and fc_dx; missing names are not captured.  None clears the capture.
        The tensors must stay alive until the capture is cleared."""
        lib, h = _lib.load(), self.handle(device_index)
        if capture is None:
            _lib.check(lib.p2m_debug_set_capture(h, None), "set_capture")
            return
        c = _lib.Capture()
        keep = []
        for name in ("z", "a", "y", "g_a", "g_z", "dx"):
            if capture.get(name) is not None:
                arr = _ptr_array(capture[name])
                keep.append(arr)
                setattr(c, name, arr)
        for name in ("fc_out", "fc_dx"):
            if capture.get(name) is not None:
                setattr(c, name, capture[name].data_ptr())
        _lib.check(lib.p2m_debug_set_capture(h, C.byref(c)), "set_capture")  # copies the arrays

    def layer_route(self, device_index: int, layer: int, batch: int, need_dx: bool = True) -> dict:
        """Debug: the paths the network schedules take for one layer (p2m_debug_layer_route)."""
        out = (C.c_int32 * 9)()
        _lib.check(_lib.load().p2m_debug_layer_route(self.handle(device_index), layer, batch, int(need_dx), out),
                   "layer_route")
        return dict(zip(("tc", "elide", "thin", "tc_dw", "dw_dz_basis", "tc_dx", "dx_elide", "tc_dt", "fuse_head"),
                        (bool(v) for v in out)))

    def layer_info(self, device_index: int):
        lib = _lib.load()
        h = self.handle(device_index)
        out = []
        for i in range(lib.p2m_model_num_layers(h)):
            buf = (C.c_int32 * 6)()
            _lib.check(lib.p2m_model_layer_info(h, i, buf), "layer_info")
            out.append(dict(level=buf[0], V=buf[1], fin=buf[2], fout=buf[3], bn=buf[4], relu=buf[5]))
        return out

    def layer_times_ms(self, device_index: int):
        lib = _lib.load()
        h = self.handle(device_index)
        n = lib.p2m_model_num_layers(h)
        buf = (C.c_float * n)()
        _lib.check(lib.p2m_model_layer_times_ms(h, buf, n), "layer_times_ms")
        return list(buf)

    def kernel_status(self, device_index: int) -> int:
        """0 unless a tensor-core kernel's bounded mbarrier wait timed out (debug aid; synchronises)."""
        out = C.c_int32(0)
        _lib.check(_lib.load().p2m_debug_kernel_status(self.handle(device_index), C.byref(out)), "kernel_status")
        return out.value

    def __deepcopy__(self, memo):  # handles are per-process device state: share, never copy
        return self

    def __del__(self):
        try:
            lib = _lib.load()
            for h in self._handles.values():
                lib.p2m_model_destroy(h)
        except Exception:
            pass


def _ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = None if t is None else t.data_ptr()
    return arr


def _param_table(fc_w, fc_b, cl_w, cl_b, bn_w, bn_b, bn_rm=None, bn_rv=None, bn_nbt=None):
    n = len(cl_w)
    none = [None] * n
    keep = [_ptr_array(cl_w), _ptr_array(cl_b), _ptr_array(bn_w), _ptr_array(bn_b),
            _ptr_array(bn_rm or none), _ptr_array(bn_rv or none), _ptr_array(bn_nbt or none)]
    p = _lib.Params()
    p.fc_w, p.fc_b = fc_w.data_ptr(), fc_b.data_ptr()
    p.cl_w, p.cl_b, p.bn_w, p.bn_b, p.bn_rm, p.bn_rv, p.bn_nbt = keep
    p._keep = keep  # keep the ctypes arrays alive
    return p


class _MeshNetFunction(torch.autograd.Function):
    """Pose2Mesh.forward / backward through p2m_meshnet_forward_opts / p2m_meshnet_backward_opts.  ``buffers`` is
    (running means, running vars, num_batches_tracked[, per-layer _lib.BnOpts array]); without the options array every
    BatchNorm takes the defaults of ``training`` (batch statistics with update, or running statistics)."""

    @staticmethod
    def forward(ctx, x, hier: BakedHierarchy, training: bool, buffers, n_layers, *params):
        lib = _lib.load()
        dev = x.device
        h = hier.handle(dev.index)
        fc_w, fc_b = params[0], params[1]
        cl_w = list(params[2:2 + n_layers])
        cl_b = list(params[2 + n_layers:2 + 2 * n_layers])
        n_bn = n_layers - 1
        bn_w = list(params[2 + 2 * n_layers:2 + 2 * n_layers + n_bn]) + [None]
        bn_b = list(params[2 + 2 * n_layers + n_bn:2 + 2 * n_layers + 2 * n_bn]) + [None]
        bn_rm, bn_rv, bn_nbt, *rest = buffers
        opts = rest[0] if rest else None
        B = x.shape[0]
        v0 = int(hier.level_size[0])
        cout = int(hier.block_chans[-1])
        y = torch.empty((B, v0, cout), device=dev, dtype=torch.float32)
        ws_bytes = lib.p2m_meshnet_workspace_bytes_opts(h, B, int(training), opts)
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        table = _param_table(fc_w, fc_b, cl_w, cl_b, bn_w, bn_b, bn_rm, bn_rv, bn_nbt)
        _lib.call("p2m_meshnet_forward_opts", dev, h, C.byref(table), opts, x, y, B, int(training), ws, ws_bytes)
        needs_grad = training and any(ctx.needs_input_grad)
        if needs_grad:  # the backward takes the options of this forward
            ctx.hier, ctx.n_layers, ctx.ws, ctx.ws_bytes, ctx.bn_opts = hier, n_layers, ws, ws_bytes, opts
            ctx.save_for_backward(x, *params)
        ctx.differentiable = needs_grad
        ctx.training = training
        return y

    @staticmethod
    def backward(ctx, dy):
        if not ctx.differentiable:
            raise RuntimeError("pose2mesh_release_b200: backward through an eval-mode MeshNet forward is not "
                               "supported (BatchNorm was folded into the conv epilogues and no activations were "
                               "kept); call .train() first")
        if ctx.ws is None:
            raise RuntimeError("pose2mesh_release_b200: the saved activations of this forward were already released "
                               "by an earlier backward (retain_graph is not supported: run the forward again)")
        lib = _lib.load()
        x, *params = ctx.saved_tensors
        n_layers, hier = ctx.n_layers, ctx.hier
        dev = x.device
        h = hier.handle(dev.index)
        n_bn = n_layers - 1
        fc_w, fc_b = params[0], params[1]
        cl_w = list(params[2:2 + n_layers])
        cl_b = list(params[2 + n_layers:2 + 2 * n_layers])
        bn_w = list(params[2 + 2 * n_layers:2 + 2 * n_layers + n_bn]) + [None]
        bn_b = list(params[2 + 2 * n_layers + n_bn:2 + 2 * n_layers + 2 * n_bn]) + [None]
        # one flat gradient buffer; per-parameter gradients are views into it
        sizes = [p.numel() for p in params]
        flat = torch.empty(sum(sizes), device=dev, dtype=torch.float32)
        grads, off = [], 0
        for p_, n in zip(params, sizes):
            grads.append(flat[off:off + n].view_as(p_))
            off += n
        g_fc_w, g_fc_b = grads[0], grads[1]
        g_cl_w = grads[2:2 + n_layers]
        g_cl_b = grads[2 + n_layers:2 + 2 * n_layers]
        g_bn_w = grads[2 + 2 * n_layers:2 + 2 * n_layers + n_bn] + [None]
        g_bn_b = grads[2 + 2 * n_layers + n_bn:2 + 2 * n_layers + 2 * n_bn] + [None]
        ptab = _param_table(fc_w, fc_b, cl_w, cl_b, bn_w, bn_b)
        gtab = _param_table(g_fc_w, g_fc_b, g_cl_w, g_cl_b, g_bn_w, g_bn_b)
        B = x.shape[0]
        dy = dy.contiguous().float()
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        sc_bytes = lib.p2m_meshnet_backward_scratch_bytes(h, B)
        scratch = torch.empty(sc_bytes, device=dev, dtype=torch.uint8)
        _lib.call("p2m_meshnet_backward_opts", dev, h, C.byref(ptab), C.byref(gtab), ctx.bn_opts, x, dy, dx, B, ctx.ws,
                  ctx.ws_bytes, scratch, sc_bytes)
        ctx.ws = None
        return (dx, None, None, None, None, *grads)


class Pose2Mesh(nn.Module):
    """Coarse-to-fine Chebyshev graph-conv stack (reference: lib/models/meshnet.py:11-117).

    Args mirror the reference: ``graph_L`` is the list returned by ``build_coarse_graphs`` (scipy CSR
    float64, fine -> coarse, joint graph last, ``levels + 1`` entries).  Unlike the reference the
    caller's list is copied, not mutated (no caller reads it afterwards; SURVEY.md §8b).
    """

    def __init__(self, num_joint_input_chan, num_mesh_output_chan, graph_L, joint_set: Optional[str] = None):
        super().__init__()
        self.num_joint_input_chan = num_joint_input_chan
        self.num_mesh_output_chan = num_mesh_output_chan
        mano = _is_mano(graph_L) if joint_set is None else (joint_set == "mano")
        self.CL_F = channel_plan(num_joint_input_chan, num_mesh_output_chan, mano)
        self.CL_K = [CHEB_K] * len(self.CL_F)
        laps = list(graph_L)
        del laps[-2]  # the reference drops the second-coarsest (48x48) Laplacian (meshnet.py:35)
        if len(laps) != len(self.CL_F) - 1:
            raise ValueError(f"graph_L has {len(graph_L)} levels but the channel plan needs {len(self.CL_F)}")
        self.graph_L = laps
        n_joint, v1 = laps[-1].shape[0], laps[-2].shape[0]
        # construction order == the reference's, so torch.manual_seed(s) gives identical weights
        self.fc = nn.Linear(n_joint * self.CL_F[0][-1], v1 * self.CL_F[1][0])
        _cl, _bn = [], []
        n_blocks = len(self.CL_F)
        for i, chans in enumerate(self.CL_F):
            for j in range(len(chans) - 1):
                fin, fout = self.CL_K[i] * chans[j], chans[j + 1]
                lin = nn.Linear(fin, fout)
                bound = float(np.sqrt(2.0 / (fin + fout)))
                lin.weight.data.uniform_(-bound, bound)
                lin.bias.data.fill_(0.0)
                _cl.append(lin)
                last = (i == n_blocks - 1) and (j == len(chans) - 2)
                _bn.append(None if last else nn.BatchNorm1d(fout))
        self.cl = nn.ModuleList(_cl)
        self.bn = nn.ModuleList(_bn)
        self._hier = BakedHierarchy(laps, self.CL_F)

    # -- knobs ---------------------------------------------------------------------------------
    def set_precision(self, precision: str):
        """'fp32' (CUDA-core FFMA), 'fp16x3' (wgmma tensor cores, error-compensated split), 'fp16' (single-pass
        wgmma with fp16 operands, inference only: a train-mode forward or a backward raises RuntimeError) or
        'fp16_mixed' (the same single-pass convs in the training forward, backward-data and weight gradient: fp16
        operands, fp32 accumulation, fp32 weights and BatchNorm; its eval forward is bitwise that of 'fp16')."""
        self._hier.set_precision(_lib.PRECISIONS[precision])
        return self

    @property
    def num_vertices(self) -> int:
        return int(self._hier.level_size[0])

    def _flat_params(self):
        n = len(self.cl)
        cl_w = [m.weight for m in self.cl]
        cl_b = [m.bias for m in self.cl]
        bn_w = [m.weight for m in self.bn if m is not None]
        bn_b = [m.bias for m in self.bn if m is not None]
        return n, [self.fc.weight, self.fc.bias, *cl_w, *cl_b, *bn_w, *bn_b]

    def _bn_buffers(self):
        rm = [None if m is None else m.running_mean for m in self.bn]
        rv = [None if m is None else m.running_var for m in self.bn]
        nbt = [None if m is None else m.num_batches_tracked for m in self.bn]
        return rm, rv, nbt

    def _bn_opts(self):
        """One p2m_bn_opts_t per layer from each BatchNorm's own state (training flag, track_running_stats, momentum,
        eps), read on every forward; the last layer's entry (no BatchNorm) is ignored by the library.  ValueError for
        a BatchNorm the native kernels do not implement."""
        opts = (_lib.BnOpts * len(self.cl))()
        for i, m in enumerate(self.bn):
            if i == len(self.cl) - 1:
                opts[i].stats = _lib.P2M_BN_RUNNING
            else:
                opts[i] = _lib.bn_opts(m)
        return opts

    def _check_eval_bn(self, what: str, modes: bool):
        """The inference entry points run the eval schedule with the defaults: running statistics and eps 1e-5 in
        every BatchNorm (modes: each BatchNorm must also be in eval mode)."""
        for m in self.bn[:len(self.cl) - 1]:
            o = _lib.bn_opts(m)
            if m.running_mean is None or m.running_var is None or o.eps != 1e-5 or (
                    modes and o.stats != _lib.P2M_BN_RUNNING):
                raise ValueError(f"{what} needs every BatchNorm in eval mode with running statistics and eps 1e-5; "
                                 "use forward() for other BatchNorm settings")

    def forward(self, x):
        opts = self._bn_opts()
        n_joint = self.graph_L[-1].shape[0]
        x = x.view(-1, n_joint, self.num_joint_input_chan)
        if not x.is_cuda:
            raise RuntimeError("pose2mesh_release_b200.Pose2Mesh runs on CUDA (sm_90a) only; got a CPU tensor "
                               "(the reference hard-codes .cuda() too: lib/models/meshnet.py:81)")
        x = x.contiguous().float()
        n, params = self._flat_params()
        for p in params:
            if p.device != x.device:
                raise RuntimeError("parameters and input live on different devices")
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise RuntimeError("pose2mesh_release_b200.Pose2Mesh needs contiguous float32 parameters "
                                   f"(got {p.dtype}); the library reads them through raw device pointers")
        return _MeshNetFunction.apply(x, self._hier, self.training, (*self._bn_buffers(), opts), n, *params)

    @torch.no_grad()
    def forward_vertices(self, x: torch.Tensor, perm_reverse, n_vertex: int) -> torch.Tensor:
        """Eval forward with the callers' gather fused into the head layer's store:
        equals ``self(x)[:, perm_reverse[:n_vertex], :]`` (lib/core/base.py:130,201; demo/run.py:170)
        without materialising the padded ``[B, V0, 3]`` tensor.  Returns ``[B, n_vertex, 3]``."""
        lib = _lib.load()
        if self.training:
            raise RuntimeError("forward_vertices is an inference entry point: call .eval() first")
        self._check_eval_bn("forward_vertices", True)
        n_joint = self.graph_L[-1].shape[0]
        x = x.view(-1, n_joint, self.num_joint_input_chan)
        if not x.is_cuda:
            raise RuntimeError("pose2mesh_release_b200 runs on CUDA (sm_90a) only; got a CPU tensor")
        x = x.contiguous().float()
        dev = x.device
        h = self._hier.handle(dev.index)
        self._set_gather(dev, perm_reverse, int(n_vertex))
        B = x.shape[0]
        y = torch.empty((B, int(n_vertex), self.num_mesh_output_chan), device=dev, dtype=torch.float32)
        ws_bytes = lib.p2m_meshnet_workspace_bytes(h, B, 0)
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        n, params = self._flat_params()
        n_bn = n - 1
        rm, rv, nbt = self._bn_buffers()
        table = _param_table(params[0], params[1], params[2:2 + n], params[2 + n:2 + 2 * n],
                             list(params[2 + 2 * n:2 + 2 * n + n_bn]) + [None],
                             list(params[2 + 2 * n + n_bn:]) + [None], rm, rv, nbt)
        _lib.call("p2m_meshnet_forward_vertices", dev, h, C.byref(table), x, y, B, ws, ws_bytes)
        return y

    def _set_gather(self, dev, perm_reverse, n_vertex):
        idx = np.ascontiguousarray(np.asarray(perm_reverse)[:n_vertex], dtype=np.int32)
        cache = self.__dict__.setdefault("_gather_maps", {})   # device -> index list currently set on that handle
        have = cache.get(dev.index)
        if have is None or have.shape != idx.shape or not np.array_equal(have, idx):
            _lib.check(_lib.load().p2m_model_set_output_gather(self._hier.handle(dev.index),
                                                               idx.ctypes.data_as(_lib.c_int32_p), int(n_vertex)),
                       "p2m_model_set_output_gather")
            cache[dev.index] = idx

    def forward_host(self, x_host: torch.Tensor, out: Optional[torch.Tensor] = None, device=None,
                     perm_reverse=None, n_vertex: Optional[int] = None) -> torch.Tensor:
        """Inference with HOST tensors through p2m_meshnet_forward_host: H2D of the poses, the eval forward, D2H of
        the meshes, synchronised.  With ``perm_reverse`` / ``n_vertex`` the callers' gather
        ``pred[:, perm_reverse[:n_vertex]]`` (lib/core/base.py:130,201) is fused into the head layer and only the
        ``[B, n_vertex, 3]`` vertices travel back (p2m_meshnet_forward_vertices_host).  bench.py's end-to-end figure."""
        lib = _lib.load()
        self._check_eval_bn("forward_host", False)
        dev = self.fc.weight.device if device is None else torch.device(device)
        h = self._hier.handle(dev.index)
        n_joint = self.graph_L[-1].shape[0]
        x_host = x_host.reshape(-1, n_joint, self.num_joint_input_chan).contiguous().float()
        B = x_host.shape[0]
        gathered = perm_reverse is not None
        rows = int(n_vertex) if gathered else self.num_vertices
        if gathered:
            self._set_gather(dev, perm_reverse, rows)
        if out is None:
            out = torch.empty((B, rows, self.num_mesh_output_chan), dtype=torch.float32, pin_memory=True)
        if tuple(out.shape) != (B, rows, self.num_mesh_output_chan) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"forward_host: `out` must be a contiguous float32 [{B}, {rows}, {self.num_mesh_output_chan}]")
        need = lib.p2m_meshnet_workspace_bytes(h, B, 0) + lib.p2m_meshnet_host_io_bytes(h, B)
        ws = getattr(self, "_host_ws", None)
        if ws is None or ws.numel() < need or ws.device != dev:
            ws = torch.empty(need, device=dev, dtype=torch.uint8)
            self._host_ws = ws
        n, params = self._flat_params()
        n_bn = n - 1
        rm, rv, nbt = self._bn_buffers()
        table = _param_table(params[0], params[1], params[2:2 + n], params[2 + n:2 + 2 * n],
                             list(params[2 + 2 * n:2 + 2 * n + n_bn]) + [None],
                             list(params[2 + 2 * n + n_bn:]) + [None], rm, rv, nbt)
        name = "p2m_meshnet_forward_vertices_host" if gathered else "p2m_meshnet_forward_host"
        _lib.call(name, dev, h, C.byref(table), x_host, out, B, ws, ws.numel())
        return out

    # the reference exposes these helpers; keep them for callers that poke at them
    def init_weights(self, W, Fin, Fout):
        scale = np.sqrt(2.0 / (Fin + Fout))
        W.uniform_(-scale, scale)
        return W

    def graph_upsample(self, x, p):
        """Nearest x p unpooling along the vertex axis (lib/models/meshnet.py:71-78)."""
        return x if p <= 1 else x.repeat_interleave(int(p), dim=1)


def get_model(num_joint_input_chan, num_mesh_output_chan, graph_L):
    """lib/models/meshnet.py:120-123."""
    return Pose2Mesh(num_joint_input_chan, num_mesh_output_chan, graph_L)
