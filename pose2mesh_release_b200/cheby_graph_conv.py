"""Functional Chebyshev graph convolution: drop-in for the reference's
``models.backbones.cheby_graph_conv.graph_conv_cheby(x, cl, bn, L, Fout, K)``
(lib/models/backbones/cheby_graph_conv.py:5-42).

The linear part ``[T0|T1|T2] W^T + b`` (basis SpMM + channel contraction, forward and backward)
runs in libp2m_b200.so through ``p2m_cheb_conv_fwd`` / ``p2m_cheb_conv_bwd``; the optional
``bn`` module is then applied exactly like the reference does (``bn(y.view(B*V, Fout))``).
The fused whole-network path used by ``Pose2Mesh.forward`` lives in meshnet.py.
"""
from __future__ import annotations

import ctypes as C
import weakref

import numpy as np
import scipy.sparse as sp
import torch

from . import _lib

_graph_cache = {}
_default_precision = _lib.default_precision()


def set_default_precision(precision: str):
    """'fp32' (CUDA cores), 'fp16x3' (wgmma tensor cores), 'fp16' (single-pass wgmma, inference only: a backward or a
    training-mode BatchNorm raises) or 'fp16_mixed' (single-pass wgmma in the forward and the backward, for mixed-
    precision training) for graph_conv_cheby calls."""
    global _default_precision
    _default_precision = _lib.PRECISIONS[precision]
    for _, gh in list(_graph_cache.values()):
        gh.apply_precision()


class GraphHandle:
    """A graph-only native handle (one Laplacian, no channel plan) per (matrix, device)."""

    def __init__(self, lap_csr: sp.csr_matrix):
        c = lap_csr.tocsr().astype(np.float32)
        c.sort_indices()
        self.V = c.shape[0]
        self.rowptr = np.ascontiguousarray(c.indptr, dtype=np.int32)
        self.colidx = np.ascontiguousarray(c.indices, dtype=np.int32)
        self.values = np.ascontiguousarray(c.data, dtype=np.float32)
        self._handles = {}

    def handle(self, device_index: int) -> int:
        h = self._handles.get(device_index)
        if h is None:
            lib = _lib.load()
            desc = _lib.ModelDesc()
            size = np.array([self.V], dtype=np.int32)
            desc.n_levels = 1
            desc.level_size = size.ctypes.data_as(_lib.c_int32_p)
            desc.rowptr = (_lib.c_int32_p * 1)(self.rowptr.ctypes.data_as(_lib.c_int32_p))
            desc.colidx = (_lib.c_int32_p * 1)(self.colidx.ctypes.data_as(_lib.c_int32_p))
            desc.values = (_lib.c_float_p * 1)(self.values.ctypes.data_as(_lib.c_float_p))
            desc.n_blocks = 0
            desc.device = device_index
            out = C.c_void_p()
            _lib.check(lib.p2m_model_create(C.byref(desc), C.byref(out)), "p2m_model_create")
            h = out.value
            _lib.check(lib.p2m_model_set_precision(h, _default_precision), "p2m_model_set_precision")
            self._handles[device_index] = h
        return h

    def apply_precision(self):
        for h in self._handles.values():
            _lib.check(_lib.load().p2m_model_set_precision(h, _default_precision), "p2m_model_set_precision")

    def kernel_status(self, device_index: int) -> int:
        out = C.c_int32(0)
        _lib.check(_lib.load().p2m_debug_kernel_status(self.handle(device_index), C.byref(out)), "kernel_status")
        return out.value

    def __del__(self):
        try:
            lib = _lib.load()
            for h in self._handles.values():
                lib.p2m_model_destroy(h)
        except Exception:
            pass


def graph_handle(L) -> GraphHandle:
    """Accepts what the reference passes (a torch sparse COO/CSR tensor, lib/models/meshnet.py:61-62,
    96) or a scipy sparse matrix; handles are cached per Laplacian object."""
    if isinstance(L, GraphHandle):
        return L
    key = id(L)
    hit = _graph_cache.get(key)
    if hit is not None and hit[0]() is L:
        return hit[1]
    if isinstance(L, torch.Tensor):
        t = L.detach().cpu()
        if t.layout == torch.sparse_csr:
            m = sp.csr_matrix((t.values().numpy(), t.col_indices().numpy(), t.crow_indices().numpy()),
                              shape=tuple(t.shape))
        else:
            t = t.coalesce() if t.is_sparse else t.to_sparse().coalesce()
            idx = t.indices().numpy()
            m = sp.csr_matrix((t.values().numpy(), (idx[0], idx[1])), shape=tuple(t.shape))
    else:
        m = sp.csr_matrix(L)
    gh = GraphHandle(m)
    try:
        # the entry (and with it the handle's device memory) goes away with the Laplacian object
        _graph_cache[key] = (weakref.ref(L, lambda _r, k=key: _graph_cache.pop(k, None)), gh)
    except TypeError:
        pass
    return gh


class ChebConvLinear(torch.autograd.Function):
    """z = [x | L~x | 2L~(L~x) - x] W^T + b  with W [Fout, 3*Fin], column = fin*3 + k."""

    @staticmethod
    def forward(ctx, x, weight, bias, gh: GraphHandle):
        lib = _lib.load()
        if not x.is_cuda:
            raise RuntimeError("pose2mesh_release_b200 runs on CUDA (sm_90a) only; got a CPU tensor")
        x = x.contiguous().float()
        B, V, fin = x.shape
        fout = weight.shape[0]
        if V != gh.V or weight.shape[1] != 3 * fin:
            raise ValueError(f"shape mismatch: x {tuple(x.shape)}, L {gh.V}, weight {tuple(weight.shape)}")
        dev = x.device
        h = gh.handle(dev.index)
        weight, bias = weight.contiguous().float(), bias.contiguous().float()
        y = torch.empty((B, V, fout), device=dev, dtype=torch.float32)
        nbytes = lib.p2m_cheb_conv_workspace_bytes(h, 0, B, fin, fout)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        a = _lib.ConvFwdArgs(level=0, batch=B, fin=fin, fout=fout, x=x.data_ptr(), weight=weight.data_ptr(),
                             bias=bias.data_ptr(), bn_mode=0, relu=0, y=y.data_ptr())
        _lib.call("p2m_cheb_conv_fwd", dev, h, C.byref(a), ws, nbytes)
        ctx.gh = gh
        ctx.save_for_backward(x, weight)
        return y

    @staticmethod
    def backward(ctx, dz):
        lib = _lib.load()
        x, weight = ctx.saved_tensors
        gh = ctx.gh
        B, V, fin = x.shape
        fout = weight.shape[0]
        dev = x.device
        h = gh.handle(dev.index)
        dz = dz.contiguous().float()
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(weight)
        db = torch.empty(fout, device=dev, dtype=torch.float32)
        nbytes = lib.p2m_cheb_conv_workspace_bytes(h, 0, B, fin, fout)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        a = _lib.ConvBwdArgs(level=0, batch=B, fin=fin, fout=fout, x=x.data_ptr(), weight=weight.data_ptr(),
                             dz=dz.data_ptr(), dx=None if dx is None else dx.data_ptr(), dweight=dw.data_ptr(),
                             dbias=db.data_ptr())
        _lib.call("p2m_cheb_conv_bwd", dev, h, C.byref(a), ws, nbytes)
        return dx, dw, db, None


def graph_conv_cheby(x, cl, bn, L, Fout, K):
    """Same signature and semantics as the reference (cheby_graph_conv.py:5): x [B,V,Fin], `cl` an
    nn.Linear(Fin*K, Fout), `bn` an nn.BatchNorm1d(Fout) or None, `L` the rescaled Laplacian."""
    if K != 3:
        raise NotImplementedError("pose2mesh_release_b200 implements the Chebyshev order the reference uses (K=3)")
    B, V, _ = x.shape
    if bn is not None and bn.training and _default_precision == _lib.P2M_PREC_FP16_TC:
        raise RuntimeError("graph_conv_cheby: precision 'fp16' is an inference precision; a training-mode BatchNorm "
                           "needs 'fp16x3' or 'fp32'")
    y = ChebConvLinear.apply(x, cl.weight, cl.bias, graph_handle(L))
    if y.shape[2] != Fout:
        raise ValueError("Fout does not match the Linear layer")
    if bn is not None:
        y = bn(y.view(B * V, Fout)).view(B, V, Fout)
    return y
