"""RMSprop on the device: a drop-in for ``torch.optim.RMSprop`` (the optimizer of every released config,
lib/funcs_utils.py:87-91) whose step is one launch of libp2m_b200.so's fused kernel per 448 parameter tensors.

torch's foreach path makes five passes over the parameters (about 13 floats of HBM traffic per parameter); the fused
step reads p, g and square_avg once and writes p and square_avg once (5 floats, 7 with momentum or centring).  The
arithmetic is torch's, operation for operation in fp32 (include/p2m_b200.h, p2m_rmsprop_step); the state (``step``,
``square_avg``, ``momentum_buffer``, ``grad_avg``) has torch's keys, shapes and dtypes, so state dicts load in either
direction.  ``step`` counters live on the parameters' device and are advanced by the kernel, and a 0-d CUDA tensor
``lr`` is read by the kernel when it runs, so a captured ``step()`` replays across ``MultiStepLR`` milestones.
"""
from __future__ import annotations

import torch

from . import _lib


class RMSprop(torch.optim.Optimizer):
    """torch.optim.RMSprop's constructor and semantics, stepped by libp2m_b200.so.  ``foreach`` and ``capturable`` are
    kept in the param groups (state dicts round-trip) and change nothing: the native step is always capturable.
    ``maximize=True`` and ``differentiable=True`` are not implemented (ValueError).  Construction accepts CPU
    parameters; ``step()`` needs contiguous float32 CUDA parameters, gradients and state on one device."""

    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False,
                 capturable=False, foreach=None, maximize=False, differentiable=False):
        if isinstance(lr, torch.Tensor) and lr.numel() != 1:
            raise ValueError("Tensor lr must be 1-element")
        for name, v in (("learning rate", lr), ("epsilon value", eps), ("momentum value", momentum),
                        ("weight_decay value", weight_decay), ("alpha value", alpha)):
            if not 0.0 <= v:
                raise ValueError(f"Invalid {name}: {v}")
        _check_supported(maximize, differentiable)
        defaults = {"lr": lr, "momentum": momentum, "alpha": alpha, "eps": eps, "centered": centered,
                    "weight_decay": weight_decay, "capturable": capturable, "foreach": foreach, "maximize": maximize,
                    "differentiable": differentiable}
        super().__init__(params, defaults)
        self._table = None  # _build_table's result, rebuilt when _pointers() changes

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            for k, v in (("momentum", 0), ("centered", False), ("foreach", None), ("maximize", False),
                         ("differentiable", False), ("capturable", False)):
                group.setdefault(k, v)
            for p in group["params"]:
                st = self.state.get(p, {})
                if len(st) != 0 and not torch.is_tensor(st["step"]):
                    st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)
        self._table = None

    def _entries(self):
        """(param, grad, state, group index) of every parameter with a gradient, its state created at its first step
        (torch's _init_group) and its step counter moved to the parameter's device."""
        out = []
        for gi, group in enumerate(self.param_groups):
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                if g.is_sparse:
                    raise RuntimeError("RMSprop does not support sparse gradients")
                for what, t in (("parameter", p), ("gradient", g)):
                    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                        raise RuntimeError(f"pose2mesh_release_b200.optim.RMSprop: every {what} must be a contiguous "
                                           f"float32 CUDA tensor; got {t.dtype} on {t.device}"
                                           f"{'' if t.is_contiguous() else ', not contiguous'}")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
                    st["square_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["momentum"] > 0:
                        st["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["centered"]:
                        st["grad_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                step = st["step"]
                if step.device != p.device or step.dtype != torch.float32:  # torch keeps it on the CPU
                    st["step"] = step.to(device=p.device, dtype=torch.float32)
                out.append((p, g, st, gi))
        return out

    def _pointers(self):
        """The segment table's contents (param, grad, square_avg, momentum_buffer, grad_avg, step pointers, numel,
        group) per parameter with a gradient, or None while a parameter with a gradient has no state yet."""
        key = []
        for gi, group in enumerate(self.param_groups):
            mom, cen = group["momentum"] > 0, group["centered"]
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                st = self.state.get(p)
                if not st:
                    return None
                key.append((p.data_ptr(), g.data_ptr(), st["square_avg"].data_ptr(),
                            st["momentum_buffer"].data_ptr() if mom else 0, st["grad_avg"].data_ptr() if cen else 0,
                            st["step"].data_ptr(), p.numel(), gi))
        return tuple(key)

    def _build_table(self):
        """Validate every parameter, gradient and state tensor (creating the state where missing) and pack the
        segment table; returns (pointer key, device, ctypes segments, {group index: table group index})."""
        entries = self._entries()
        if not entries:
            return None
        dev = entries[0][0].device
        for p, g, st, gi in entries:
            group = self.param_groups[gi]
            for t in (st["square_avg"], st["momentum_buffer"] if group["momentum"] > 0 else None,
                      st["grad_avg"] if group["centered"] else None):
                if t is not None and not (t.device == dev and t.dtype == torch.float32 and t.is_contiguous()
                                          and t.numel() == p.numel()):
                    raise RuntimeError("pose2mesh_release_b200.optim.RMSprop: the state must be contiguous float32 "
                                       f"tensors of the parameter's size on {dev}")
            if p.device != dev or g.device != dev or g.numel() != p.numel():
                raise RuntimeError(f"pose2mesh_release_b200.optim.RMSprop: parameters and gradients must be on one "
                                   f"device ({dev}) and of equal size")
        key = self._pointers()
        local = {}
        segs = (_lib.RmspropSegment * len(key))()
        for s, k in zip(segs, key):
            s.param, s.grad, s.square_avg, s.momentum_buffer, s.grad_avg, s.step, s.numel, _ = k
            s.group = local.setdefault(k[7], len(local))
        return key, dev, segs, local

    @torch.no_grad()
    def step(self, closure=None):
        """One RMSprop step of every parameter with a gradient; ``closure`` as in torch.optim (re-evaluates the model
        with gradients enabled and returns the loss, which step returns).  The tensors are validated and the segment
        table packed when a data pointer, size or group changes; otherwise the cached table is launched as it is."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            _check_supported(group["maximize"], group["differentiable"])
        key = self._pointers()
        if self._table is None or key is None or self._table[0] != key:
            self._table = self._build_table()
            if self._table is None:
                return loss
        _, dev, segs, local = self._table
        groups = (_lib.RmspropGroup * len(local))()
        for gi, k in local.items():
            group, d = self.param_groups[gi], groups[k]
            lr = group["lr"]
            if isinstance(lr, torch.Tensor):
                if not (lr.is_cuda and lr.device == dev and lr.dtype == torch.float32 and lr.numel() == 1):
                    raise RuntimeError(f"pose2mesh_release_b200.optim.RMSprop: a tensor lr must be a one-element "
                                       f"float32 tensor on {dev}; got {lr.dtype} on {lr.device}")
                d.lr, d.lr_device = 0.0, lr.data_ptr()
            else:
                d.lr, d.lr_device = float(lr), None
            d.alpha, d.eps = float(group["alpha"]), float(group["eps"])
            d.weight_decay, d.momentum = float(group["weight_decay"]), float(group["momentum"])
            d.centered = int(bool(group["centered"]))
        _lib.call("p2m_rmsprop_step", dev, segs, len(segs), groups, len(local))
        return loss


def _check_supported(maximize, differentiable):
    if maximize:
        raise ValueError("pose2mesh_release_b200.optim.RMSprop: maximize=True is not implemented")
    if differentiable:
        raise ValueError("pose2mesh_release_b200.optim.RMSprop: differentiable=True is not implemented")

