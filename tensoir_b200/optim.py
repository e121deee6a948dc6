"""FusedAdam: torch.optim.Adam's update (train_tensoIR.py:206, :315-317) for all parameters in ONE kernel launch
(csrc/tir_adam.cu), with the density L1 regulariser's gradient folded in, the gradients cleared in the same pass (the
backward kernels accumulate into persistent buffers) and a device-side ``found_inf`` skip flag — SURVEY.md §8 f3.

State layout follows torch.optim.Adam (``state[p] = {'step', 'exp_avg', 'exp_avg_sq'}``, ``step`` a 0-dim fp32 device
tensor as with ``capturable=True``), so optimizer checkpoints are interchangeable.  Like torch, every parameter counts its
own steps: one that gets no gradient is skipped and its count stays put, so a parameter that joins late starts its bias
corrections at step 1.  Learning rates may be floats or 0-dim device tensors (CUDA-graph replay, static_step.lr_tensors).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def _same_layout(a, b):
    return a.shape == b.shape and all(sa == sb for sa, sb, n in zip(a.stride(), b.stride(), a.shape) if n > 1)


def _moment(t, p):
    """A loaded exp_avg / exp_avg_sq laid out like its parameter: the kernel walks all four tensors in p's memory order."""
    if t.device == p.device and t.dtype == torch.float32 and _same_layout(t, p):
        return t
    return torch.empty_like(p, memory_format=torch.preserve_format).copy_(t)


def _own_step(step, dev):
    """``state["step"]`` as the parameter's own 0-dim fp32 tensor on ``dev``.  A loaded checkpoint may hold it as a
    number or a CPU tensor (torch.optim.Adam without capturable), or as a view that other parameters share."""
    if (torch.is_tensor(step) and step.device == dev and step.dtype == torch.float32 and step.dim() == 0
            and step.untyped_storage().nbytes() == 4):
        return step
    return torch.as_tensor(step).to(device=dev, dtype=torch.float32).reshape(()).clone()


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, l1=None, clear_grad=True):
        """``l1``: {parameter: coefficient} — adds coefficient * sign(parameter) to that parameter's gradient, i.e. the
        gradient of ``coefficient * parameter.abs().sum()`` (for ``w * mean|x|`` pass ``w / x.numel()``)."""
        # weight_decay / amsgrad / maximize: torch.optim.Adam's options at the values this update implements, so that a
        # state_dict of this optimizer loads into torch's
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=0.0, amsgrad=False, maximize=False))
        self.l1 = {id(p): float(c) for p, c in (l1 or {}).items()}
        self.clear_grad = bool(clear_grad)
        self._key = None
        self._keep = None

    def density_l1(self, model, weight):
        """Fold ``weight * model.density_L1()`` (tensoRF_rotated_lights.py:74-78: sum of mean |plane| + mean |line|)
        into the step; the caller then drops the term from its autograd loss."""
        for p in list(model.density_plane) + list(model.density_line):
            self.l1[id(p)] = float(weight) / p.numel()
        self._key = None

    def _dense(self, t):
        return t.is_contiguous() or (t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last))

    def _build(self, entries, dev):
        lib = _lib.load()
        chunk = lib.tir_adam_chunk_elems()
        table = (_lib.TirAdamTensor * len(entries))()
        prefix = [0]
        keep = []
        for k, (p, g, st, grp) in enumerate(entries):
            if not _same_layout(g, p) or not self._dense(p):
                raise _lib.TirError("FusedAdam needs dense parameters whose gradients share their layout "
                                    f"(got strides {tuple(p.stride())} / {tuple(g.stride())})")
            t = table[k]
            t.p, t.g, t.m, t.v, t.n = p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), p.numel()
            t.step = st["step"].data_ptr()
            lr = grp["lr"]
            if isinstance(lr, torch.Tensor):
                t.lr_dev, t.lr = lr.data_ptr(), 0.0
                keep.append(lr)
            else:
                t.lr_dev, t.lr = None, float(lr)
            t.l1 = self.l1.get(id(p), 0.0)
            prefix.append(prefix[-1] + (p.numel() + chunk - 1) // chunk)
        raw = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).clone()
        self._table = raw.to(dev)
        self._prefix = torch.tensor(prefix, dtype=torch.int64).to(dev)
        self._bias = torch.empty(2 * len(entries), device=dev)       # per entry: 1 - beta1^t, sqrt(1 - beta2^t)
        self._n, self._chunks = len(entries), prefix[-1]
        self._keep = keep

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        entries, dev = [], None
        beta1 = beta2 = eps = None
        for grp in self.param_groups:
            b1, b2 = grp["betas"]
            if beta1 is None:
                beta1, beta2, eps = float(b1), float(b2), float(grp["eps"])
            elif (beta1, beta2, eps) != (float(b1), float(b2), float(grp["eps"])):
                raise _lib.TirError("FusedAdam: betas / eps must be the same for every parameter group")
            if grp.get("weight_decay", 0.0) or grp.get("amsgrad", False) or grp.get("maximize", False):
                raise _lib.TirError("FusedAdam implements Adam without weight_decay, amsgrad or maximize")
            for p in grp["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                else:
                    st["step"] = _own_step(st["step"], p.device)
                    st["exp_avg"] = _moment(st["exp_avg"], p)
                    st["exp_avg_sq"] = _moment(st["exp_avg_sq"], p)
                dev = p.device
                entries.append((p, p.grad, st, grp))
        if not entries:
            return loss
        key = tuple((p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                     st["step"].data_ptr(),
                     grp["lr"].data_ptr() if isinstance(grp["lr"], torch.Tensor) else float(grp["lr"]),
                     self.l1.get(id(p), 0.0)) for p, g, st, grp in entries)
        if key != self._key:
            self._build(entries, dev)
            self._key = key
        lib = _lib.load()
        fi = getattr(self, "found_inf", None)
        _lib.check(lib.tir_adam_step(C.c_void_p(self._table.data_ptr()), self._n, C.c_void_p(self._prefix.data_ptr()),
                                     self._chunks, C.c_void_p(self._bias.data_ptr()), beta1, beta2, eps,
                                     None if fi is None else C.c_void_p(fi.data_ptr()), int(self.clear_grad),
                                     _lib.stream_ptr()), "tir_adam_step")
        return loss

    def zero_grad(self, set_to_none: bool = False):
        """With ``clear_grad`` the step itself leaves every gradient zeroed and IN PLACE (the fused backward kernels keep
        accumulating into the same buffers), so this is a no-op unless the caller insists on dropping them."""
        if set_to_none or not self.clear_grad:
            return super().zero_grad(set_to_none=set_to_none)
