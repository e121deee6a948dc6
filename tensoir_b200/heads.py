"""Fused appearance heads for the primary march: appearance gather -> light factor -> basis_mat -> positional
encoding -> 3-layer MLP in ONE tensor-core kernel launch (csrc/tir_mlp.cu), as a differentiable op.

The forward dumps the activations (light-scaled products, MLP input, both hidden layers); the backward is a short
hand-written chain of GEMMs on those dumps (no autograd graph, no recomputation) that ends in the appearance scatter
kernel.  Replaces, per head, compute_{app,intrin}feature + MLPRender_Fea / MLPBRDF_PEandFeature
(tensoRF_rotated_lights.py:167-224, tensorBase_rotated_lights.py:122-208) and their ~60 autograd nodes.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, ops
from .device_field import mlp_struct
from .vm_autograd import _grad_shadows, _ptr_array, _to_param_layout


def _wgrad(g, a, splits=32):
    """g^T @ a for tall-skinny operands ([n, <=128]^T @ [n, <=150], n ~ 2e4).  cuBLAS tiles only the tiny output
    (6 CTAs on 132 SMs); splitting the reduction over n into `splits` batched GEMMs fills the machine."""
    n = g.shape[0]
    per = n // splits
    if per < 64:
        return g.t() @ a
    main = per * splits
    out = torch.bmm(g[:main].view(splits, per, -1).transpose(1, 2), a[:main].view(splits, per, -1)).sum(0)
    if main < n:
        out = out + g[main:].t() @ a[main:]
    return out


def _head_forward(model, head, light, xn, x_in, li, w0, need, bufs=None):
    """One fused kernel launch; returns (out, xl, inp, h1, h2) (the dumps are None when no gradient is needed).
    ``bufs`` = (xl, inp, h1, h2) destination tensors (slices of stacked buffers) to dump into instead of new ones."""
    lib = _lib.load()
    f = ops.device_field(model).refresh(model)
    keep = []
    mlp = mlp_struct(model, head, keep, light=light)
    n, dev = xn.shape[0], xn.device
    act = 1 if head == "renderModule_normal" else 0
    out = torch.empty(n, mlp.out_dim, device=dev)
    k0, in_dim, hid = 3 * f.aC, w0.shape[1], w0.shape[0]
    if need and bufs is not None:
        xl, inp, h1, h2 = bufs
    else:
        xl = torch.empty(n, k0, device=dev) if need else None
        inp = torch.empty(n, in_dim, device=dev) if need else None
        h1 = torch.empty(n, hid, device=dev) if need else None
        h2 = torch.empty(n, hid, device=dev) if need else None
    nul = C.c_void_p(0)
    _lib.check(lib.tir_app_mlp_points_save(
        C.byref(f), C.byref(mlp), _lib.dptr(xn), _lib.dptr(x_in),
        None if (li is None or li.numel() == 0 or light != "index") else _lib.dptr(li, torch.int32), n, act,
        _lib.dptr(out), _lib.dptr(xl) if need else nul, _lib.dptr(inp) if need else nul,
        _lib.dptr(h1) if need else nul, _lib.dptr(h2) if need else nul, _lib.stream_ptr()), "tir_app_mlp_points_save")
    return out, xl, inp, h1, h2


def _wgrad_batched(g, a):
    """Per-head g_h^T @ a_h for stacked operands g [H,n,M], a [H,n,K] -> [H,M,K]; reduction over n split like _wgrad:
    8 slices per head from three heads on, 16 for two and _wgrad's 32 for a single head."""
    H, n, M = g.shape
    splits = 8 * max(1, 4 // H)
    per = n // splits
    if per < 64:
        return torch.bmm(g.transpose(1, 2), a)
    main = per * splits
    out = torch.bmm(g[:, :main].reshape(H * splits, per, M).transpose(1, 2),
                    a[:, :main].reshape(H * splits, per, -1)).view(H, splits, M, -1).sum(1)
    if main < n:
        out = out + torch.bmm(g[:, main:].transpose(1, 2), a[:, main:])
    return out


def _heads_backward_batched(is_tanh, g_out, out, xl, inp, h1, h2, w0, w1, w2, basis):
    """Hand-written backward of the MLP, PE and basis_mat of H heads at once (equal sample counts) on their dumped
    activations, as batched GEMMs and stacked elementwise ops.  is_tanh [H] bool; g_out / out [H,n,4] (3-output heads zero-padded); xl [H,n,3*aC];
    inp [H,n,in_dim]; h1, h2 [H,n,hid]; w0 [H,hid,in_dim]; w1 [H,hid,hid]; w2 [H,4,hid] (zero-padded rows).
    -> gw0, gb0, gw1, gb1, gw2 [H,4,hid], gb2 [H,4], gbasis (summed over heads), gxl [H,n,3*aC]."""
    H, n, _ = out.shape
    dact = torch.where(is_tanh.view(H, 1, 1), 1 - out * out, out * (1 - out))
    gz3 = g_out * dact
    gw2, gb2 = torch.bmm(gz3.transpose(1, 2), h2), gz3.sum(1)
    gz2 = torch.bmm(gz3, w2) * (h2 > 0)
    gw1, gb1 = _wgrad_batched(gz2, h1), gz2.sum(1)
    gz1 = torch.bmm(gz2, w1) * (h1 > 0)
    gw0, gb0 = _wgrad_batched(gz1, inp), gz1.sum(1)
    gin = torch.bmm(gz1, w0)                                   # [H, n, in_dim]
    F, pe = basis.shape[0], 2
    s0, c0 = F + 3, F + 3 + F * pe
    freqs = 2.0 ** torch.arange(pe, device=out.device, dtype=inp.dtype)
    gs, gc = gin[..., s0:s0 + F * pe].reshape(H, n, F, pe), gin[..., c0:c0 + F * pe].reshape(H, n, F, pe)
    sn, cs = inp[..., s0:s0 + F * pe].reshape(H, n, F, pe), inp[..., c0:c0 + F * pe].reshape(H, n, F, pe)
    gfeat = gin[..., :F] + ((gs * cs - gc * sn) * freqs).sum(-1)           # [H, n, F]
    gbasis = _wgrad(gfeat.reshape(H * n, F), xl.reshape(H * n, -1))
    gxl = (gfeat.reshape(H * n, F) @ basis).view(H, n, -1)
    return gw0, gb0, gw1, gb1, gw2, gb2, gbasis, gxl


class _FusedHeadsMulti(torch.autograd.Function):
    """H heads with equal sample counts, each at its own points.  Forward: one kernel launch per head, dumping into
    stacked [H, n, *] buffers.  Backward: ONE stacked chain (_heads_backward_batched) for all heads, then one
    appearance scatter per group of heads that share their points, all into the same gradient buffers."""

    @staticmethod
    def forward(ctx, model, specs, basis, light_w, *rest):
        nh = len(specs)                      # specs: (head, light, group)
        per = rest[:9 * nh]                  # per head: xn, x_in, li, w0, b0, w1, b1, w2, b2
        need = any(ctx.needs_input_grad)
        n, dev = per[0].shape[0], per[0].device
        f = ops.device_field(model).refresh(model)
        k0, in_dim, hid = 3 * f.aC, per[3].shape[1], per[3].shape[0]
        bufs = None
        if need:
            bufs = (torch.empty(nh, n, k0, device=dev), torch.empty(nh, n, in_dim, device=dev),
                    torch.empty(nh, n, hid, device=dev), torch.empty(nh, n, hid, device=dev))
        outs, saved = [], []
        for h, (head, light, _) in enumerate(specs):
            xn, x_in, li, w0, b0, w1, b1, w2, b2 = per[9 * h:9 * h + 9]
            out, *_ = _head_forward(model, head, light, xn, x_in, li, w0, need,
                                    None if bufs is None else tuple(b[h] for b in bufs))
            outs.append(out)
            if need:
                saved += [out, xn, li, w0, w1, w2]
        ctx.model, ctx.specs = model, specs
        ctx.has_light = light_w is not None
        ctx.save_for_backward(basis, light_w if light_w is not None else torch.empty(0, device=dev),
                              *(bufs if need else ()), *saved)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *g_outs):
        basis, light_w, xl, inp, h1, h2, *saved = ctx.saved_tensors
        model, specs = ctx.model, ctx.specs
        nh, n, dev = len(specs), xl.shape[1], xl.device
        outs = [saved[6 * h] for h in range(nh)]
        xns = [saved[6 * h + 1] for h in range(nh)]
        lis = [saved[6 * h + 2] for h in range(nh)]
        out_p, g_p = torch.zeros(nh, n, 4, device=dev), torch.zeros(nh, n, 4, device=dev)
        w2_p = torch.zeros(nh, 4, h2.shape[2], device=dev)
        is_tanh = torch.zeros(nh, dtype=torch.bool, device=dev)
        for h, (head, _, _) in enumerate(specs):
            od = outs[h].shape[1]
            out_p[h, :, :od] = outs[h]
            if g_outs[h] is not None:
                g_p[h, :, :od] = g_outs[h]
            w2_p[h, :od] = saved[6 * h + 5]
            if head == "renderModule_normal":
                is_tanh[h].fill_(True)          # device-side fill (graph-capturable)
        w0 = torch.stack([saved[6 * h + 3] for h in range(nh)])
        w1 = torch.stack([saved[6 * h + 4] for h in range(nh)])
        gw0, gb0, gw1, gb1, gw2, gb2, gbasis, gxl = _heads_backward_batched(is_tanh, g_p, out_p, xl, inp, h1, h2, w0,
                                                                           w1, w2_p, basis)
        lib = _lib.load()
        df = ops.device_field(model)
        f = df.refresh(model)
        gp, gl = _grad_shadows(df, "app")
        glight, per_grads = None, []
        groups = {}
        for h, (_, _, grp) in enumerate(specs):
            groups.setdefault(grp, []).append(h)
        for members in groups.values():
            xn = xns[members[0]]
            x0 = _raw_products(model, xn) if any(specs[h][1] != "none" for h in members) else None
            gx0 = None
            for h in members:
                light = specs[h][1]
                if light == "none":
                    g_h = gxl[h]
                elif light == "index":                               # xl = x0 * light_line[li]
                    idx = lis[h].long()
                    gl_h = torch.zeros_like(light_w).index_add_(0, idx, gxl[h] * x0)
                    glight = gl_h if glight is None else glight + gl_h
                    g_h = gxl[h] * light_w.index_select(0, idx)
                else:                                                # xl = x0 * mean over lights
                    gl_h = ((gxl[h] * x0).sum(0, keepdim=True) / light_w.shape[0]).expand_as(light_w)
                    glight = gl_h if glight is None else glight + gl_h
                    g_h = gxl[h] * light_w.mean(0, keepdim=True)
                gx0 = g_h if gx0 is None else gx0 + g_h
            gx0 = gx0.contiguous()
            _lib.check(lib.tir_vm_app_products_bwd(C.byref(f), _lib.dptr(xn), n, _lib.dptr(gx0), _ptr_array(gp),
                                                   _ptr_array(gl), _lib.stream_ptr()), "tir_vm_app_products_bwd")
        for h in range(nh):
            od = outs[h].shape[1]
            per_grads += [None, None, None, gw0[h], gb0[h], gw1[h], gb1[h], gw2[h, :od], gb2[h, :od]]
        return (None, None, gbasis, glight if ctx.has_light else None, *per_grads, *_to_param_layout(gp, gl))


def fused_heads_multi(model, specs):
    """Evaluate several heads, each at its own points, with ONE stacked backward.
    specs: list of (head, xn, x_in, light_idx or None, light) — all with the same number of points; heads given the
    SAME ``xn`` tensor object share one backward scatter.  -> tuple of [n, out_dim_h]."""
    dev = specs[0][1].device
    ll = getattr(model, "light_line", None)
    use_light = ll is not None and any(s[4] != "none" for s in specs)
    light_w = ll.weight if use_light else None
    flat, meta, seen = [], [], {}
    n = None
    for head, xn, x_in, li, light in specs:
        grp = seen.setdefault(id(xn), len(seen))
        mod = getattr(model, head)
        xn_c = xn.detach().reshape(-1, 3).float().contiguous()
        if n is None:
            n = xn_c.shape[0]
        elif xn_c.shape[0] != n:
            raise ValueError("fused_heads_multi needs the same number of points for every head")
        x_in = x_in.detach().reshape(-1, 3).float().contiguous()
        li = (torch.empty(0, dtype=torch.int32, device=dev) if li is None
              else li.detach().reshape(-1).to(torch.int32).contiguous())
        flat += [xn_c, x_in, li, mod.mlp[0].weight, mod.mlp[0].bias, mod.mlp[2].weight, mod.mlp[2].bias,
                 mod.mlp[4].weight, mod.mlp[4].bias]
        meta.append((head, light if ll is not None else "none", grp))
    params = list(model.app_plane) + list(model.app_line)
    return _FusedHeadsMulti.apply(model, tuple(meta), model.basis_mat.weight, light_w, *flat, *params)


def _raw_products(model, xn):
    lib = _lib.load()
    f = ops.device_field(model).refresh(model)
    out = torch.empty(xn.shape[0], 3 * f.aC, device=xn.device)
    _lib.check(lib.tir_vm_app_products(C.byref(f), _lib.dptr(xn), xn.shape[0], _lib.dptr(out), _lib.stream_ptr()),
               "tir_vm_app_products")
    return out


def fused_head(model, head: str, xn, x_in, light_idx=None, light: str = "index"):
    """One head at the points ``xn``: head in {'renderModule' (x_in = view dir, sigmoid), 'renderModule_brdf' (x_in =
    position, sigmoid, 4 outputs), 'renderModule_normal' (position, tanh)}, light in {'index', 'mean', 'none'}.
    out = act(MLP([feat, x_in, PE(feat), PE(x_in)])) with feat = basis_mat(plane*line(xn) * lightvec) -> [n, out_dim]."""
    return fused_heads_multi(model, [(head, xn, x_in, light_idx, light)])[0]
