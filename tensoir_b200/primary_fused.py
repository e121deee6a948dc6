"""TensorBase.forward with is_relight=True (models/tensorBase_rotated_lights.py:868-1036) as ONE autograd node around
the fused C entry points ``tir_primary_march`` / ``tir_primary_app_list`` / ``tir_primary_heads`` /
``tir_primary_backward`` (csrc/tir_primary.cu): 12 kernel launches forward, 9 backward, no torch glue in between.

All sample lists live in a cached workspace of static capacity; their real lengths stay on the device.  Eagerly the
host reads the three status words once per forward (the only synchronisation) to grow the workspace when a list did not
fit — then the march is simply run again, so eager results never depend on capacities.  Under CUDA-graph capture
(``static_step.py``) nothing is read back: the lengths go into the step's statistics and an overflow raises the step's
device-side flag instead.
"""
from __future__ import annotations

import ctypes as C
from collections import namedtuple

import torch

from . import _lib, ops
from .device_field import mlp_struct

HEAD_RGB, HEAD_BRDF, HEAD_BRDF_JITTER, HEAD_NORMAL = 0, 1, 2, 3
NORMALS = {"derived_plus_predicted": 0, "purely_predicted": 1, "purely_derived": 2}


TirHeadJob, TirPrimaryWork, TirPrimaryBwdWork, TirPrimaryGrads = (_lib.TirHeadJob, _lib.TirPrimaryWork,
                                                                 _lib.TirPrimaryBwdWork, _lib.TirPrimaryGrads)


class Workspace:
    """Scratch of one primary march: per-ray arrays, the valid list, the appearance list and (training) the
    activation dumps + backward scratch.  Re-used across calls; grown, never shrunk."""

    def __init__(self, device, point_sets=2):
        self.dev = device
        self.point_sets = point_sets      # 1: no jittered point set (radiance-only forward), so no second x0 dump
        self.n_rays = self.cap_valid = self.cap_app = 0
        self.n_jobs = 0
        self.grad = False
        self.busy = False          # holds the activation dumps of a forward whose backward has not run yet
        self.t = {}

    def _alloc(self, name, shape, dtype=torch.float32):
        self.t[name] = torch.empty(shape, dtype=dtype, device=self.dev)

    def ensure(self, n_rays, cap_valid, cap_app, n_jobs, grad):
        if (n_rays == self.n_rays and cap_valid <= self.cap_valid and cap_app <= self.cap_app and n_jobs <= self.n_jobs
                and (self.grad or not grad)):
            return False
        cap_valid, cap_app = max(cap_valid, self.cap_valid), max(cap_app, self.cap_app)
        n_jobs, grad = max(n_jobs, self.n_jobs), grad or self.grad
        self.t = {}
        a = self._alloc
        a("counts", n_rays, torch.int32); a("offsets", n_rays + 1, torch.int64)
        a("t_last", n_rays); a("acc", n_rays); a("depth", n_rays)
        a("a_counts", n_rays, torch.int32); a("a_offsets", n_rays + 1, torch.int64)
        a("packed", (n_rays, 14))
        a("v_ray", cap_valid, torch.int32); a("v_sample", cap_valid, torch.int32)
        a("v_xn", (cap_valid, 3)); a("v_z", cap_valid); a("v_dist", cap_valid)
        a("v_feat", cap_valid); a("v_sigma", cap_valid); a("v_weight", cap_valid); a("v_trans", cap_valid)
        a("a_src", cap_app, torch.int64); a("a_ray", cap_app, torch.int32)
        a("a_w", cap_app); a("a_xn", (cap_app, 3)); a("a_xj", (cap_app, 3))
        a("dn_feat", cap_app); a("dn_dfdx", (cap_app, 3))
        a("status", 4, torch.int64)
        for j in range(n_jobs):
            a(f"out{j}", (cap_app, 4))
        if grad:
            a("x0_0", (cap_app, 144))
            if self.point_sets > 1:
                a("x0_1", (cap_app, 144))
            a("g_packed", (n_rays, 14)); a("g_acc", n_rays); a("g_depth", n_rays)
            a("g_weight", cap_valid); a("g_feat", cap_valid)
            a("g_dn_feat", cap_app); a("g_dn_dfdx", (cap_app, 3))
            for j in range(n_jobs):
                a(f"inp{j}", (cap_app, 150)); a(f"h1_{j}", (cap_app, 128)); a(f"h2_{j}", (cap_app, 128))
                a(f"g_out{j}", (cap_app, 4)); a(f"gz1_{j}", (cap_app, 128)); a(f"gz2_{j}", (cap_app, 128))
                a(f"gfeat{j}", (cap_app, 32)); a(f"gx0_{j}", (cap_app, 144))
        self.n_rays, self.cap_valid, self.cap_app, self.n_jobs, self.grad = n_rays, cap_valid, cap_app, n_jobs, grad
        return True

    def work_struct(self, noise, n_jobs, grad):
        w = TirPrimaryWork()
        w.cap_valid, w.cap_app = self.cap_valid, self.cap_app
        t = self.t
        for k in ("counts", "offsets", "t_last", "acc", "depth", "a_counts", "a_offsets", "packed", "v_ray", "v_sample",
                  "v_xn", "v_z", "v_dist", "v_feat", "v_sigma", "v_weight", "v_trans", "a_src", "a_ray", "a_w", "a_xn",
                  "a_xj", "dn_feat", "dn_dfdx", "status"):
            setattr(w, k, t[k].data_ptr())
        w.noise = None if noise is None else noise.data_ptr()
        for j in range(n_jobs):
            w.out[j] = t[f"out{j}"].data_ptr()
            if grad:
                w.inp[j], w.h1[j], w.h2[j] = t[f"inp{j}"].data_ptr(), t[f"h1_{j}"].data_ptr(), t[f"h2_{j}"].data_ptr()
        if grad:
            w.x0[0] = t["x0_0"].data_ptr()
            w.x0[1] = t["x0_1"].data_ptr() if "x0_1" in t else None
        return w

    def bwd_struct(self, n_jobs):
        b = TirPrimaryBwdWork()
        t = self.t
        for k in ("g_packed", "g_acc", "g_depth", "g_weight", "g_feat", "g_dn_feat", "g_dn_dfdx"):
            setattr(b, k, t[k].data_ptr())
        for j in range(n_jobs):
            b.g_out[j], b.gz1[j], b.gz2[j] = t[f"g_out{j}"].data_ptr(), t[f"gz1_{j}"].data_ptr(), t[f"gz2_{j}"].data_ptr()
            b.gfeat[j], b.gx0[j] = t[f"gfeat{j}"].data_ptr(), t[f"gx0_{j}"].data_ptr()
        return b


# Every head job of the primary march: (module, role, point set, x_in, light mode when the model has a light_line, act).
# The relight phase (tensorBase:930-1004) runs all of them, renderModule_normal only when the normals are predicted; the
# radiance-only phase runs the renderModule row alone: the view direction in, light_line[light_idx] if the model has one.
_JOB_SPEC = (("renderModule", HEAD_RGB, 0, 0, 1, 0),
             ("renderModule_brdf", HEAD_BRDF, 0, 1, 2, 0),
             ("renderModule_brdf", HEAD_BRDF_JITTER, 1, 1, 2, 0),
             ("renderModule_normal", HEAD_NORMAL, 0, 1, 2, 1))
HEADS = ("renderModule", "renderModule_brdf", "renderModule_normal")


def _jobs(model, keep, heads=HEADS):
    """The job table of a node over the head modules ``heads`` -> (TirHeadJob array, n_jobs, module of every job,
    normals kind)."""
    kind = NORMALS[model.normals_kind]
    has_light = getattr(model, "light_line", None) is not None
    spec = [s for s in _JOB_SPEC if s[0] in heads and not (s[1] == HEAD_NORMAL and kind == 2)]
    arr = (TirHeadJob * len(spec))()
    for j, (head, role, ps, x_in, lm, act) in enumerate(spec):
        arr[j].mlp = mlp_struct(model, head, keep, light="index" if has_light else "none")
        arr[j].point_set, arr[j].x_in, arr[j].act, arr[j].role = ps, x_in, act, role
        arr[j].light_mode = lm if has_light else 0
    return arr, len(spec), [s[0] for s in spec], kind


def _radiance_job(model, keep):
    """The one job of the radiance-only node: the renderModule row of the job table."""
    return _jobs(model, keep, HEADS[:1])[0][0]


def _workspace(model, key, dev, need, point_sets):
    """The cached workspace of ``model.__dict__[key]``, marked busy until the backward when ``need``."""
    ws = model.__dict__.get(key)
    if ws is None or ws.dev != dev:
        ws = Workspace(dev, point_sets)
        model.__dict__[key] = ws
    if ws.busy and model.__dict__.get("_tir_static") is None:
        # a previous training forward still waits for its backward (several chunks per step): its dumps live in the
        # cached workspace, so this call gets a private one
        ws = Workspace(dev, point_sets)
    ws.busy = need
    return ws


def _march(lib, f, rays, cfg, ws, n_jobs, need, counters, st):
    """tir_primary_march + tir_primary_app_list -> (work struct, appearance rows; None in shape-static mode)."""
    n_rays = rays.shape[0]
    cptr = None if counters is None else _lib.dptr(counters, torch.int64)
    if st is not None:
        ws.ensure(n_rays, st["cap_valid"], st["cap_app"], n_jobs, need)
    else:
        ws.ensure(n_rays, max(ws.cap_valid, 96 * n_rays + 1024), max(ws.cap_app, 8 * n_rays + 1024), n_jobs, need)
    stream = _lib.stream_ptr()
    snap = counters.clone() if (counters is not None and st is None) else None
    n_app = None
    while True:
        w = ws.work_struct(None, n_jobs, need)
        _lib.check(lib.tir_primary_march(C.byref(f), _lib.dptr(rays), n_rays, C.byref(cfg), C.byref(w), cptr, stream),
                   "tir_primary_march")
        if st is not None:
            # shape-static mode: the kernels already left the real list lengths and the overflow flag on the device
            st["stats"][0:2].copy_(ws.t["status"][0:2])
            st["overflow_step"].add_(ws.t["status"][2])
            break
        n_valid, n_app, _, _ = ws.t["status"].tolist()          # the one host read of the eager forward
        if n_valid <= ws.cap_valid and n_app <= ws.cap_app:
            break
        if counters is not None:      # the march runs again: do not count its rays twice
            counters.copy_(snap)
        ws.ensure(n_rays, int(1.25 * n_valid) + 1024, int(1.25 * n_app) + 1024, n_jobs, need)
    if counters is not None:
        counters[_lib.CNT_APP] += ws.t["status"][1]
    _lib.check(lib.tir_primary_app_list(C.byref(f), n_rays, C.byref(w), stream), "tir_primary_app_list")
    return w, n_app


def _vm_factors(model):
    """The VM factors in the order density planes, density lines, app planes, app lines."""
    return list(model.density_plane) + list(model.density_line) + list(model.app_plane) + list(model.app_line)


def _head_params(model, head):
    m = getattr(model, head).mlp
    return [m[0].weight, m[0].bias, m[2].weight, m[2].bias, m[4].weight, m[4].bias]


def _params(model, heads):
    """Autograd inputs of a primary node: VM factors, basis, [light_line], 6 tensors per head."""
    params = _vm_factors(model) + [model.basis_mat.weight]
    ll = getattr(model, "light_line", None)
    if ll is not None:
        params.append(ll.weight)
    for head in heads:
        params += _head_params(model, head)
    return params


def _vm_target(p, inplace):
    """(buffer the kernels accumulate into, what autograd gets) for a VM factor: its own .grad when that is dense in
    the parameter's channel-last layout, else a zeroed buffer in the kernels' layout and its view in the parameter's
    shape."""
    g = p.grad
    if (inplace and g is not None and g.dtype == torch.float32 and g.shape == p.shape and p.shape[0] == 1
            and all(a == b for a, b, n in zip(g.stride(), p.stride(), p.shape) if n > 1)
            and p.is_contiguous(memory_format=torch.channels_last)):
        return g, None
    _, Cc, H, W = p.shape
    buf = torch.zeros((H, W, Cc), device=p.device, dtype=torch.float32)
    return buf, buf.permute(2, 0, 1).unsqueeze(0)


def _grad_target(p, inplace):
    """(buffer the kernels accumulate into, what autograd gets): the parameter's own .grad when it is a plain fp32
    tensor of the same layout (then autograd gets None: no zero-fill, no AccumulateGrad add), else zeros."""
    g = p.grad
    if inplace and g is not None and g.dtype == torch.float32 and g.shape == p.shape and g.is_contiguous() \
            and p.is_contiguous():
        return g, None
    z = torch.zeros_like(p)
    return z, z


def _grad_targets(model, heads, job_heads):
    """The parameter gradients of a node over the head modules ``heads`` whose job j runs ``job_heads[j]`` ->
    (TirPrimaryGrads, the gradients autograd gets in the order of _params(model, heads): None for a head without a job).

    When a parameter already HAS a dense .grad (kept zeroed in place by tensoir_b200.optim.FusedAdam, or the views of a
    dp.GradBucket) the kernels accumulate straight into it and autograd gets None for that input: for the VM factors
    (17-31 M floats) no 70 MB allocation + memset + AccumulateGrad pass per step.  With ``model._tir_grad_inplace``
    off, or without such a .grad, a zeroed buffer is returned the usual way."""
    inplace = model.__dict__.get("_tir_grad_inplace", True)
    gr = TirPrimaryGrads()
    grads = []
    for k, p in enumerate(_vm_factors(model)):
        buf, ret = _vm_target(p, inplace)
        (gr.dplane, gr.dline, gr.aplane, gr.aline)[k // 3][k % 3] = buf.data_ptr()
        grads.append(ret)
    buf, ret = _grad_target(model.basis_mat.weight, inplace)
    gr.basis = buf.data_ptr()
    grads.append(ret)
    ll = getattr(model, "light_line", None)
    if ll is not None:
        buf, ret = _grad_target(ll.weight, inplace)
        gr.light_line = buf.data_ptr()
        grads.append(ret)
    for head in heads:
        slots = [j for j, h in enumerate(job_heads) if h == head]
        if not slots:
            grads += [None] * 6
            continue
        ts = [_grad_target(t, inplace) for t in _head_params(model, head)]
        for j in slots:
            gr.w0[j], gr.b0[j], gr.w1[j], gr.b1[j], gr.w2[j], gr.b2[j] = [t[0].data_ptr() for t in ts]
        grads += [t[1] for t in ts]
    return gr, tuple(grads)


# ctx.keep of the two nodes: what their backwards read, and the host tensors (keep) their job tables and march configs
# point into.  cfg: the TirMarchCfg of the march, noise: the smoothness term's xyz noise, li: int32 light index per ray,
# bg: the background flag.
_RelightKeep = namedtuple("_RelightKeep", "keep jobs n_jobs kind cfg noise li rays ws jitter")
_RadianceKeep = namedtuple("_RadianceKeep", "keep jobs li rays ws jitter bg")


def _forward_common(ctx, model, rays, light_idx, is_train, n_samples, jitter, heads, ws_key):
    """What both nodes' forwards do before their own C call: field refresh, job table, march config, workspace, march
    and appearance list; ``ctx`` gets the model and the heads its backward hands gradients to -> (library, field,
    work struct, appearance rows (None in shape-static mode), keep, jobs, normals kind, march config, int32 light
    indices, workspace)."""
    lib = _lib.load()
    need = any(ctx.needs_input_grad)
    f = ops.device_field(model).refresh(model, force=bool(is_train))
    keep = []
    jobs, n_jobs, job_heads, kind = _jobs(model, keep, heads)
    cfg = ops.march_cfg(model, n_samples=n_samples, jitter=jitter, keep=keep)
    point_sets = 1 + max(jobs[j].point_set for j in range(n_jobs))
    ws = _workspace(model, ws_key, rays.device, need, point_sets)
    li = light_idx.reshape(-1).to(torch.int32).contiguous()
    w, n_app = _march(lib, f, rays, cfg, ws, n_jobs, need, model.__dict__.get("_tir_counters"),
                      model.__dict__.get("_tir_static"))
    ctx.model, ctx.heads, ctx.job_heads = model, heads, job_heads
    return lib, f, w, n_app, keep, jobs, kind, cfg, li, ws


def _f32(t):
    return None if t is None else t.contiguous().float()


def _ptr(t):
    return None if t is None else _lib.dptr(t)


# per-ray shape of the maps of TensorBase.forward's 12-tuple: rgb, depth, normal, albedo, roughness, fresnel, acc,
# normals_diff, normals_orientation, acc_mask; the albedo and roughness smoothness losses follow
_MAP_SHAPES = ((3,), (), (3,), (3,), (1,), (3,), (), (1,), (1,), ())
_RAY_MAPS = (0, 1, 2, 3, 4, 5, 7, 8)        # the entries TirRayMaps holds, in its field order


def _ray_maps(ts):
    maps = _lib.TirRayMaps()
    for k, t in zip(("rgb", "depth", "normal", "albedo", "rough", "fresnel", "nd", "no"), ts):
        setattr(maps, k, None if t is None else t.data_ptr())
    return maps


class _PrimaryRelight(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, rays, light_idx, white_bg, is_train, n_samples, bg_flag, jitter, *params):
        lib, f, w, n_app, keep, jobs, kind, cfg, li, ws = _forward_common(ctx, model, rays, light_idx, is_train,
                                                                          n_samples, jitter, HEADS, "_tir_primary_ws")
        dev, n_rays = rays.device, rays.shape[0]
        # xyz noise of the smoothness term: randn_like(xyz_sampled[app_mask]) (tensorBase:937), drawn on the device in
        # list order; the eager path draws exactly n_app rows like the reference
        draw = model.__dict__.get("_tir_randn_like")       # test hook: replay the oracle's stream / deterministic noise
        rows = ws.cap_app if model.__dict__.get("_tir_static") is not None else int(n_app)
        noise = torch.zeros(ws.cap_app, 3, device=dev)
        if rows > 0:
            x_a = ws.t["a_xn"][:rows]
            noise[:rows] = draw(x_a) if draw is not None else torch.randn_like(x_a)
        w.noise = noise.data_ptr()
        outs = [torch.empty((n_rays,) + _MAP_SHAPES[k], device=dev) for k in _RAY_MAPS]
        mask = torch.empty(n_rays, dtype=torch.bool, device=dev)
        losses = torch.empty(2, device=dev)
        counters = model.__dict__.get("_tir_counters")
        _lib.check(lib.tir_primary_heads(C.byref(f), jobs, len(jobs), kind, _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                         n_rays, C.byref(w), float(model.fixed_fresnel), int(bool(bg_flag)),
                                         C.byref(_ray_maps(outs)), _lib.dptr(mask, torch.bool), _lib.dptr(losses),
                                         None if counters is None else _lib.dptr(counters, torch.int64),
                                         _lib.stream_ptr()), "tir_primary_heads")
        if kind == 1:
            _lib.launch_count -= 1          # no derived-normal gather
        acc = ws.t["acc"].clone()
        ctx.bg = int(bool(bg_flag))
        ctx.keep = _RelightKeep(keep, jobs, len(jobs), kind, cfg, noise, li, rays, ws, jitter)
        ctx.mark_non_differentiable(mask)
        rgb, depth, normal, albedo, rough, fresnel, nd, no = outs
        return rgb, depth, normal, albedo, rough, fresnel, acc, nd, no, mask, losses[0], losses[1]

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_normal, g_albedo, g_rough, g_fresnel, g_acc, g_nd, g_no, _g_mask, g_la, g_lr):
        k, model = ctx.keep, ctx.model
        lib = _lib.load()
        f = ops.device_field(model).refresh(model)
        gs = [_f32(t) for t in (g_rgb, g_depth, g_normal, g_albedo, g_rough, g_fresnel, g_nd, g_no)]
        g_acc = _f32(g_acc)
        g_la, g_lr = [None if t is None else _f32(t.reshape(1)) for t in (g_la, g_lr)]
        w, b = k.ws.work_struct(k.noise, k.n_jobs, True), k.ws.bwd_struct(k.n_jobs)
        gr, grads = _grad_targets(model, ctx.heads, ctx.job_heads)
        _lib.check(lib.tir_primary_backward(C.byref(f), k.jobs, k.n_jobs, k.kind, _lib.dptr(k.rays),
                                            _lib.dptr(k.li, torch.int32), k.rays.shape[0], C.byref(w), C.byref(b),
                                            float(model.fixed_fresnel), ctx.bg, C.byref(_ray_maps(gs)), _ptr(g_acc),
                                            _ptr(g_la), _ptr(g_lr), C.byref(gr), _lib.stream_ptr()),
                   "tir_primary_backward")
        if k.kind == 1:
            _lib.launch_count -= 1          # no derived-normal scatter
        k.ws.busy = False
        return (None,) * 8 + grads


class _PrimaryRadiance(torch.autograd.Function):
    """TensorBase.forward with is_relight=False (training's warm-up phase) around tir_primary_march / _app_list /
    _radiance (9 launches) and tir_primary_radiance_backward (6 launches) -> (rgb_map, depth_map, acc_map)."""

    @staticmethod
    def forward(ctx, model, rays, light_idx, is_train, n_samples, bg_flag, jitter, *params):
        lib, f, w, _, keep, jobs, _, _, li, ws = _forward_common(ctx, model, rays, light_idx, is_train, n_samples,
                                                                 jitter, HEADS[:1], "_tir_radiance_ws")
        n_rays, dev = rays.shape[0], rays.device
        rgb, depth = torch.empty(n_rays, 3, device=dev), torch.empty(n_rays, device=dev)
        _lib.check(lib.tir_primary_radiance(C.byref(f), jobs, _lib.dptr(rays), _lib.dptr(li, torch.int32), n_rays,
                                            C.byref(w), int(bool(bg_flag)), _lib.dptr(rgb), _lib.dptr(depth),
                                            _lib.stream_ptr()), "tir_primary_radiance")
        ctx.keep = _RadianceKeep(keep, jobs, li, rays, ws, jitter, int(bool(bg_flag)))
        return rgb, depth, ws.t["acc"].clone()

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_acc):
        k, model = ctx.keep, ctx.model
        lib = _lib.load()
        f = ops.device_field(model).refresh(model)
        g_rgb, g_depth, g_acc = _f32(g_rgb), _f32(g_depth), _f32(g_acc)
        w, b = k.ws.work_struct(None, 1, True), k.ws.bwd_struct(1)
        gr, grads = _grad_targets(model, ctx.heads, ctx.job_heads)
        _lib.check(lib.tir_primary_radiance_backward(C.byref(f), k.jobs, _lib.dptr(k.rays),
                                                     _lib.dptr(k.li, torch.int32), k.rays.shape[0], C.byref(w),
                                                     C.byref(b), k.bg, _ptr(g_rgb), _ptr(g_depth), _ptr(g_acc),
                                                     C.byref(gr), _lib.stream_ptr()), "tir_primary_radiance_backward")
        k.ws.busy = False
        return (None,) * 7 + grads


def supported(model) -> bool:
    return (getattr(model, "shadingMode", None) == "MLP_Fea" and model.normals_kind in NORMALS
            and int(model.app_dim) == 27 and not model.__dict__.get("_tir_modular", False))


def _host_draws(model, n_rays, dev, white_bg, is_train):
    """Host-side draws in the reference's order: per-ray jitter on the CPU (tensorBase:714-718), then the background
    coin, which white_bg short-circuits (tensorBase:979 / :1004) -> (jitter or None, background flag)."""
    jitter = None
    if is_train:
        st = model.__dict__.get("_tir_static")
        jitter = st["jitter"] if st is not None else torch.rand(n_rays, 1).to(dev)
    return jitter, white_bg or (is_train and bool(torch.rand((1,)) < 0.5))


def _forward(model, rays_chunk, white_bg, is_train, slots, run):
    """TensorBase.forward's 12-tuple with the outputs of ``run(rays, background flag, jitter)`` (a node's apply) at
    ``slots``, the rest None.  An empty batch runs no node: its maps are empty and its losses NaN, as torch.mean over
    zero rays is in the reference."""
    rays = rays_chunk.float().contiguous()
    n_rays, dev = rays.shape[0], rays.device
    if n_rays == 0:
        outs = [torch.full((), float("nan"), device=dev) if k >= len(_MAP_SHAPES) else
                torch.zeros((0,) + _MAP_SHAPES[k], device=dev, dtype=torch.bool if k == 9 else None) for k in slots]
    else:
        jitter, bg = _host_draws(model, n_rays, dev, white_bg, is_train)
        outs = run(rays, bg, jitter)
    ret = [None] * 12
    for k, t in zip(slots, outs):
        ret[k] = t
    return tuple(ret)


def forward_relight(model, rays_chunk, light_idx, white_bg=True, is_train=False, N_samples=-1):
    """-> the 12-tuple of TensorBase.forward (is_relight=True)."""
    return _forward(model, rays_chunk, white_bg, is_train, range(12), lambda rays, bg, jitter: _PrimaryRelight.apply(
        model, rays, light_idx, white_bg, is_train, N_samples, bg, jitter, *_params(model, HEADS)))


def forward_radiance(model, rays_chunk, light_idx, white_bg=True, is_train=False, N_samples=-1):
    """-> the 12-tuple of TensorBase.forward (is_relight=False): rgb_map, depth_map, acc_map, the rest None."""
    return _forward(model, rays_chunk, white_bg, is_train, (0, 1, 6), lambda rays, bg, jitter: _PrimaryRadiance.apply(
        model, rays, light_idx, is_train, N_samples, bg, jitter, *_params(model, HEADS[:1])))
