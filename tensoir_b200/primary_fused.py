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

import torch

from . import _lib, ops
from .device_field import mlp_struct

HEAD_RGB, HEAD_BRDF, HEAD_BRDF_JITTER, HEAD_NORMAL = 0, 1, 2, 3
NORMALS = {"derived_plus_predicted": 0, "purely_predicted": 1, "purely_derived": 2}
MAXH = _lib.MAX_HEADS


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


def _jobs(model, keep):
    """(TirHeadJob array, n_jobs, module name of every job)."""
    kind = NORMALS[model.normals_kind]
    has_light = getattr(model, "light_line", None) is not None
    spec = [("renderModule", HEAD_RGB, 0, 0, 1 if has_light else 0, 0),
            ("renderModule_brdf", HEAD_BRDF, 0, 1, 2 if has_light else 0, 0),
            ("renderModule_brdf", HEAD_BRDF_JITTER, 1, 1, 2 if has_light else 0, 0)]
    if kind != 2:
        spec.append(("renderModule_normal", HEAD_NORMAL, 0, 1, 2 if has_light else 0, 1))
    arr = (TirHeadJob * len(spec))()
    for j, (head, role, ps, x_in, lm, act) in enumerate(spec):
        arr[j].mlp = mlp_struct(model, head, keep, light="index" if has_light else "none")
        arr[j].point_set, arr[j].x_in, arr[j].light_mode, arr[j].act, arr[j].role = ps, x_in, lm, act, role
    return arr, len(spec), [s[0] for s in spec], kind


def _cl_zeros(p):
    """Zeroed gradient buffer in the kernels' channel-last layout + its view in the parameter's shape."""
    _, Cc, H, W = p.shape
    buf = torch.zeros((H, W, Cc), device=p.device, dtype=torch.float32)
    return buf, buf.permute(2, 0, 1).unsqueeze(0)


def _workspace(model, key, dev, need, point_sets=2):
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


def _vm_grad_buffers(model):
    """Gradient buffers of the VM factors (17-31 M floats), in the order density planes, density lines, app planes, app
    lines -> (buffers the kernels accumulate into, what autograd gets for each factor).  When a parameter already HAS
    a dense channel-last .grad (kept zeroed in place by tensoir_b200.optim.FusedAdam, or the views of a dp.GradBucket)
    the kernels accumulate straight into it and autograd gets None for that input: no 70 MB allocation + memset +
    AccumulateGrad pass per step.  Otherwise a zeroed buffer in the kernels' layout is returned the usual way."""
    vm = list(model.density_plane) + list(model.density_line) + list(model.app_plane) + list(model.app_line)
    bufs, views = [], []
    for p in vm:
        g = p.grad
        if (g is not None and g.dtype == torch.float32 and g.shape == p.shape and p.shape[0] == 1
                and all(a == b for a, b, n in zip(g.stride(), p.stride(), p.shape) if n > 1)
                and p.is_contiguous(memory_format=torch.channels_last)
                and model.__dict__.get("_tir_grad_inplace", True)):
            bufs.append(g)
            views.append(None)
        else:
            b_, v_ = _cl_zeros(p)
            bufs.append(b_)
            views.append(v_)
    return bufs, views


def _set_vm_grads(gr, bufs):
    for k in range(3):
        gr.dplane[k], gr.dline[k] = bufs[k].data_ptr(), bufs[3 + k].data_ptr()
        gr.aplane[k], gr.aline[k] = bufs[6 + k].data_ptr(), bufs[9 + k].data_ptr()


def _grad_target(p, inplace):
    """(buffer the kernels accumulate into, what autograd gets): the parameter's own .grad when it is a plain fp32
    tensor of the same layout (then autograd gets None: no zero-fill, no AccumulateGrad add), else zeros."""
    g = p.grad
    if inplace and g is not None and g.dtype == torch.float32 and g.shape == p.shape and g.is_contiguous() \
            and p.is_contiguous():
        return g, None
    z = torch.zeros_like(p)
    return z, z


class _PrimaryRelight(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, rays, light_idx, white_bg, is_train, n_samples, bg_flag, jitter, *params):
        lib = _lib.load()
        cd = lib
        dev = rays.device
        st = model.__dict__.get("_tir_static")
        need = any(ctx.needs_input_grad)
        n_rays = rays.shape[0]
        df = ops.device_field(model)
        f = df.refresh(model, force=bool(is_train))
        keep = []
        jobs, n_jobs, heads, kind = _jobs(model, keep)
        cfg = ops.march_cfg(model, n_samples=n_samples, jitter=jitter, keep=keep)
        counters = model.__dict__.get("_tir_counters")
        cptr = None if counters is None else _lib.dptr(counters, torch.int64)
        ws = _workspace(model, "_tir_primary_ws", dev, need)
        li = light_idx.reshape(-1).to(torch.int32).contiguous()
        stream = _lib.stream_ptr()
        w, n_app = _march(cd, f, rays, cfg, ws, n_jobs, need, counters, st)
        # xyz noise of the smoothness term: randn_like(xyz_sampled[app_mask]) (tensorBase:937), drawn on the device in
        # list order; the eager path draws exactly n_app rows like the reference
        draw = model.__dict__.get("_tir_randn_like")       # test hook: replay the oracle's stream / deterministic noise
        rows = ws.cap_app if st is not None else int(n_app)
        noise = torch.zeros(ws.cap_app, 3, device=dev)
        if rows > 0:
            x_a = ws.t["a_xn"][:rows]
            noise[:rows] = draw(x_a) if draw is not None else torch.randn_like(x_a)
        w.noise = noise.data_ptr()
        outs = [torch.empty(n_rays, 3, device=dev), torch.empty(n_rays, device=dev), torch.empty(n_rays, 3, device=dev),
                torch.empty(n_rays, 3, device=dev), torch.empty(n_rays, 1, device=dev), torch.empty(n_rays, 3, device=dev),
                torch.empty(n_rays, 1, device=dev), torch.empty(n_rays, 1, device=dev)]
        maps = _lib.TirRayMaps()
        for k, t in zip(("rgb", "depth", "normal", "albedo", "rough", "fresnel", "nd", "no"), outs):
            setattr(maps, k, t.data_ptr())
        mask = torch.empty(n_rays, dtype=torch.bool, device=dev)
        losses = torch.empty(2, device=dev)
        _lib.check(cd.tir_primary_heads(C.byref(f), jobs, n_jobs, kind, _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                        n_rays, C.byref(w), float(model.fixed_fresnel), int(bool(bg_flag)),
                                        C.byref(maps), _lib.dptr(mask, torch.bool), _lib.dptr(losses), cptr, stream),
                   "tir_primary_heads")
        if kind == 1:
            _lib.launch_count -= 1          # no derived-normal gather
        acc = ws.t["acc"].clone()
        ctx.model, ctx.need, ctx.heads = model, need, heads
        ctx.cfg_args = (white_bg, bool(bg_flag), n_samples, bool(is_train))
        ctx.keep = (keep, jobs, n_jobs, kind, cfg, noise, li, rays, ws, jitter)
        ctx.mark_non_differentiable(mask)
        rgb, depth, normal, albedo, rough, fresnel, nd, no = outs
        return rgb, depth, normal, albedo, rough, fresnel, acc, nd, no, mask, losses[0], losses[1]

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_normal, g_albedo, g_rough, g_fresnel, g_acc, g_nd, g_no, _g_mask, g_la, g_lr):
        model = ctx.model
        keep, jobs, n_jobs, kind, cfg, noise, li, rays, ws, jitter = ctx.keep
        lib = _lib.load()
        cd = lib
        df = ops.device_field(model)
        f = df.refresh(model)
        dev = rays.device
        n_rays = rays.shape[0]

        def c(t):
            return None if t is None else t.contiguous().float()
        gs = [c(t) for t in (g_rgb, g_depth, g_normal, g_albedo, g_rough, g_fresnel, g_nd, g_no)]
        gmaps = _lib.TirRayMaps()
        for k, t in zip(("rgb", "depth", "normal", "albedo", "rough", "fresnel", "nd", "no"), gs):
            setattr(gmaps, k, None if t is None else t.data_ptr())
        g_acc, g_la, g_lr = c(g_acc), (None if g_la is None else c(g_la.reshape(1))), (None if g_lr is None else
                                                                                       c(g_lr.reshape(1)))
        w = ws.work_struct(noise, n_jobs, True)
        b = ws.bwd_struct(n_jobs)
        gr = TirPrimaryGrads()
        bufs, views = _vm_grad_buffers(model)
        _set_vm_grads(gr, bufs)
        inplace = model.__dict__.get("_tir_grad_inplace", True)

        def target(p):
            return _grad_target(p, inplace)
        g_basis, r_basis = target(model.basis_mat.weight)
        gr.basis = g_basis.data_ptr()
        ll = getattr(model, "light_line", None)
        g_light, r_light = target(ll.weight) if ll is not None else (None, None)
        gr.light_line = None if g_light is None else g_light.data_ptr()
        mod_grads = {}
        for j, head in enumerate(ctx.heads):
            if head not in mod_grads:
                m = getattr(model, head).mlp
                mod_grads[head] = [target(t) for t in (m[0].weight, m[0].bias, m[2].weight, m[2].bias, m[4].weight,
                                                       m[4].bias)]
            g = mod_grads[head]
            gr.w0[j], gr.b0[j], gr.w1[j], gr.b1[j], gr.w2[j], gr.b2[j] = [t[0].data_ptr() for t in g]
        white_bg, bg_flag, n_samples, is_train = ctx.cfg_args
        _lib.check(cd.tir_primary_backward(C.byref(f), jobs, n_jobs, kind, _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                           n_rays, C.byref(w), C.byref(b), float(model.fixed_fresnel), int(bg_flag),
                                           C.byref(gmaps), None if g_acc is None else _lib.dptr(g_acc),
                                           None if g_la is None else _lib.dptr(g_la),
                                           None if g_lr is None else _lib.dptr(g_lr), C.byref(gr), _lib.stream_ptr()),
                   "tir_primary_backward")
        if kind == 1:
            _lib.launch_count -= 1          # no derived-normal scatter
        ws.busy = False
        # gradients in the order of `params` (see forward_relight): VM factors, basis, [light_line], 3 x 6 MLP tensors
        out = list(views) + [r_basis] + ([r_light] if ll is not None else [])
        for head in ("renderModule", "renderModule_brdf", "renderModule_normal"):
            out += [t[1] for t in mod_grads[head]] if head in mod_grads else [None] * 6
        return (None, None, None, None, None, None, None, None, *out)


def supported(model) -> bool:
    return (getattr(model, "shadingMode", None) == "MLP_Fea" and model.normals_kind in NORMALS
            and int(model.app_dim) == 27 and not model.__dict__.get("_tir_modular", False))


def forward_relight(model, rays_chunk, light_idx, white_bg=True, is_train=False, N_samples=-1):
    """-> the 12-tuple of TensorBase.forward (is_relight=True)."""
    rays = rays_chunk.float().contiguous()
    n_rays = rays.shape[0]
    dev = rays.device
    if n_rays == 0:        # torch.mean over zero rays is NaN in the reference; keep that contract on the empty batch
        z3, z1, z = torch.zeros(0, 3, device=dev), torch.zeros(0, 1, device=dev), torch.zeros(0, device=dev)
        nan = torch.full((), float("nan"), device=dev)
        return (z3, z, z3.clone(), z3.clone(), z1, z3.clone(), z.clone(), z1.clone(), z1.clone(), z > 0.5, nan,
                nan.clone())
    jitter, bg = _host_draws(model, n_rays, dev, white_bg, is_train)
    params = _params(model, ("renderModule", "renderModule_brdf", "renderModule_normal"))
    return _PrimaryRelight.apply(model, rays, light_idx, white_bg, is_train, N_samples, bg, jitter, *params)


def _host_draws(model, n_rays, dev, white_bg, is_train):
    """Host-side draws in the reference's order: per-ray jitter on the CPU (tensorBase:714-718), then the background
    coin, which white_bg short-circuits (tensorBase:979 / :1004) -> (jitter or None, background flag)."""
    jitter = None
    if is_train:
        st = model.__dict__.get("_tir_static")
        jitter = st["jitter"] if st is not None else torch.rand(n_rays, 1).to(dev)
    return jitter, white_bg or (is_train and bool(torch.rand((1,)) < 0.5))


def _params(model, heads):
    """Autograd inputs of a primary node: VM factors, basis, [light_line], 6 tensors per head."""
    params = list(model.density_plane) + list(model.density_line) + list(model.app_plane) + list(model.app_line)
    params.append(model.basis_mat.weight)
    ll = getattr(model, "light_line", None)
    if ll is not None:
        params.append(ll.weight)
    for head in heads:
        m = getattr(model, head).mlp
        params += [m[0].weight, m[0].bias, m[2].weight, m[2].bias, m[4].weight, m[4].bias]
    return params


# ---- radiance-only primary (is_relight=False): training's warm-up phase -------------------------------------------------
def _radiance_job(model, keep):
    """The one head of the radiance branch: renderModule on the view direction, light_line[light_idx] if the model has
    one (tensorBase:930-946, is_relight=False)."""
    has_light = getattr(model, "light_line", None) is not None
    job = TirHeadJob()
    job.mlp = mlp_struct(model, "renderModule", keep, light="index" if has_light else "none")
    job.point_set, job.x_in, job.light_mode, job.act, job.role = 0, 0, 1 if has_light else 0, 0, HEAD_RGB
    return job


class _PrimaryRadiance(torch.autograd.Function):
    """TensorBase.forward with is_relight=False around tir_primary_march / _app_list / _radiance (9 launches) and
    tir_primary_radiance_backward (6 launches) -> (rgb_map, depth_map, acc_map)."""

    @staticmethod
    def forward(ctx, model, rays, light_idx, is_train, n_samples, bg_flag, jitter, *params):
        lib = _lib.load()
        dev = rays.device
        need = any(ctx.needs_input_grad)
        n_rays = rays.shape[0]
        f = ops.device_field(model).refresh(model, force=bool(is_train))
        keep = []
        job = _radiance_job(model, keep)
        cfg = ops.march_cfg(model, n_samples=n_samples, jitter=jitter, keep=keep)
        ws = _workspace(model, "_tir_radiance_ws", dev, need, point_sets=1)
        w, _ = _march(lib, f, rays, cfg, ws, 1, need, model.__dict__.get("_tir_counters"),
                      model.__dict__.get("_tir_static"))
        li = light_idx.reshape(-1).to(torch.int32).contiguous()
        rgb, depth = torch.empty(n_rays, 3, device=dev), torch.empty(n_rays, device=dev)
        _lib.check(lib.tir_primary_radiance(C.byref(f), C.byref(job), _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                            n_rays, C.byref(w), int(bool(bg_flag)), _lib.dptr(rgb), _lib.dptr(depth),
                                            _lib.stream_ptr()), "tir_primary_radiance")
        acc = ws.t["acc"].clone()
        ctx.model = model
        ctx.keep = (keep, job, li, rays, ws, jitter, int(bool(bg_flag)))
        return rgb, depth, acc

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_acc):
        model = ctx.model
        keep, job, li, rays, ws, jitter, bg = ctx.keep
        lib = _lib.load()
        f = ops.device_field(model).refresh(model)

        def c(t):
            return None if t is None else t.contiguous().float()
        g_rgb, g_depth, g_acc = c(g_rgb), c(g_depth), c(g_acc)
        w = ws.work_struct(None, 1, True)
        b = ws.bwd_struct(1)
        gr = TirPrimaryGrads()
        bufs, views = _vm_grad_buffers(model)
        _set_vm_grads(gr, bufs)
        inplace = model.__dict__.get("_tir_grad_inplace", True)
        g_basis, r_basis = _grad_target(model.basis_mat.weight, inplace)
        gr.basis = g_basis.data_ptr()
        ll = getattr(model, "light_line", None)
        g_light, r_light = _grad_target(ll.weight, inplace) if ll is not None else (None, None)
        gr.light_line = None if g_light is None else g_light.data_ptr()
        m = model.renderModule.mlp
        mg = [_grad_target(t, inplace) for t in (m[0].weight, m[0].bias, m[2].weight, m[2].bias, m[4].weight,
                                                  m[4].bias)]
        gr.w0[0], gr.b0[0], gr.w1[0], gr.b1[0], gr.w2[0], gr.b2[0] = [t[0].data_ptr() for t in mg]

        def ptr(t):
            return None if t is None else _lib.dptr(t)
        _lib.check(lib.tir_primary_radiance_backward(C.byref(f), C.byref(job), _lib.dptr(rays),
                                                     _lib.dptr(li, torch.int32), rays.shape[0], C.byref(w), C.byref(b),
                                                     bg, ptr(g_rgb), ptr(g_depth), ptr(g_acc), C.byref(gr),
                                                     _lib.stream_ptr()), "tir_primary_radiance_backward")
        ws.busy = False
        # gradients in the order of `params` (see forward_radiance): VM factors, basis, [light_line], renderModule
        out = list(views) + [r_basis] + ([r_light] if ll is not None else []) + [t[1] for t in mg]
        return (None,) * 7 + tuple(out)


def forward_radiance(model, rays_chunk, light_idx, white_bg=True, is_train=False, N_samples=-1):
    """-> the 12-tuple of TensorBase.forward (is_relight=False): rgb_map, depth_map, acc_map, the rest None."""
    rays = rays_chunk.float().contiguous()
    n_rays = rays.shape[0]
    dev = rays.device
    if n_rays == 0:
        z = torch.zeros(0, device=dev)
        rgb, depth, acc = torch.zeros(0, 3, device=dev), z, z.clone()
    else:
        jitter, bg = _host_draws(model, n_rays, dev, white_bg, is_train)
        params = _params(model, ("renderModule",))
        rgb, depth, acc = _PrimaryRadiance.apply(model, rays, light_idx, is_train, N_samples, bg, jitter, *params)
    return rgb, depth, None, None, None, None, acc, None, None, None, None, None
