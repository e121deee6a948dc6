"""Tensor-level wrappers of the C-ABI entry points (one per hot-path kernel).

Every wrapper takes a TensorVMSplit-like ``model`` (parameters in the reference layout), keeps its
DeviceField shadow fresh, allocates outputs/scratch with torch, and launches on the current stream.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from .device_field import DeviceField, mlp_struct


def device_field(model) -> DeviceField:
    df = model.__dict__.get("_tir_device_field")
    if df is None:
        df = DeviceField()
        model.__dict__["_tir_device_field"] = df
    return df


def new_counters(device) -> torch.Tensor:
    return torch.zeros(_lib.CNT_SLOTS, dtype=torch.int64, device=device)


def counters_dict(counters: torch.Tensor) -> dict:
    c = counters.tolist()
    return {"mask": c[_lib.CNT_MASK], "density": c[_lib.CNT_DENSITY], "app": c[_lib.CNT_APP],
            "rays": c[_lib.CNT_RAYS], "overflow": c[_lib.CNT_OVERFLOW]}


def _f32c(t):
    return t.detach().to(torch.float32).contiguous()


def _i32c(t):
    return None if t is None else t.detach().reshape(-1).to(torch.int32).contiguous()


def march_cfg(model, *, table: Optional[torch.Tensor] = None, n_samples: int = -1,
              jitter: Optional[torch.Tensor] = None, keep: list):
    cfg = _lib.TirMarchCfg()
    cfg.flags = _lib.MARCH_CELL_BRICKS          # DeviceField packs the occupancy bricks behind the cell bytes
    if table is not None:
        zt = _f32c(table.reshape(-1))
        keep.append(zt)
        cfg.sampling, cfg.n_samples, cfg.z_table = _lib.SAMPLE_TABLE, zt.numel(), zt.data_ptr()
        cfg.step, cfg.near, cfg.far, cfg.jitter = 0.0, 0.0, 0.0, None
    else:
        cfg.sampling = _lib.SAMPLE_STEP
        cfg.n_samples = int(n_samples if n_samples > 0 else model.nSamples)
        cfg.step = model._host_geom["step"]
        cfg.near, cfg.far = float(model.near_far[0]), float(model.near_far[1])
        cfg.z_table = None
        if jitter is not None:
            j = _f32c(jitter.reshape(-1))
            keep.append(j)
            cfg.jitter = j.data_ptr()
        else:
            cfg.jitter = None
    return cfg


def equal_z_table(n_sample, near, far, device):
    """z_vals of sample_ray_equally (relight_utils.py:716-717), computed with the same torch ops."""
    t = torch.linspace(0., 1., n_sample, device=device)
    return near * (1. - t) + far * t


def density_points(model, xn):
    """compute_densityfeature + feature2density on normalised points -> (feature, sigma)."""
    lib = _lib.load()
    f = device_field(model).refresh(model)
    xn = _f32c(xn.reshape(-1, 3))
    n = xn.shape[0]
    feat = torch.empty(n, device=xn.device)
    sig = torch.empty(n, device=xn.device)
    _lib.check(lib.tir_density_points(C.byref(f), _lib.dptr(xn), n, _lib.dptr(feat), _lib.dptr(sig),
                                      _lib.stream_ptr()), "tir_density_points")
    return feat, sig


def alpha_mask_points(model, xyz):
    """alphaMask.sample_alpha(xyz) > 0 -> bool [n]."""
    lib = _lib.load()
    f = device_field(model).refresh(model)
    xyz = _f32c(xyz.reshape(-1, 3))
    n = xyz.shape[0]
    out = torch.empty(n, device=xyz.device, dtype=torch.uint8)
    _lib.check(lib.tir_alpha_mask_points(C.byref(f), _lib.dptr(xyz), n, _lib.dptr(out, torch.uint8),
                                         _lib.stream_ptr()), "tir_alpha_mask_points")
    return out.bool()


def march_density(model, rays_o, rays_d, *, table=None, n_samples=-1, jitter=None, counters=None):
    """-> (t_last, acc, depth)."""
    lib = _lib.load()
    f = device_field(model).refresh(model)
    keep = []
    cfg = march_cfg(model, table=table, n_samples=n_samples, jitter=jitter, keep=keep)
    ro, rd = _f32c(rays_o.reshape(-1, 3)), _f32c(rays_d.reshape(-1, 3))
    if lean_counters(model):
        cfg.flags |= _lib.MARCH_LEAN_COUNTERS
    n = ro.shape[0]
    t_last = torch.ones(n, device=ro.device)
    acc = torch.zeros(n, device=ro.device)
    depth = torch.zeros(n, device=ro.device)
    _lib.check(lib.tir_march_density(C.byref(f), _lib.dptr(ro), _lib.dptr(rd), n, C.byref(cfg), _lib.dptr(t_last),
                                     _lib.dptr(acc), _lib.dptr(depth),
                                     None if counters is None else _lib.dptr(counters, torch.int64),
                                     _lib.stream_ptr()), "tir_march_density")
    return t_last, acc, depth


class SampleScratch:
    """Reusable app-sample list (TirAppSample[capacity]) + device counter."""

    def __init__(self, device, capacity):
        self.capacity = int(capacity)
        self.buf = torch.empty(self.capacity * _lib.APP_SAMPLE_BYTES, dtype=torch.uint8, device=device)
        self.count = torch.zeros(1, dtype=torch.int32, device=device)

    def samples(self):
        """Decode the filled part of the list -> dict of tensors (tests / diagnostics)."""
        n = min(int(self.count.item()), self.capacity)
        raw = self.buf[: n * _lib.APP_SAMPLE_BYTES].view(n, _lib.APP_SAMPLE_BYTES)
        f = raw[:, :16].contiguous().view(torch.float32).view(n, 4)
        i = raw[:, 16:].contiguous().view(torch.int32).view(n, 2)
        return {"xn": f[:, :3], "weight": f[:, 3], "ray": i[:, 0], "sample": i[:, 1]}


def _scratch(model, device, need):
    sc = model.__dict__.get("_tir_scratch")
    if sc is None or sc.capacity < need or sc.buf.device != device:
        sc = SampleScratch(device, need)
        model.__dict__["_tir_scratch"] = sc
    sc.count.zero_()
    return sc


def march_radiance(model, rays_o, rays_d, light_idx=None, *, table=None, n_samples=-1, jitter=None,
                   counters=None, capacity=None, head="renderModule"):
    """compute_radiance over explicit rays -> (t_last, acc, depth, rgb, scratch)."""
    lib = _lib.load()
    f = device_field(model).refresh(model)
    keep = []
    cfg = march_cfg(model, table=table, n_samples=n_samples, jitter=jitter, keep=keep)
    if lean_counters(model):
        cfg.flags |= _lib.MARCH_LEAN_COUNTERS
    mlp = mlp_struct(model, head, keep, light="index" if light_idx is not None else "none")
    ro, rd = _f32c(rays_o.reshape(-1, 3)), _f32c(rays_d.reshape(-1, 3))
    li = _i32c(light_idx)
    n = ro.shape[0]
    dev = ro.device
    t_last = torch.ones(n, device=dev)
    acc = torch.zeros(n, device=dev)
    depth = torch.zeros(n, device=dev)
    rgb = torch.zeros(n, 3, device=dev)
    cap = capacity if capacity is not None else max(1 << 16, min(n * cfg.n_samples, 8 * n + (1 << 16)))
    sc = _scratch(model, dev, cap)
    _lib.check(lib.tir_march_radiance(C.byref(f), C.byref(mlp), _lib.dptr(ro), _lib.dptr(rd),
                                      None if li is None else _lib.dptr(li, torch.int32), n, C.byref(cfg),
                                      _lib.dptr(t_last), _lib.dptr(acc), _lib.dptr(depth), _lib.dptr(rgb),
                                      _lib.dptr(sc.buf, torch.uint8), _lib.dptr(sc.count, torch.int32), sc.capacity,
                                      None if counters is None else _lib.dptr(counters, torch.int64),
                                      _lib.stream_ptr()), "tir_march_radiance")
    return t_last, acc, depth, rgb, sc


def lean_counters(model) -> bool:
    """True when the model runs its marches in production mode (``model.__dict__['_tir_lean']``): the mask / density
    counters then count the queries actually made (include/tensoir_b200.h: TIR_MARCH_LEAN_COUNTERS)."""
    return bool(model.__dict__.get("_tir_lean", False))


def density_volume(model, f) -> "_lib.TirDensityVolume":
    """The density feature baked at the grid vertices the secondary march can read (tir_density_volume_extent /
    tir_density_volume_build), built from the factors ``f`` points at, on the current stream.  Callers build it on every
    march: it is never reused across calls, so it can never be older than the parameters.  The storage is sized to the
    whole grid and kept on the model, so its address is stable for CUDA-graph capture; it is replaced only when the grid
    changes."""
    lib = _lib.load()
    lo, n = (C.c_int32 * 3)(), (C.c_int32 * 3)()
    _lib.check(lib.tir_density_volume_extent(C.byref(f), lo, n), "tir_density_volume_extent")
    size = f.grid[0] * f.grid[1] * f.grid[2]
    dev = model.density_plane[0].device
    buf = model.__dict__.get("_tir_density_vol")
    if buf is None or buf.numel() != size or buf.device != dev:
        buf = torch.empty(size, device=dev)
        model.__dict__["_tir_density_vol"] = buf
    vol = _lib.TirDensityVolume()
    vol.data, vol.lo, vol.n = buf.data_ptr(), lo, n
    _lib.check(lib.tir_density_volume_build(C.byref(f), C.byref(vol), size, _lib.stream_ptr()),
               "tir_density_volume_build")
    return vol


def secondary_radiance(model, surf_xyz, normals, light_idx, dirs, *, n_sample=96, near=0.05, far=1.5,
                       counters=None, capacity=None):
    """Secondary shading of render_with_BRDF -> (vis [n_pts,n_dirs,1], indirect [n_pts,n_dirs,3], scratch)."""
    lib = _lib.load()
    f = device_field(model).refresh(model)
    keep = []
    dev = surf_xyz.device
    cfg = march_cfg(model, table=equal_z_table(n_sample, near, far, dev), keep=keep)
    if lean_counters(model):
        cfg.flags |= _lib.MARCH_LEAN_COUNTERS
    mlp = mlp_struct(model, "renderModule", keep, light="index")
    sx, nr, dr = _f32c(surf_xyz.reshape(-1, 3)), _f32c(normals.reshape(-1, 3)), _f32c(dirs.reshape(-1, 3))
    li = _i32c(light_idx)
    n_pts, n_dirs = sx.shape[0], dr.shape[0]
    vis = torch.zeros(n_pts, n_dirs, 1, device=dev)
    ind = torch.zeros(n_pts, n_dirs, 3, device=dev)
    if n_pts == 0:
        return vis, ind, None
    st = model.__dict__.get("_tir_static")
    per_slot = 4 if st is None else int(st.get("sec_per_slot", 4))
    cap = capacity if capacity is not None else max(1 << 16, per_slot * n_pts * n_dirs)
    vol = density_volume(model, f)
    while True:
        sc = _scratch(model, dev, cap)
        _lib.check(lib.tir_secondary_radiance_vol(C.byref(f), C.byref(mlp), _lib.dptr(sx), _lib.dptr(nr),
                                                  _lib.dptr(li, torch.int32), n_pts, _lib.dptr(dr), n_dirs,
                                                  C.byref(cfg), C.byref(vol), _lib.dptr(vis), _lib.dptr(ind),
                                                  _lib.dptr(sc.buf, torch.uint8), _lib.dptr(sc.count, torch.int32),
                                                  sc.capacity,
                                                  None if counters is None else _lib.dptr(counters, torch.int64),
                                                  _lib.stream_ptr()), "tir_secondary_radiance_vol")
        if st is not None:
            # shape-static mode (CUDA-graph capture): no host sync; the step's overflow flag turns an overflowed step
            # into a no-op that the host redoes with a larger scratch list (static_step.py)
            from .primary import note_count
            note_count(st, 3, sc.count[0], sc.capacity)
            break
        need = int(sc.count.item())        # the march counts every appearance sample, also those it could not store
        if need <= sc.capacity:
            break
        # the list was too short: samples were dropped -> redo with a list that fits (never silently lose samples)
        if counters is not None:
            raise _lib.TirError(f"secondary appearance list overflowed ({need} > {sc.capacity}) while counters are "
                                f"being accumulated; pass capacity >= {need}")
        cap = need + (need >> 3)
        vis.zero_()
        ind.zero_()
    return vis, ind, sc


def app_mlp_points(model, xn, x_in, light_idx=None, *, head="renderModule", light="index"):
    """renderModule*(compute_*feature(xn), x_in) on explicit points -> [n,out_dim]."""
    lib = _lib.load()
    f = device_field(model).refresh(model)
    keep = []
    mlp = mlp_struct(model, head, keep, light=light)
    act = 1 if head == "renderModule_normal" else 0
    xn, xi = _f32c(xn.reshape(-1, 3)), _f32c(x_in.reshape(-1, 3))
    li = _i32c(light_idx) if light == "index" else None
    n = xn.shape[0]
    out = torch.empty(n, mlp.out_dim, device=xn.device)
    _lib.check(lib.tir_app_mlp_points_save(C.byref(f), C.byref(mlp), _lib.dptr(xn), _lib.dptr(xi),
                                           None if li is None else _lib.dptr(li, torch.int32), n, act, _lib.dptr(out),
                                           None, None, None, None, _lib.stream_ptr()), "tir_app_mlp_points_save")
    return out


class SecondaryStages:
    """The two stages of tir_secondary_radiance_vol as separately launchable stages (bench / profiling):
    ``march()`` = density-volume build + cosine test + density march + compaction, ``mlp()`` = appearance gather + MLP
    on the list."""

    def __init__(self, model, surf_xyz, normals, light_idx, dirs, n_sample=96, near=0.05, far=1.5):
        self.model = model
        self.lib = _lib.load()
        self.f = device_field(model).refresh(model)
        self.keep = []
        dev = surf_xyz.device
        self.cfg = march_cfg(model, table=equal_z_table(n_sample, near, far, dev), keep=self.keep)
        if lean_counters(model):
            self.cfg.flags |= _lib.MARCH_LEAN_COUNTERS
        self.mlp_s = mlp_struct(model, "renderModule", self.keep, light="index")
        self.sx, self.nr, self.dr = _f32c(surf_xyz.reshape(-1, 3)), _f32c(normals.reshape(-1, 3)), _f32c(dirs.reshape(-1, 3))
        self.li = _i32c(light_idx)
        self.n_pts, self.n_dirs = self.sx.shape[0], self.dr.shape[0]
        self.vis = torch.zeros(self.n_pts, self.n_dirs, 1, device=dev)
        self.ind = torch.zeros(self.n_pts, self.n_dirs, 3, device=dev)
        self.sc = SampleScratch(dev, max(1 << 16, 4 * self.n_pts * self.n_dirs))
        self.counters = new_counters(dev)

    def march(self):
        self.sc.count.zero_()
        self.counters.zero_()
        vol = density_volume(self.model, self.f)
        _lib.check(self.lib.tir_secondary_march_vol(C.byref(self.f), _lib.dptr(self.sx), _lib.dptr(self.nr),
                                                    self.n_pts, _lib.dptr(self.dr), self.n_dirs, C.byref(self.cfg),
                                                    C.byref(vol), _lib.dptr(self.vis),
                                                    _lib.dptr(self.sc.buf, torch.uint8),
                                                    _lib.dptr(self.sc.count, torch.int32), self.sc.capacity,
                                                    _lib.dptr(self.counters, torch.int64), _lib.stream_ptr()),
                   "tir_secondary_march_vol")

    def mlp(self):
        _lib.check(self.lib.tir_app_mlp(C.byref(self.f), C.byref(self.mlp_s), _lib.dptr(self.sc.buf, torch.uint8),
                                        _lib.dptr(self.sc.count, torch.int32), self.sc.capacity, _lib.dptr(self.dr),
                                        self.n_dirs, _lib.dptr(self.li, torch.int32), _lib.dptr(self.ind),
                                        _lib.stream_ptr()), "tir_app_mlp")


def generate_rays(c2w, view_idx, pix_idx, H=800, W=800, cam_angle_x=0.6911):
    """Rays [n,6] of (view, pixel) ids generated on the device (SURVEY.md 8 f4): the per-step host work of the train
    loop (fancy-indexing the all_rays table, train_tensoIR.py:239-242, and copying 24 B/ray) becomes an 8 B/ray id copy.
    c2w [n_views,4,4] on the device; pix = j*W + i."""
    import math
    lib = _lib.load()
    c2w = _f32c(c2w.reshape(-1, 4, 4))
    v, p = _i32c(view_idx), _i32c(pix_idx)
    n = v.shape[0]
    rays = torch.empty(n, 6, device=c2w.device)
    focal = 0.5 * W / math.tan(0.5 * cam_angle_x)
    _lib.check(lib.tir_generate_rays(_lib.dptr(c2w), _lib.dptr(v, torch.int32), _lib.dptr(p, torch.int32), n, H, W,
                                     float(focal), _lib.dptr(rays), _lib.stream_ptr()), "tir_generate_rays")
    return rays
