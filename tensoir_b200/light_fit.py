"""Estimate the lighting of photographs: fit environment maps to posed views of a checkpoint whose geometry and
materials are held fixed (the inverse-lighting half of inverse rendering).

relight() (tensoir_b200.relighting) shades a surface hit under an H_e x W_e lat-long map with an estimator whose
expectation is, per colour channel c,

    sum_k T[c, i, k] L[k, c],   T[c, i, k] = (albedo*rescale/pi + GGX)_c * vis_k * cos_k * dOmega_k

over the map's K = H_e*W_e texels, dOmega_k = pdf / pdf_return = 2 pi^2 sin(theta_k) / K of Environment_Light's own
tables.  With the model fixed, T does not depend on the light, so one transport per view serves every light of a
dataset, and fitting a map to photographs is, per channel and light, the convex problem

    minimise 1/2 |T_c L - y_c|^2 + 1/2 lam_s |D L|^2 + 1/2 lam_r |L|^2   subject to L >= 0

with y the photographs' linear values and D the lat-long neighbour differences (wrapping in longitude).  The transport
is written by the tir_transport kernels (csrc/tir_transport.cu) around the unchanged density march; the normal
equations are accumulated in fp64 (G_c = sum T_c^T T_c, B_c = sum T_c^T Y_c) and solved by accelerated projected
gradient on the device.

The model is relight()'s: direct light only, with shadows.  Interreflections in real photographs are not modelled and
end up in the fitted map; what the surfaces never see (texels below every fitted point's horizon, or always shadowed)
is not constrained by the data and is filled in by the smoothness term.
"""
from __future__ import annotations

import json
import math
import os
import types

import numpy as np
import torch

from . import _lib
from . import relighting as R

FIT_RES = (16, 32)
PIXELS_PER_VIEW = 65536
# Regularisers relative to trace(G_c) / K, and the solver's stopping rule, chosen on the exact round trip of
# tests/test_light_fit_gpu.py (a sky gradient plus a sun lobe, 8-bit photos of 8 views of the lego scene, 16x32 map).
# Measured on an H100: smooth 0, 1e-4, 1e-3, 1e-2, 1e-1 gave held-out PSNR 58.65, 58.70, 58.61, 56.34, 49.73 dB and a
# mean per-texel error of 0.052, 0.045, 0.041, 0.061, 0.089 (mean |L*| 0.33); 1e-3 recovers the map best and converges
# within the iteration cap (5424 steps), while smaller weights do not.  The ridge only keeps unseen texels bounded.
SMOOTH = 1e-3
RIDGE = 1e-6
MAX_ITERS = 10000
TOL = 1e-6
SATURATED = 254.5 / 255    # a photo channel at or above this code was clipped by the camera: it only bounds L below
SEED = 20211202
UNOBSERVED = 1e-3          # a texel whose Gram diagonal is below this fraction of the largest one is reported unseen


# ---- arguments ---------------------------------------------------------------------------------------------------

def check_res(H_e, W_e):
    if not (isinstance(H_e, int) and isinstance(W_e, int) and W_e == 2 * H_e and 4 <= H_e <= 32):
        raise ValueError(f"fit resolution must be H x 2H with 4 <= H <= 32, got {H_e}x{W_e}")
    return H_e, W_e


def parse_res(spec):
    """'16x32' -> (16, 32)."""
    try:
        h, w = (int(x) for x in str(spec).lower().split("x"))
    except ValueError:
        raise ValueError(f"fit resolution must look like 16x32, got {spec!r}") from None
    return check_res(h, w)


def parse_views(spec, n_views):
    """View indices of ``spec``: a comma list ('0,3,7'), a slice 'a:b:step' (any part may be empty) or 'none'.
    Raises ValueError for a malformed spec, an index outside [0, n_views) or a repeated index."""
    s = str(spec).strip()
    if s.lower() == "none" or s == "":
        return []
    try:
        if ":" in s:
            parts = s.split(":")
            if len(parts) > 3:
                raise ValueError
            a, b, c = (parts + [""] * 3)[:3]
            step = int(c) if c else 1
            if step <= 0:
                raise ValueError
            start, stop = int(a) if a else 0, int(b) if b else n_views
            if start < 0 or stop < 0:
                raise ValueError
            idx = list(range(start, min(stop, n_views), step))
        else:
            idx = [int(x) for x in s.split(",")]
    except ValueError:
        raise ValueError(f"views must be 'i,j,...', 'a:b:step' or 'none', got {spec!r}") from None
    bad = [i for i in idx if not 0 <= i < n_views]
    if bad:
        raise ValueError(f"view index {bad[0]} outside [0, {n_views})")
    if len(set(idx)) != len(idx):
        raise ValueError(f"repeated view index in {spec!r}")
    return idx


# ---- tables and colour ---------------------------------------------------------------------------------------------

def texel_tables(H_e=FIT_RES[0], W_e=FIT_RES[1], device="cpu"):
    """Per texel of an H_e x W_e lat-long map, in Environment_Light's order: unit directions ``dirs`` [K, 3] (the bits
    of Environment_Light.hdr_dir) and solid angles ``dOmega`` [K] = 2 pi^2 sin(theta) / K (pdf / pdf_return of any
    positive map), fp32.  A map fitted on these texels and given to relight() is shaded under these directions."""
    from .relight import latlong_tables
    check_res(H_e, W_e)
    sin_t, dirs = latlong_tables(H_e, W_e)
    domega = (sin_t * (2 * np.pi * np.pi / (H_e * W_e))).view(-1, 1).expand(H_e, W_e).reshape(-1)
    return dirs.reshape(-1, 3).contiguous().to(device), domega.contiguous().to(device)


def srgb_to_linear(y):
    """The inverse of relight()'s tone map (tir::tone: clamp, then sRGB with the 1e-6 offset) on [0, 1], in fp64."""
    y = torch.as_tensor(y).double().clamp(0.0, 1.0)
    return torch.where(y <= 12.92 * 0.0031308, y / 12.92, ((y + 0.055) / 1.055) ** 2.4 - 1e-6).clamp(min=0.0)


def linear_to_srgb(x):
    """tir::tone in fp64."""
    t = torch.as_tensor(x).double().clamp(0.0, 1.0)
    return torch.where(t <= 0.0031308, t * 12.92, 1.055 * (t + 1e-6) ** (1 / 2.4) - 0.055)


# ---- transport -------------------------------------------------------------------------------------------------------

def transport_sample(grid, rays, depth, normal, acc, acc_mask_threshold):
    """tir_transport_sample on contiguous fp32 device tensors -> (pos [n, K], list_o, list_d) with the list cut to its
    length, which is the one host read of the chunk."""
    lib = _lib.load()
    dirs, _ = grid
    n, K = int(rays.shape[0]), int(dirs.shape[0])
    pos = torch.empty(n, K, dtype=torch.int32, device=rays.device)
    list_o, list_d = R.append_list(
        n * K, rays.device, "transport visibility list", None,
        lambda *tail: _lib.check(lib.tir_transport_sample(
            _lib.dptr(dirs), K, _lib.dptr(rays), _lib.dptr(depth), _lib.dptr(normal), _lib.dptr(acc), n,
            float(acc_mask_threshold), _lib.dptr(pos, torch.int32), *tail, _lib.stream_ptr()), "tir_transport_sample"))
    return pos, list_o, list_d


def transport_build(grid, rays, normal, albedo, rough, fresnel, acc, acc_mask_threshold, rescale_value, pos, vis,
                    vis_equation):
    """tir_transport_build -> T [3, n, K] fp32 on the device."""
    lib = _lib.load()
    dirs, domega = grid
    n, K = int(rays.shape[0]), int(dirs.shape[0])
    dev = rays.device
    T = torch.empty(3, n, K, device=dev)
    resc = R.rescale3(rescale_value, dev)
    _lib.check(lib.tir_transport_build(_lib.dptr(dirs), _lib.dptr(domega), K, _lib.dptr(rays), _lib.dptr(normal),
                                       _lib.dptr(albedo), _lib.dptr(rough), int(rough.shape[1]), _lib.dptr(fresnel),
                                       _lib.dptr(acc), n, float(acc_mask_threshold), _lib.dptr(resc),
                                       _lib.dptr(pos, torch.int32), _lib.dptr(vis), R.vis_kind(vis_equation),
                                       _lib.dptr(T), _lib.stream_ptr()),
               "tir_transport_build")
    return T


@torch.no_grad()
def transport_chunk(tensoIR, rays, maps, rescale_value, grid, acc_mask_threshold=0.5, vis_equation='nerv'):
    """The transport T [3, n, K] of one chunk of primary rays to the texels of ``grid`` = texel_tables(...) on the
    device.  ``maps`` = (depth, normal, albedo, roughness [n,1] or [n,3], fresnel, acc), the tuple relight_chunk_fused
    takes.  Rows with acc <= acc_mask_threshold are 0."""
    R.vis_kind(vis_equation)
    if int(rays.shape[0]) == 0:
        return torch.zeros(3, 0, int(grid[0].shape[0]), device=rays.device)
    rays, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(rays, maps)
    pos, list_o, list_d = transport_sample(grid, rays, depth, normal, acc, acc_mask_threshold)
    vis = R.march_list(tensoIR, list_o, list_d, vis_equation)
    return transport_build(grid, rays, normal, albedo, rough, fresnel, acc, acc_mask_threshold, rescale_value, pos,
                           vis, vis_equation)


# ---- normal equations and the solve ----------------------------------------------------------------------------------

class Normals:
    """The normal equations of the fit, fp64 on the device: per channel c, G[c] = sum T_c^T T_c [K, K] and, per light
    l, B[c, :, l] = sum T_c^T y_c,l, plus yy[c, l] = sum y^2 (for the residual) and the pixel counts.  The Gram matrix
    is shared by every light, so a pixel channel enters only when it is usable under all of them."""

    def __init__(self, K, n_lights, device):
        self.K, self.L = int(K), int(n_lights)
        self.G = torch.zeros(3, K, K, dtype=torch.float64, device=device)
        self.B = torch.zeros(3, K, n_lights, dtype=torch.float64, device=device)
        self.yy = torch.zeros(3, n_lights, dtype=torch.float64, device=device)
        self.used = [0, 0, 0]           # pixel channels that entered, per channel
        self.saturated = 0              # hit pixel channels left out because some photo clipped them
        self.missed = 0                 # sampled pixels the model does not hit (acc <= threshold)

    def add(self, T, y, use):
        """T [3, n, K] fp32, y [L, n, 3] linear targets, use [n, 3] bool: the pixel channels that enter."""
        for c in range(3):
            rows = use[:, c].nonzero().reshape(-1)
            Tc = T[c].index_select(0, rows).double()
            self.G[c] += Tc.T @ Tc
            yc = y[:, :, c].index_select(1, rows).double()
            for l in range(self.L):                 # one product per light: a fit's maps do not depend on its company
                self.B[c, :, l] += Tc.T @ yc[l]
                self.yy[c, l] += yc[l] @ yc[l]
            self.used[c] += int(rows.numel())

    def residual_rms(self, X):
        """Root mean square of T L - y over the pixel channels that entered, per light, from the normal equations.
        X [L, K, 3]."""
        out = []
        for l in range(self.L):
            ss = 0.0
            for c in range(3):
                x = X[l, :, c].double()
                ss += float(x @ (self.G[c] @ x) - 2 * (x @ self.B[c, :, l]) + self.yy[c, l])
            out.append(math.sqrt(max(ss, 0.0) / max(sum(self.used), 1)))
        return out

    def unobserved(self):
        d = torch.diagonal(self.G, dim1=1, dim2=2).sum(0)
        top = float(d.max()) if d.numel() else 0.0
        return int((d < UNOBSERVED * top).sum()) if top > 0 else self.K


def difference_operator(H_e, W_e, device="cpu"):
    """D [(2 H_e - 1) W_e, K] fp64: L[h, w+1] - L[h, w] for every texel (w wrapping) and L[h+1, w] - L[h, w] between
    rows."""
    K = H_e * W_e
    idx = torch.arange(K).view(H_e, W_e)
    a = torch.cat([idx.roll(-1, 1).reshape(-1), idx[1:].reshape(-1)])
    b = torch.cat([idx.reshape(-1), idx[:-1].reshape(-1)])
    D = torch.zeros(a.numel(), K, dtype=torch.float64)
    r = torch.arange(a.numel())
    D[r, a] += 1.0
    D[r, b] -= 1.0
    return D.to(device)


def system(G, H_e, W_e, smooth=SMOOTH, ridge=RIDGE):
    """Q [3, K, K] = G_c + s_c (smooth D^T D + ridge I), s_c = trace(G_c) / K: the Hessian of the objective."""
    K = G.shape[-1]
    D = difference_operator(H_e, W_e, G.device)
    s = torch.diagonal(G, dim1=1, dim2=2).sum(-1) / K
    reg = float(smooth) * (D.T @ D) + float(ridge) * torch.eye(K, dtype=torch.float64, device=G.device)
    return G + s.view(3, 1, 1) * reg


@torch.no_grad()
def solve(G, B, H_e, W_e, smooth=SMOOTH, ridge=RIDGE, max_iters=MAX_ITERS, tol=TOL):
    """Minimise 1/2 x^T Q_c x - B_c^T x over x >= 0 for every channel c and light (column of B) with Q = system(G):
    accelerated projected gradient (FISTA, step 1 / largest eigenvalue of Q_c, momentum restarted per channel when it
    points uphill), from x = 0, until the largest relative change of a step over the channels falls below ``tol`` or
    after ``max_iters`` steps.  Every light is solved on its own, so a light's map does not depend on which others are
    fitted with it; for given G and B the result is deterministic.
    G [3, K, K], B [3, K, L] fp64 -> (X [L, K, 3] fp64, [{"iterations", "change"} per light])."""
    G, B = G.double(), B.double()
    K, L = G.shape[-1], B.shape[-1]
    Q = system(G, H_e, W_e, smooth, ridge)
    top = torch.linalg.eigvalsh(Q)[:, -1]
    step = torch.where(top > 0, 1.0 / top.clamp(min=1e-300), torch.ones_like(top)).view(3, 1, 1)
    X = torch.zeros(L, K, 3, dtype=torch.float64, device=G.device)
    info = []
    for l in range(L):
        b = B[:, :, l:l + 1]
        x = torch.zeros(3, K, 1, dtype=torch.float64, device=G.device)
        y, t = x, torch.ones(3, 1, 1, dtype=torch.float64, device=G.device)
        it, change = 0, 0.0
        for it in range(1, int(max_iters) + 1):
            x_new = (y - step * (torch.bmm(Q, y) - b)).clamp(min=0.0)
            dx = x_new - x
            rel = dx.norm(dim=(1, 2)) / x_new.norm(dim=(1, 2)).clamp(min=1e-300)
            uphill = ((y - x_new) * dx).sum(dim=(1, 2), keepdim=True) > 0
            t_new = (1 + torch.sqrt(1 + 4 * t * t)) / 2
            y = torch.where(uphill, x_new, x_new + ((t - 1) / t_new) * dx)
            t = torch.where(uphill, torch.ones_like(t), t_new)
            x = x_new
            change = float(rel.max())
            if change < tol:
                break
        X[l] = x[:, :, 0].T
        info.append({"iterations": it, "change": change})
    return X, info


def objective(G, B, X, H_e, W_e, smooth=SMOOTH, ridge=RIDGE):
    """1/2 x^T Q x - B^T x summed over channels, per light (X [L, K, 3]); add 1/2 |y|^2 for the least-squares value."""
    Q = system(G.double(), H_e, W_e, smooth, ridge)
    return [sum(float(0.5 * X[l, :, c] @ (Q[c] @ X[l, :, c]) - B[c, :, l] @ X[l, :, c]) for c in range(3))
            for l in range(X.shape[0])]


# ---- the fit -----------------------------------------------------------------------------------------------------------

def _opt(args, name, default):
    v = getattr(args, name, None)
    return default if v is None else v


def usable(y, hit):
    """The pixel channels that enter the fit, [n, 3] bool: hit by the model and below SATURATED in the photo of every
    light (y [L, n, 3] sRGB).  One Gram matrix serves all lights only if they all see the same pixel channels."""
    return hit[:, None] & (y < SATURATED).all(0)


def _sample_pixels(mask, count, gen):
    """``count`` pixel indices inside ``mask`` [H*W] bool, drawn without replacement, in raster order."""
    inside = mask.nonzero().reshape(-1)
    if inside.numel() > count:
        inside = inside[torch.randperm(inside.numel(), generator=gen)[:count]].sort().values
    return inside


def _fit_chunks(tensoIR, dataset, views, grid, rescale, opt, device):
    """Per chunk of the sampled pixels of the fit views: (T, y_srgb [L, n, 3], use [n, 3], hit [n]).  The pixel draw
    is seeded, so two passes see the same pixels."""
    gen = torch.Generator().manual_seed(int(opt["seed"]))
    L = len(dataset.light_names)
    for idx in views:
        item = dataset[idx]
        rays_v = item['rays'].squeeze(0)
        n_pix = rays_v.shape[0]
        mask = item['rgbs_mask'].squeeze(0).reshape(-1).bool()
        pix = _sample_pixels(mask, int(opt["pixels_per_view"]), gen)
        photos = item['rgbs'].squeeze(0).reshape(L, n_pix, 3)
        for s in range(0, pix.numel(), int(opt["batch_size"])):
            p = pix[s:s + int(opt["batch_size"])]
            rays = rays_v.index_select(0, p).to(device)
            li = torch.zeros(p.numel(), 1, dtype=torch.int32, device=device)
            _, depth, normal, albedo, rough, fresnel, acc, *_ = tensoIR(rays, li, is_train=False, white_bg=True,
                                                                        ndc_ray=False, N_samples=-1)
            T = transport_chunk(tensoIR, rays, (depth, normal, albedo, rough, fresnel, acc), rescale, grid,
                                opt["acc_mask_threshold"], opt["vis_equation"])
            y = photos.index_select(1, p).to(device).double()
            hit = acc.detach().reshape(-1) > opt["acc_mask_threshold"]
            yield T, y, usable(y, hit), hit


class _Views:
    """``dataset`` restricted to some views and some of its lights, in relight()'s item contract."""

    def __init__(self, dataset, views, lights):
        self.base, self.views = dataset, list(views)
        self.keep = [list(dataset.light_names).index(n) for n in lights]
        self.light_names = list(lights)
        self.img_wh, self.near_far, self.split = dataset.img_wh, dataset.near_far, dataset.split

    def __len__(self):
        return len(self.views)

    def __getitem__(self, i):
        item = dict(self.base[self.views[i]])
        W, H = self.img_wh
        rgbs = item['rgbs'].squeeze(0).reshape(len(self.base.light_names), H * W, 3)
        item['rgbs'] = rgbs[self.keep]
        return item


@torch.no_grad()
def fit_lights(dataset, args, tensoIR=None):
    """Fit one environment map per light of ``dataset`` to its photographs.  ``dataset`` follows relight()'s item
    contract (rays, rgbs [L, H*W, 3] sRGB in [0, 1], rgbs_mask, albedo, light_names, split).  ``args`` needs ckpt (when
    ``tensoIR`` is None), out and batch_size, and may carry fit_views / eval_views (lists or parse_views specs;
    defaults '0::10' and '5::10'), fit_res ('16x32' or (H, W)), pixels_per_view, smooth, ridge, seed,
    acc_mask_threshold, vis_equation and geo_buffer_path (where relight() of the evaluation views writes; default
    {out}/eval).
    Writes {out}/{light}.hdr (linear radiance at the fit resolution) for every map with positive total intensity and
    {out}/fit_report.json; with evaluation views, relight()'s files under geo_buffer_path for them under the fitted
    maps, shaded with the fit's own rescale ratio.  -> (the report as written, {light: fitted map [H_e, W_e, 3] fp32
    numpy}, before the .hdr's RGBE rounding)."""
    from .evaluation import compute_rescale_ratio
    from .relight import write_hdr
    if tensoIR is None:
        tensoIR = R._load_model(args, torch.device("cuda"))
        if tensoIR is None:
            return None, None
    device = tensoIR.device if hasattr(tensoIR, "device") else torch.device("cuda")
    names = list(dataset.light_names)
    res = _opt(args, "fit_res", FIT_RES)
    H_e, W_e = parse_res(res) if isinstance(res, str) else check_res(*res)
    views = {}
    for k, default in (("fit_views", "0::10"), ("eval_views", "5::10")):
        v = _opt(args, k, default)
        views[k] = parse_views(v, len(dataset)) if isinstance(v, str) else parse_views(",".join(map(str, v)) or "none",
                                                                                         len(dataset))
    if not views["fit_views"]:
        raise ValueError("no views to fit")
    opt = dict(pixels_per_view=int(_opt(args, "pixels_per_view", PIXELS_PER_VIEW)), batch_size=int(args.batch_size),
               seed=int(_opt(args, "seed", SEED)),
               acc_mask_threshold=float(_opt(args, "acc_mask_threshold", R.SCRIPT_DEFAULTS["acc_mask_threshold"])),
               vis_equation=_opt(args, "vis_equation", R.SCRIPT_DEFAULTS["vis_equation"]))
    R.vis_kind(opt["vis_equation"])
    smooth, ridge = float(_opt(args, "smooth", SMOOTH)), float(_opt(args, "ridge", RIDGE))
    if smooth < 0 or ridge < 0:
        raise ValueError(f"smooth and ridge must be >= 0, got {smooth}, {ridge}")
    out = args.out
    os.makedirs(out, exist_ok=True)

    grid = texel_tables(H_e, W_e, device)
    _, rescale = compute_rescale_ratio(tensoIR, dataset)
    rescale = rescale.to(device)
    K, L = H_e * W_e, len(names)
    ne = Normals(K, L, device)
    for T, y, use, hit in _fit_chunks(tensoIR, dataset, views["fit_views"], grid, rescale, opt, device):
        ne.add(T, srgb_to_linear(y), use)
        ne.missed += int((~hit).sum())
        ne.saturated += int((hit[:, None] & ~use).sum())
    X, info = solve(ne.G, ne.B, H_e, W_e, smooth, ridge)
    maps = X.float()

    # second pass over the same pixels: the fitted maps' sRGB error on the pixel channels that entered the fit
    se = torch.zeros(L, dtype=torch.float64, device=device)
    for T, y, use, _ in _fit_chunks(tensoIR, dataset, views["fit_views"], grid, rescale, opt, device):
        pred = torch.einsum('cnk,lkc->lnc', T.double(), X)
        err = (linear_to_srgb(pred) - y) ** 2
        se += (err * use[None]).sum(dim=(1, 2))
    n_used = max(sum(ne.used), 1)
    rms = ne.residual_rms(X)
    unseen = ne.unobserved()
    report = {"fit_res": [H_e, W_e], "texels": K, "fit_views": views["fit_views"], "eval_views": views["eval_views"],
              "pixels_per_view": opt["pixels_per_view"], "smooth": smooth, "ridge": ridge,
              "rescale": [float(v) for v in rescale.reshape(-1).tolist()], "lights": {}}
    written = []
    for l, name in enumerate(names):
        total = float(maps[l].sum())
        mse = float(se[l]) / n_used
        entry = {"views": len(views["fit_views"]), "pixels_used": sum(ne.used), "pixels_excluded": ne.saturated,
                 "pixels_missed": ne.missed, "residual_rms_linear": rms[l],
                 "psnr_srgb": -10.0 * math.log10(mse) if mse > 0 else float("inf"), "unobserved_texels": unseen,
                 "iterations": info[l]["iterations"], "final_change": info[l]["change"], "written": total > 0}
        if total > 0:
            write_hdr(os.path.join(out, f"{name}.hdr"), maps[l].reshape(H_e, W_e, 3).cpu().numpy())
            written.append(name)
        else:
            entry["reason"] = "the fitted map has zero total intensity and cannot be importance-sampled"
            print(f"fit_lights: {name}: {entry['reason']}; not written")
        report["lights"][name] = entry
    with open(os.path.join(out, "fit_report.json"), "w") as f:
        json.dump(report, f, indent=1)

    if views["eval_views"] and written:
        ev = types.SimpleNamespace(**vars(args))
        ev.hdrdir = out
        ev.geo_buffer_path = getattr(args, "geo_buffer_path", None) or os.path.join(out, "eval")
        R.relight(_Views(dataset, views["eval_views"], written), ev, tensoIR, rescale_value=rescale)
    return report, {name: maps[l].reshape(H_e, W_e, 3).cpu().numpy() for l, name in enumerate(names)}
