"""Relighting pass (scripts/relight_importance.py:30-340 + Environment_Light, models/relight_utils.py:110-205) as a
device-resident loop: inverse-CDF importance sampling of the environment map instead of ``torch.multinomial`` over
[bs, H*W] (2 M bins per pixel), visibility of every (surface point, sampled light) pair through the fused density
march (tir_march_density), GGX + Lambert, pdf-weighted mean, sRGB, compositing over the environment background.
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.nn.functional as F

from . import ops
from .relight_utils import GGX_specular, linear2srgb_torch, safe_l2_normalize


def read_hdr(path):
    """relight_utils.py:598-611 (cv2 Radiance .hdr reader, RGB order)."""
    import cv2
    with open(path, 'rb') as h:
        buffer_ = np.frombuffer(h.read(), np.uint8)
    bgr = cv2.imdecode(buffer_, cv2.IMREAD_UNCHANGED)
    return cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)


def write_hdr(path, rgb):
    """Write float [H,W,3] RGB radiance as a Radiance .hdr (RGBE, cv2) that read_hdr reads back to within RGBE precision:
    each channel to one mantissa step, 2^-8 of the power of two above the pixel's largest channel."""
    import cv2
    bgr = np.ascontiguousarray(np.asarray(rgb, dtype=np.float32)[..., ::-1])
    if not cv2.imwrite(path, bgr):
        raise OSError(f"could not write {path}")


def latlong_tables(H, W):
    """The texel tables of an H x W lat-long map as Environment_Light builds them, fp32 on the CPU: sin of the row
    centres' polar angle [H] and the unit direction of every texel [H, W, 3] (row 0 looks up, column 0 along -x)."""
    sin_t = torch.sin(torch.linspace(0 + 0.5 / H, np.pi - 0.5 / H, H))
    lat, lng = np.pi / H, 2 * np.pi / W
    phi, theta = torch.meshgrid([torch.linspace(np.pi / 2 - 0.5 * lat, -np.pi / 2 + 0.5 * lat, H),
                                 torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, W)], indexing='ij')
    dirs = torch.stack([torch.cos(theta) * torch.cos(phi), torch.sin(theta) * torch.cos(phi),
                        torch.sin(phi)], dim=-1).view(H, W, 3)
    return sin_t, dirs


class Environment_Light:
    """Same tables as the reference class (hdr_rgbs / hdr_pdf_sample / hdr_pdf_return / hdr_dir per light name);
    ``hdr_path`` may be a directory of .hdr files (reference behaviour) or a dict {name: [H,W,3] array}."""

    def __init__(self, hdr_path, device='cuda'):
        if isinstance(hdr_path, dict):
            maps = hdr_path
        else:
            maps = {f.split(".")[0]: read_hdr(os.path.join(hdr_path, f)) for f in sorted(os.listdir(hdr_path))
                    if f.endswith(".hdr")}
        self.device = device
        self.hdr_rgbs, self.hdr_pdf_sample, self.hdr_pdf_return, self.hdr_dir, self._cdf = {}, {}, {}, {}, {}
        for name, arr in maps.items():
            rgb = torch.as_tensor(np.asarray(arr)).float()
            inten = torch.sum(rgb, dim=2, keepdim=True)
            H, W, _ = inten.shape
            sin_t, dirs = latlong_tables(H, W)
            pdf = inten * sin_t.view(-1, 1, 1)
            pdf = pdf / torch.sum(pdf)
            pdf_ret = pdf * H * W / (2 * np.pi * np.pi * sin_t.view(-1, 1, 1))
            self.hdr_rgbs[name] = rgb.to(device)
            self.hdr_pdf_sample[name] = pdf.to(device)
            self.hdr_pdf_return[name] = pdf_ret.to(device)
            self.hdr_dir[name] = dirs.to(device)
            # inverse-CDF table (fp64 accumulation so that the last bin closes at 1)
            cdf = torch.cumsum(pdf.view(-1).double(), 0)
            self._cdf[name] = (cdf / cdf[-1]).to(device)

    @torch.no_grad()
    def sample_light(self, light_name, bs, num_samples, sample_type="importance", light_dir_idx=None):
        """relight_utils.py:150-188 -> (light_dir, light_rgb, light_pdf).  The reference draws
        ``torch.multinomial(pdf.expand(bs, H*W), num_samples, replacement=True)`` (O(bs*H*W)); sampling with replacement
        from a categorical is exactly inverse-CDF sampling, done here with one searchsorted over the H*W-entry CDF
        (O(bs*num_samples*log(H*W))).  Same distribution, different random stream; pass ``light_dir_idx`` to replay
        given indices."""
        if sample_type != "importance":
            raise NotImplementedError(sample_type)
        dev = self.hdr_rgbs[light_name].device
        if light_dir_idx is None:
            u = torch.rand(bs, num_samples, device=dev, dtype=torch.float64)
            cdf = self._cdf[light_name]
            light_dir_idx = torch.searchsorted(cdf, u, right=True).clamp_(max=cdf.numel() - 1)
        idx = light_dir_idx.reshape(-1)
        ld = self.hdr_dir[light_name].view(-1, 3).index_select(0, idx).view(bs, num_samples, 3)
        lr = self.hdr_rgbs[light_name].view(-1, 3).index_select(0, idx).view(bs, num_samples, 3)
        lp = self.hdr_pdf_return[light_name].view(-1).index_select(0, idx).view(bs, num_samples, 1)
        return ld, lr, lp

    def get_light(self, light_name, incident_dir):
        """relight_utils.py:193-205: bilinear background lookup."""
        env = self.hdr_rgbs[light_name].permute(2, 0, 1).unsqueeze(0)
        phi = torch.arccos(incident_dir[:, 2]).reshape(-1) - 1e-6
        theta = torch.atan2(incident_dir[:, 1], incident_dir[:, 0]).reshape(-1)
        qy = (phi / np.pi) * 2 - 1
        qx = -theta / np.pi
        grid = torch.stack((qx, qy)).permute(1, 0).unsqueeze(0).unsqueeze(0)
        return F.grid_sample(env, grid, align_corners=True).squeeze().permute(1, 0).reshape(-1, 3)


@torch.no_grad()
def relight_chunk(tensoIR, envir_light, light_name, rays, maps, rescale_value, light_dir_idx=None, num_samples=512,
                  acc_mask_threshold=0.5, vis_equation='nerv'):
    """Per-chunk body of relight() (relight_importance.py:99-181).  ``maps`` = (depth, normal, albedo, roughness,
    fresnel, acc) from ``tensoIR(rays, light_idx, is_train=False, ...)``.  -> (with_bg, without_bg) [n,3]."""
    depth, normal, albedo, rough, fresnel, acc = maps
    dev = rays.device
    mask = acc > acc_mask_threshold
    idx = torch.nonzero(mask).reshape(-1)
    rays_o, rays_d = rays[:, :3], rays[:, 3:]
    surf = (rays_o + depth.unsqueeze(-1) * rays_d).index_select(0, idx)
    m_n, m_a = normal.index_select(0, idx), albedo.index_select(0, idx)
    m_r, m_f = rough.index_select(0, idx), fresnel.index_select(0, idx)
    bs = idx.shape[0]
    surf2l, l_rgb, l_pdf = envir_light.sample_light(light_name, bs, num_samples, light_dir_idx=light_dir_idx)
    surf2c = safe_l2_normalize(-rays_d.index_select(0, idx), dim=-1)
    cosine = torch.einsum("ijk,ik->ij", surf2l, m_n)
    cmask = cosine > 1e-6
    vis = torch.zeros((bs, num_samples), device=dev)
    sel = torch.nonzero(cmask.reshape(-1)).reshape(-1)
    if sel.numel() > 0:
        pts = surf[:, None, :].expand(-1, num_samples, -1).reshape(-1, 3).index_select(0, sel)
        dirs = surf2l.reshape(-1, 3).index_select(0, sel)
        table = ops.equal_z_table(96, 0.05, 1.5, dev)
        t_last, acc_s, _ = ops.march_density(tensoIR, pts, dirs, table=table,
                                             counters=tensoIR.__dict__.get("_tir_counters"))
        vis.view(-1).index_copy_(0, sel, t_last if vis_equation == 'nerv' else 1 - acc_s)
    spec = GGX_specular(m_n, surf2c, surf2l, m_r, m_f)
    brdf = (m_a * rescale_value).unsqueeze(1).expand(-1, num_samples, -1) / np.pi + spec
    contrib = brdf * (vis.unsqueeze(-1) * l_rgb) * cosine[:, :, None] / l_pdf
    srgb = torch.clamp(torch.mean(contrib, dim=1), min=0.0, max=1.0)
    if srgb.shape[0] > 0:
        srgb = linear2srgb_torch(srgb)
    without_bg = torch.ones((rays.shape[0], 3), device=dev).index_copy_(0, idx, srgb)
    bg = linear2srgb_torch(torch.clamp(envir_light.get_light(light_name, rays_d), min=0.0, max=1.0))
    acc_t = torch.where(acc[..., None] <= 0.9, torch.zeros_like(acc[..., None]), acc[..., None])
    with_bg = acc_t * without_bg + (1.0 - acc_t) * bg
    return with_bg, without_bg


@torch.no_grad()
def relight_view(tensoIR, envir_light, light_names, frame_rays, light_rotation_idx=0, batch_size=4096,
                 rescale_value=1.0, num_samples=512, acc_mask_threshold=0.5, vis_equation='nerv'):
    """One test view of relight() (relight_importance.py:71-186): chunked primary march + one relight_chunk per
    environment map.  -> {name: (with_bg [H*W,3], without_bg [H*W,3])}, plus the primary maps."""
    dev = frame_rays.device
    out = {n: ([], []) for n in light_names}
    prim = []
    for s in range(0, frame_rays.shape[0], batch_size):
        rays = frame_rays[s:s + batch_size]
        li = torch.full((rays.shape[0], 1), light_rotation_idx, dtype=torch.int32, device=dev)
        rgb, depth, normal, albedo, rough, fresnel, acc, *_ = tensoIR(rays, li, is_train=False, white_bg=True,
                                                                      ndc_ray=False, N_samples=-1)
        prim.append((rgb, depth, normal, albedo, rough, acc))
        maps = (depth, normal, albedo, rough.repeat(1, 3) if rough.shape[-1] == 1 else rough, fresnel, acc)
        for n in light_names:
            w, wo = relight_chunk(tensoIR, envir_light, n, rays, maps, rescale_value, None, num_samples,
                                  acc_mask_threshold, vis_equation)
            out[n][0].append(w)
            out[n][1].append(wo)
    res = {n: (torch.cat(v[0]), torch.cat(v[1])) for n, v in out.items()}
    res["_primary"] = tuple(torch.cat([p[i] for p in prim]) for i in range(6))
    return res


@torch.no_grad()
def relight_views_sharded(tensoIR, envir_light, light_names, view_rays, *, gt=None, rank=None, world=None, **kw):
    """The test-view loop of relight() (relight_importance.py:63-71) sharded over ranks (SURVEY.md §8e: views are
    independent; no data-path collective).  ``view_rays(i)`` returns the [H*W, 6] rays of view ``i`` (or pass a
    sequence of ray tensors); ``gt`` optionally maps (view, light name) -> [H*W, 3] reference image for PSNR.
    -> (local {view: relight_view result}, metrics of ALL views {view: {name: psnr or mean}} on every rank)."""
    from .dp import gather_view_results, shard_views
    n_views = len(view_rays) if hasattr(view_rays, "__len__") else kw.pop("n_views")
    get = view_rays.__getitem__ if hasattr(view_rays, "__getitem__") else view_rays
    local, metrics = {}, {}
    for v in shard_views(n_views, rank, world):
        res = relight_view(tensoIR, envir_light, light_names, get(v), **kw)
        local[v] = res
        m = {}
        for n in light_names:
            img = res[n][0]
            if gt is not None:
                mse = torch.mean((img - gt(v, n).to(img.device)) ** 2)
                m[n] = float(-10.0 * torch.log10(mse.clamp_min(1e-20)))
            else:
                m[n] = float(img.mean())
        metrics[v] = m
    return local, gather_view_results(metrics)
