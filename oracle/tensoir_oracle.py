"""CPU oracle for the TensoIR volume-rendering hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in ``tensoir_b200/`` (the product) may import this
module; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs use it, and there only as the checker / the CPU baseline.

This is a *restatement* (not a copy) of the reference's PyTorch algorithm as plain
functions over an :class:`OracleField` record.  Every function cites the reference
``file:line`` (relative to the reference's root) that it follows, and keeps the reference's
operation order so that on CPU it reproduces the reference bit-for-bit.

Parity pinning: ``tests/golden/make_golden.py`` imports the real reference from
a checkout of it, runs it on small seeded inputs and stores
inputs + outputs under ``tests/golden/*.pt``; ``tests/test_oracle_golden.py`` replays the
oracle against those fixtures (bit-exact on CPU).  The reference ships no golden vectors of
its own (SURVEY.md §4), so those generated fixtures are the pin.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

MAT_MODE = ((0, 1), (0, 2), (1, 2))  # tensorBase_rotated_lights.py:398
VEC_MODE = (2, 1, 0)                 # tensorBase_rotated_lights.py:399


# ----------------------------------------------------------------------------------------
# field record
# ----------------------------------------------------------------------------------------
@dataclass
class Mlp:
    """Three Linear layers of MLPRender_Fea / MLPBRDF_PEandFeature
    (tensorBase_rotated_lights.py:122-146, :182-208)."""
    w0: torch.Tensor
    b0: torch.Tensor
    w1: torch.Tensor
    b1: torch.Tensor
    w2: torch.Tensor
    b2: torch.Tensor

    def params(self):
        return [self.w0, self.b0, self.w1, self.b1, self.w2, self.b2]


@dataclass
class OracleField:
    aabb: torch.Tensor                      # [2,3]
    grid_size: List[int]                    # [gx, gy, gz]
    density_plane: List[torch.Tensor]       # 3 x [1,Cd,G[m1],G[m0]]
    density_line: List[torch.Tensor]        # 3 x [1,Cd,G[v],1]
    app_plane: List[torch.Tensor]
    app_line: List[torch.Tensor]
    basis_w: torch.Tensor                   # [app_dim, sum(Ca)]
    mlp_rgb: Mlp
    light_line_w: Optional[torch.Tensor] = None   # [L, sum(Ca)]; None => tensoRF_init model
    mlp_brdf: Optional[Mlp] = None
    mlp_normal: Optional[Mlp] = None
    lgt_sgs: Optional[List[torch.Tensor]] = None  # rotated: [one tensor]; general: L tensors
    light_rotation: Optional[List[int]] = None    # rotated model only
    light_num: int = 1
    alpha_volume: Optional[torch.Tensor] = None   # [1,1,Z,Y,X] float
    alpha_aabb: Optional[torch.Tensor] = None
    density_shift: float = -10.0
    distance_scale: float = 25.0
    step_ratio: float = 0.5
    near_far: Tuple[float, float] = (2.0, 6.0)
    weight_thres: float = 1e-4
    fea2dense: str = "softplus"
    pos_pe: int = 2
    view_pe: int = 2
    fea_pe: int = 2
    envmap_h: int = 16
    envmap_w: int = 32
    fixed_fresnel: float = 0.04
    normals_kind: str = "derived_plus_predicted"
    counters: dict = field(default_factory=dict)

    # --- derived quantities: update_stepSize, tensorBase_rotated_lights.py:608-619
    def derived(self):
        aabb_size = self.aabb[1] - self.aabb[0]
        inv_aabb = 2.0 / aabb_size
        gs = torch.LongTensor(list(self.grid_size)).to(self.aabb.device)
        units = aabb_size / (gs - 1)
        step = torch.mean(units) * self.step_ratio
        diag = torch.sqrt(torch.sum(torch.square(aabb_size)))
        n_samples = int((diag / step).item()) + 1
        return aabb_size, inv_aabb, units, step, n_samples

    def count(self, key, n):
        self.counters[key] = self.counters.get(key, 0) + int(n)

    def parameters(self):
        ps = list(self.density_plane) + list(self.density_line) + list(self.app_plane) + list(self.app_line)
        ps += [self.basis_w] + self.mlp_rgb.params()
        if self.light_line_w is not None:
            ps.append(self.light_line_w)
        for m in (self.mlp_brdf, self.mlp_normal):
            if m is not None:
                ps += m.params()
        if self.lgt_sgs is not None:
            ps += list(self.lgt_sgs)
        return ps

    def to(self, device=None, dtype=None):
        """Move every tensor to ``device`` and/or cast it to ``dtype``.  The functions below create their
        intermediates in the default dtype, so a float64 field is evaluated under
        ``torch.set_default_dtype(torch.float64)``."""
        def mv(t):
            return None if t is None else t.to(device=device, dtype=dtype)
        for name in ("aabb", "basis_w", "light_line_w", "alpha_volume", "alpha_aabb"):
            setattr(self, name, mv(getattr(self, name)))
        for name in ("density_plane", "density_line", "app_plane", "app_line"):
            setattr(self, name, [mv(t) for t in getattr(self, name)])
        for name in ("mlp_rgb", "mlp_brdf", "mlp_normal"):
            m = getattr(self, name)
            if m is not None:
                setattr(self, name, Mlp(*[mv(t) for t in m.params()]))
        if self.lgt_sgs is not None:
            self.lgt_sgs = [mv(t) for t in self.lgt_sgs]
        return self


def _mlp_from_sd(sd, prefix):
    return Mlp(sd[f"{prefix}.mlp.0.weight"], sd[f"{prefix}.mlp.0.bias"],
               sd[f"{prefix}.mlp.2.weight"], sd[f"{prefix}.mlp.2.bias"],
               sd[f"{prefix}.mlp.4.weight"], sd[f"{prefix}.mlp.4.bias"])


def field_from_state_dict(sd, aabb, grid_size, *, kind="rotated", light_rotation=None, light_num=None,
                          lgt_sgs_list=None, alpha_volume=None, alpha_aabb=None, **consts) -> OracleField:
    """Build an OracleField from a reference-format state_dict (key names: SURVEY.md §8b,
    verified against tensoRF_rotated_lights.py:11-29)."""
    sd = {k: v.detach().clone() for k, v in sd.items()}
    f = OracleField(
        aabb=aabb.detach().clone().float(), grid_size=[int(g) for g in grid_size],
        density_plane=[sd[f"density_plane.{i}"] for i in range(3)],
        density_line=[sd[f"density_line.{i}"] for i in range(3)],
        app_plane=[sd[f"app_plane.{i}"] for i in range(3)],
        app_line=[sd[f"app_line.{i}"] for i in range(3)],
        basis_w=sd["basis_mat.weight"], mlp_rgb=_mlp_from_sd(sd, "renderModule"))
    if kind != "init":
        f.light_line_w = sd["light_line.weight"]
        f.mlp_brdf = _mlp_from_sd(sd, "renderModule_brdf")
        f.mlp_normal = _mlp_from_sd(sd, "renderModule_normal")
        f.light_num = int(f.light_line_w.shape[0]) if light_num is None else int(light_num)
        if kind == "rotated":
            f.lgt_sgs = [sd["lgtSGs"]]
            f.light_rotation = [int(r) for r in (light_rotation if light_rotation is not None else [0])]
        else:
            f.lgt_sgs = [t.detach().clone() for t in lgt_sgs_list]
            f.light_rotation = None
    if alpha_volume is not None:
        f.alpha_volume = alpha_volume.detach().clone().float().view(1, 1, *alpha_volume.shape[-3:])
        f.alpha_aabb = (alpha_aabb if alpha_aabb is not None else aabb).detach().clone().float()
    for k, v in consts.items():
        if not hasattr(f, k):
            raise KeyError(k)
        setattr(f, k, v)
    return f


# ----------------------------------------------------------------------------------------
# small pieces
# ----------------------------------------------------------------------------------------
def positional_encoding(positions, freqs):
    """tensorBase_rotated_lights.py:12-17 — index layout d*F+f, then [sin | cos]."""
    bands = (2 ** torch.arange(freqs).float()).to(positions.device)
    pts = (positions[..., None] * bands).reshape(positions.shape[:-1] + (freqs * positions.shape[-1],))
    return torch.cat([torch.sin(pts), torch.cos(pts)], dim=-1)


def raw2alpha(sigma, dist):
    """tensorBase_rotated_lights.py:21-28 (same code tensorBase_init.py:16-23)."""
    alpha = 1. - torch.exp(-sigma * dist)
    ones = torch.ones(alpha.shape[0], 1).to(alpha.device)
    T = torch.cumprod(torch.cat([ones, 1. - alpha + 1e-10], -1), -1)
    weights = alpha * T[:, :-1]
    return alpha, weights, T[:, -1:]


def safe_l2_normalize(x, dim=None, eps=1e-6):
    """dataLoader/ray_utils.py:278, relight_utils.py:13."""
    return F.normalize(x, p=2, dim=dim, eps=eps)


def linear2srgb(t):
    """relight_utils.py:489-515 (+ the clip of :518-533)."""
    if torch.min(t) < 0 or torch.max(t) > 1:
        t = torch.clamp(t, min=0, max=1)
    lin = t * 12.92
    nonlin = 1.055 * torch.pow(t + 1e-6, 1 / 2.4) - (1.055 - 1)
    return torch.where(t <= 0.0031308, lin, nonlin)


def normalize_coord(f: OracleField, xyz):
    """tensorBase_rotated_lights.py:640-641."""
    _, inv_aabb, _, _, _ = f.derived()
    return (xyz - f.aabb[0]) * inv_aabb - 1


def sample_alpha(f: OracleField, xyz):
    """AlphaGridMask.sample_alpha, tensorBase_rotated_lights.py:112-119."""
    inv = 1.0 / (f.alpha_aabb[1] - f.alpha_aabb[0]) * 2
    g = (xyz - f.alpha_aabb[0]) * inv - 1
    return F.grid_sample(f.alpha_volume, g.view(1, -1, 1, 1, 3), align_corners=True).view(-1)


def feature2density(f: OracleField, feat):
    """tensorBase_rotated_lights.py:813-817."""
    if f.fea2dense == "softplus":
        return F.softplus(feat + f.density_shift)
    return F.relu(feat)


# ----------------------------------------------------------------------------------------
# VM gathers
# ----------------------------------------------------------------------------------------
def _vm_coords(xyz):
    """Coordinate stacks of tensoRF_rotated_lights.py:98-100."""
    cp = torch.stack((xyz[..., MAT_MODE[0]], xyz[..., MAT_MODE[1]], xyz[..., MAT_MODE[2]])).detach().view(3, -1, 1, 2)
    cl = torch.stack((xyz[..., VEC_MODE[0]], xyz[..., VEC_MODE[1]], xyz[..., VEC_MODE[2]]))
    cl = torch.stack((torch.zeros_like(cl), cl), dim=-1).detach().view(3, -1, 1, 2)
    return cp, cl


def density_feature(f: OracleField, xyz):
    """TensorVMSplit.compute_densityfeature, tensoRF_rotated_lights.py:95-110."""
    cp, cl = _vm_coords(xyz)
    n = xyz.shape[0]
    out = torch.zeros((n,), device=xyz.device)
    for k in range(3):
        p = F.grid_sample(f.density_plane[k], cp[[k]], align_corners=True).view(-1, n)
        l = F.grid_sample(f.density_line[k], cl[[k]], align_corners=True).view(-1, n)
        out = out + torch.sum(p * l, dim=0)
    f.count("density", n)
    return out


def grid_sample_clamped(image, optical):
    """Twice-differentiable sampler of relight_utils.py:57-107: bilinear weights from the
    unclamped corner coordinates, corner *indices* clamped (extrapolates, no zero pad)."""
    N, C, IH, IW = image.shape
    _, H, W, _ = optical.shape
    ix = ((optical[..., 0] + 1) / 2) * (IW - 1)
    iy = ((optical[..., 1] + 1) / 2) * (IH - 1)
    with torch.no_grad():
        x0 = torch.floor(ix)
        y0 = torch.floor(iy)
        x1 = x0 + 1
        y1 = y0 + 1
    nw = (x1 - ix) * (y1 - iy)
    ne = (ix - x0) * (y1 - iy)
    sw = (x1 - ix) * (iy - y0)
    se = (ix - x0) * (iy - y0)
    with torch.no_grad():
        cx0 = torch.clamp(x0, 0, IW - 1)
        cx1 = torch.clamp(x1, 0, IW - 1)
        cy0 = torch.clamp(y0, 0, IH - 1)
        cy1 = torch.clamp(y1, 0, IH - 1)
    flat = image.contiguous().view(N, C, IH * IW)

    def tap(yy, xx):
        idx = (yy * IW + xx).long().view(N, 1, H * W).repeat(1, C, 1)
        return torch.gather(flat, 2, idx).view(N, C, H, W)

    return (tap(cy0, cx0) * nw.view(N, 1, H, W) + tap(cy0, cx1) * ne.view(N, 1, H, W) +
            tap(cy1, cx0) * sw.view(N, 1, H, W) + tap(cy1, cx1) * se.view(N, 1, H, W))


def density_feature_with_xyz_grad(f: OracleField, xyz):
    """compute_densityfeature_with_xyz_grad, tensoRF_rotated_lights.py:113-129 (no detach)."""
    cp = torch.stack((xyz[..., MAT_MODE[0]], xyz[..., MAT_MODE[1]], xyz[..., MAT_MODE[2]])).view(3, -1, 1, 2)
    cl = torch.stack((xyz[..., VEC_MODE[0]], xyz[..., VEC_MODE[1]], xyz[..., VEC_MODE[2]]))
    cl = torch.stack((torch.zeros_like(cl), cl), dim=-1).view(3, -1, 1, 2)
    n = xyz.shape[0]
    out = torch.zeros((n,), device=xyz.device)
    for k in range(3):
        p = grid_sample_clamped(f.density_plane[k], cp[[k]]).view(-1, n)
        l = grid_sample_clamped(f.density_line[k], cl[[k]]).view(-1, n)
        out = out + torch.sum(p * l, dim=0)
    return out


def _app_products(f: OracleField, xyz):
    """Shared first half of compute_{both,app,intrin}feature, tensoRF_rotated_lights.py:141-153."""
    cp, cl = _vm_coords(xyz)
    n = xyz.shape[0]
    ps, ls = [], []
    for k in range(3):
        ps.append(F.grid_sample(f.app_plane[k], cp[[k]], align_corners=True).view(-1, n))
        ls.append(F.grid_sample(f.app_line[k], cl[[k]], align_corners=True).view(-1, n))
    f.count("app", n)
    return torch.cat(ps), torch.cat(ls)


def _light_mean(f: OracleField, like):
    """mean over lights of light_line, tensoRF_rotated_lights.py:160-161."""
    idx = torch.arange(f.light_num).to(like.device, dtype=torch.int32)
    return torch.mean(F.embedding(idx, f.light_line_w), dim=0).unsqueeze(-1).expand_as(like)


def both_feature(f: OracleField, xyz, light_idx):
    """compute_bothfeature, tensoRF_rotated_lights.py:132-165 -> (radiance_feat, intrinsic_feat)."""
    p, l = _app_products(f, xyz)
    lc = F.embedding(light_idx.to(xyz.device), f.light_line_w).squeeze(1).permute(1, 0)
    rad = F.linear((p * l * lc).T, f.basis_w)
    intr = F.linear((p * l * _light_mean(f, lc)).T, f.basis_w)
    return rad, intr


def app_feature(f: OracleField, xyz, light_idx=None):
    """compute_appfeature, tensoRF_rotated_lights.py:197-224; with light_idx=None the
    light-free tensoRF_init.py:222-236 variant."""
    p, l = _app_products(f, xyz)
    if f.light_line_w is None or light_idx is None:
        return F.linear((p * l).T, f.basis_w)
    lc = F.embedding(light_idx.to(xyz.device), f.light_line_w).squeeze(1).permute(1, 0)
    return F.linear((p * l * lc).T, f.basis_w)


def intrin_feature(f: OracleField, xyz):
    """compute_intrinfeature, tensoRF_rotated_lights.py:167-195."""
    p, l = _app_products(f, xyz)
    return F.linear((p * l * _light_mean(f, p)).T, f.basis_w)


def _mlp(m: Mlp, x):
    h = F.relu(F.linear(x, m.w0, m.b0))
    h = F.relu(F.linear(h, m.w1, m.b1))
    return F.linear(h, m.w2, m.b2)


def mlp_render_fea(f: OracleField, m: Mlp, viewdirs, feats):
    """MLPRender_Fea.forward, tensorBase_rotated_lights.py:136-146:
    [feat, dir, PE(feat), PE(dir)] -> sigmoid."""
    x = [feats, viewdirs]
    if f.fea_pe > 0:
        x.append(positional_encoding(feats, f.fea_pe))
    if f.view_pe > 0:
        x.append(positional_encoding(viewdirs, f.view_pe))
    return torch.sigmoid(_mlp(m, torch.cat(x, dim=-1)))


def mlp_pe_and_feature(f: OracleField, m: Mlp, pts, feats, act):
    """MLPBRDF_PEandFeature.forward, tensorBase_rotated_lights.py:198-208:
    [feat, pts, PE(feat), PE(pts)] -> act."""
    x = [feats, pts]
    if f.fea_pe > 0:
        x.append(positional_encoding(feats, f.fea_pe))
    if f.pos_pe > 0:
        x.append(positional_encoding(pts, f.pos_pe))
    return act(_mlp(m, torch.cat(x, dim=-1)))


def derived_normals(f: OracleField, xyz):
    """compute_derived_normals, tensorBase_rotated_lights.py:839-856."""
    with torch.enable_grad():
        xyz.requires_grad_(True)
        sigma = feature2density(f, density_feature_with_xyz_grad(f, xyz))
        g = torch.autograd.grad(outputs=sigma, inputs=xyz, grad_outputs=torch.ones_like(sigma),
                                create_graph=True, retain_graph=True, only_inputs=True)[0]
        return (-safe_l2_normalize(g, dim=-1)).view(-1, 3)


def relative_smoothness(values, values_j):
    """compute_relative_smoothness_loss, tensorBase_rotated_lights.py:858-863."""
    base = torch.maximum(values, values_j).clip(min=1e-6)
    return torch.sum(((values - values_j) / base) ** 2, dim=-1, keepdim=True)


# ----------------------------------------------------------------------------------------
# ray sampling
# ----------------------------------------------------------------------------------------
def sample_ray(f: OracleField, rays_o, rays_d, is_train=True, n_samples=-1, jitter=None):
    """TensorBase.sample_ray, tensorBase_rotated_lights.py:705-724.  ``jitter`` ([N,1], CPU)
    replaces the reference's CPU ``torch.rand_like`` draw when given."""
    _, _, _, step, n_default = f.derived()
    n_samples = n_samples if n_samples > 0 else n_default
    near, far = f.near_far
    vec = torch.where(rays_d == 0, torch.full_like(rays_d, 1e-6), rays_d)
    rate_a = (f.aabb[1] - rays_o) / vec
    rate_b = (f.aabb[0] - rays_o) / vec
    t_min = torch.minimum(rate_a, rate_b).amax(-1).clamp(min=near, max=far)
    rng = torch.arange(n_samples)[None].float()
    if is_train:
        rng = rng.repeat(rays_d.shape[-2], 1)
        rng += (torch.rand_like(rng[:, [0]]) if jitter is None else jitter.cpu())
    z = t_min[..., None] + step * rng.to(rays_o.device)
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z[..., None]
    out = ((f.aabb[0] > pts) | (pts > f.aabb[1])).any(dim=-1)
    return pts, z, ~out


def sample_ray_equally(f: OracleField, rays_o, rays_d, n_sample, near, far):
    """relight_utils.py:707-722 (device taken from the inputs instead of the 'cuda' default)."""
    t = torch.linspace(0., 1., n_sample, device=rays_o.device)
    z = (near * (1. - t) + far * t).unsqueeze(0)
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z.view(1, -1, 1)
    out = ((f.aabb[0] > pts) | (pts > f.aabb[1])).any(dim=-1)
    return pts, z, ~out


def _refine_valid(f: OracleField, xyz, ray_valid):
    """alpha-mask refinement, tensorBase_rotated_lights.py:892-897."""
    if f.alpha_volume is None:
        return ray_valid
    f.count("mask", int(ray_valid.sum()))
    alphas = sample_alpha(f, xyz[ray_valid])
    invalid = ~ray_valid
    invalid[ray_valid] |= (~(alphas > 0))
    return ~invalid


# ----------------------------------------------------------------------------------------
# secondary marches
# ----------------------------------------------------------------------------------------
@torch.no_grad()
def compute_transmittance(f: OracleField, surf_pts, light_in_dir, n_sample=128, vis_near=0.1, vis_far=2.0):
    """relight_utils.py:657-705 -> (nerv_vis, nerfactor_vis)."""
    xyz, z, valid = sample_ray_equally(f, surf_pts, light_in_dir, n_sample, vis_near, vis_far)
    dists = torch.cat((z[:, 1:] - z[:, :-1], torch.zeros_like(z[:, :1])), dim=-1)
    valid = _refine_valid(f, xyz, valid)
    sigma = torch.zeros(xyz.shape[:-1], device=xyz.device)
    if valid.any():
        xyz = normalize_coord(f, xyz)
        sigma[valid] = feature2density(f, density_feature(f, xyz[valid]))
    _, weight, trans = raw2alpha(sigma, dists * f.distance_scale)
    return trans.squeeze(-1), 1 - torch.sum(weight, -1)


@torch.no_grad()
def compute_radiance(f: OracleField, surf_pts, light_in_dir, light_idx, n_sample=128, vis_near=0.05, vis_far=1.5,
                     return_aux=False):
    """relight_utils.py:777-834 -> (nerv_vis, nerfactor_vis, indirect_light)."""
    xyz, z, valid = sample_ray_equally(f, surf_pts, light_in_dir, n_sample, vis_near, vis_far)
    dists = torch.cat((z[:, 1:] - z[:, :-1], torch.zeros_like(z[:, :1])), dim=-1)
    light_idx = light_idx.view(-1, 1, 1).expand((*xyz.shape[:-1], 1))
    viewdirs = light_in_dir.view(-1, 1, 3).expand(xyz.shape)
    valid = _refine_valid(f, xyz, valid)
    sigma = torch.zeros(xyz.shape[:-1], device=xyz.device)
    indirect = torch.zeros((*xyz.shape[:2], 3), device=xyz.device)
    if valid.any():
        xyz = normalize_coord(f, xyz)
        sigma[valid] = feature2density(f, density_feature(f, xyz[valid]))
    _, weight, trans = raw2alpha(sigma, dists * f.distance_scale)
    app_mask = weight > f.weight_thres
    if app_mask.any():
        feat = app_feature(f, xyz[app_mask], light_idx[app_mask])
        indirect[app_mask] = mlp_render_fea(f, f.mlp_rgb, viewdirs[app_mask], feat)
    acc = torch.sum(weight, -1)
    out = (trans.squeeze(-1), 1 - acc, torch.sum(weight[..., None] * indirect, -2))
    if return_aux:
        return out + (valid, app_mask, weight)
    return out


@torch.no_grad()
def compute_secondary_shading_effects(f: OracleField, surface_pts, surf2light, light_idx, n_sample=96,
                                      vis_near=0.05, vis_far=1.5, chunk_size=15000):
    """relight_utils.py:344-399."""
    dev = surface_pts.device
    vis = torch.zeros((surface_pts.shape[0]), dtype=torch.float32).to(dev)
    ind = torch.zeros((surface_pts.shape[0], 3), dtype=torch.float32).to(dev)
    f.count("secondary_rays", surface_pts.shape[0])
    for idx in torch.split(torch.arange(surface_pts.shape[0]), chunk_size):
        v, _, i = compute_radiance(f, surface_pts[idx], surf2light[idx], light_idx[idx], n_sample, vis_near, vis_far)
        vis[idx] = v
        ind[idx] = i
    return vis.reshape(-1, 1), ind.reshape(-1, 3)


# ----------------------------------------------------------------------------------------
# lights + BRDF
# ----------------------------------------------------------------------------------------
def generate_envir_map_dir(envmap_h, envmap_w):
    """tensorBase_rotated_lights.py:435-453 (is_jittor=False)."""
    lat = np.pi / envmap_h
    lng = 2 * np.pi / envmap_w
    phi, theta = torch.meshgrid([torch.linspace(np.pi / 2 - 0.5 * lat, -np.pi / 2 + 0.5 * lat, envmap_h),
                                 torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, envmap_w)], indexing='ij')
    sin_phi = torch.sin(torch.pi / 2 - phi)
    weight = (4 * torch.pi * sin_phi / torch.sum(sin_phi)).to(torch.float32).reshape(-1)
    dirs = torch.stack([torch.cos(theta) * torch.cos(phi), torch.sin(theta) * torch.cos(phi),
                        torch.sin(phi)], dim=-1).view(-1, 3)
    return weight, dirs


def gen_light_incident_dirs(f: OracleField, method='fixed_envirmap', jitter=None):
    """tensorBase_rotated_lights.py:492-574 (fixed_envirmap / stratified_sampling /
    stratifed_sample_equal_areas).  ``jitter`` = (a, b) uniform [H,W] CPU tensors replacing the
    two ``torch.rand_like`` draws."""
    H, W = f.envmap_h, f.envmap_w
    if method == 'fixed_envirmap':
        return generate_envir_map_dir(H, W)[1].reshape(-1, 3)
    lng = 2 * np.pi / W
    if method == 'stratified_sampling':
        lat = np.pi / H
        phi_b, theta_b = torch.meshgrid([torch.linspace(np.pi / 2 - 0.5 * lat, -np.pi / 2 + 0.5 * lat, H),
                                         torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, W)], indexing='ij')
        ra = torch.rand_like(phi_b) if jitter is None else jitter[0]
        rb = torch.rand_like(theta_b) if jitter is None else jitter[1]
        phi, theta = phi_b + lat * (ra - 0.5), theta_b + lng * (rb - 0.5)
    elif method == 'stratifed_sample_equal_areas':
        sz = 2 / H
        s_b, theta_b = torch.meshgrid([torch.linspace(1 - 0.5 * sz, -1 + 0.5 * sz, H),
                                       torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, W)], indexing='ij')
        ra = torch.rand_like(s_b) if jitter is None else jitter[0]
        rb = torch.rand_like(theta_b) if jitter is None else jitter[1]
        phi, theta = torch.asin(s_b + sz * (ra - 0.5)), theta_b + lng * (rb - 0.5)
    else:
        raise NotImplementedError(method)
    return torch.stack([torch.cos(theta) * torch.cos(phi), torch.sin(theta) * torch.cos(phi),
                        torch.sin(phi)], dim=-1).reshape(-1, 3)


def render_envmap_sg(lgt_sgs, viewdirs):
    """tensorBase_rotated_lights.py:70-86."""
    viewdirs = viewdirs.to(lgt_sgs.device).unsqueeze(-2)
    dots = list(viewdirs.shape[:-2])
    M = lgt_sgs.shape[0]
    sg = lgt_sgs.view([1, ] * len(dots) + [M, 7]).expand(dots + [M, 7])
    lobes = sg[..., :3] / (torch.norm(sg[..., :3], dim=-1, keepdim=True))
    lam = torch.abs(sg[..., 3:4])
    mu = torch.abs(sg[..., -3:])
    rgb = mu * torch.exp(lam * (torch.sum(viewdirs * lobes, dim=-1, keepdim=True) - 1.))
    return torch.sum(rgb, dim=-2)


def light_rotation_matrices(light_rotation):
    """tensorBase_rotated_lights.py:478-488."""
    mats = []
    for r in light_rotation:
        a = torch.tensor(r / 180 * torch.pi).to(torch.float32)
        mats.append(torch.tensor([[torch.cos(a), -torch.sin(a), 0], [torch.sin(a), torch.cos(a), 0],
                                  [0, 0, 1]]).to(torch.float32))
    return torch.stack(mats, dim=0)


def get_light_rgbs(f: OracleField, dirs):
    """SG branch of get_light_rgbs: rotated tensorBase_rotated_lights.py:577-588; general
    tensorBase_general_multi_lights.py:568-582 -> [light_num, n, 3]."""
    dev = dirs.device
    if f.light_rotation is not None:
        d = dirs.reshape(1, -1, 3)
        rot = light_rotation_matrices(f.light_rotation).to(dev)
        d = torch.matmul(d, rot).reshape(-1, 3)
        return render_envmap_sg(f.lgt_sgs[0].to(dev), d).reshape(f.light_num, -1, 3)
    d = dirs.reshape(-1, 3)
    return torch.stack([render_envmap_sg(s.to(dev), d).reshape(-1, 3) for s in f.lgt_sgs], dim=0)


def ggx_specular(normal, pts2c, pts2l, roughness, fresnel):
    """GGX_specular, relight_utils.py:17-50."""
    L = F.normalize(pts2l, dim=-1)
    V = F.normalize(pts2c, dim=-1)
    H = F.normalize((L + V[:, None, :]) / 2.0, dim=-1)
    N = F.normalize(normal, dim=-1)
    NoV = torch.sum(V * N, dim=-1, keepdim=True)
    N = N * NoV.sign()
    NoL = torch.sum(N[:, None, :] * L, dim=-1, keepdim=True).clamp_(1e-6, 1)
    NoV = torch.sum(N * V, dim=-1, keepdim=True).clamp_(1e-6, 1)
    NoH = torch.sum(N[:, None, :] * H, dim=-1, keepdim=True).clamp_(1e-6, 1)
    VoH = torch.sum(V[:, None, :] * H, dim=-1, keepdim=True).clamp_(1e-6, 1)
    alpha = roughness * roughness
    alpha2 = alpha * alpha
    k = (alpha + 2 * roughness + 1.0) / 8.0
    FMi = ((-5.55473) * VoH - 6.98316) * VoH
    frac0 = fresnel[:, None, :] + (1 - fresnel[:, None, :]) * torch.pow(2.0, FMi)
    frac = frac0 * alpha2[:, None, :]
    nom0 = NoH * NoH * (alpha2[:, None, :] - 1) + 1
    nom1 = NoV * (1 - k) + k
    nom2 = NoL * (1 - k[:, None, :]) + k[:, None, :]
    nom = (4 * np.pi * nom0 * nom0 * nom1[:, None, :] * nom2).clamp_(1e-6, 4 * np.pi)
    return frac / nom


def render_with_brdf(f: OracleField, depth, normal, albedo, roughness3, fresnel, rays, light_idx,
                     sample_method='fixed_envirmap', chunk_size=15000, second_nsample=96, second_near=0.05,
                     second_far=1.5, light_jitter=None, use_linear2srgb=True):
    """render_with_BRDF, relight_utils.py:403-483."""
    dev = depth.device
    rays_o, rays_d = rays[..., :3], rays[..., 3:]
    surface_xyz = rays_o + depth.unsqueeze(-1) * rays_d
    area_w = generate_envir_map_dir(f.envmap_h, f.envmap_w)[0].to(dev)
    dirs = gen_light_incident_dirs(f, sample_method, light_jitter).to(dev)
    surf2l = dirs.reshape(1, -1, 3).repeat(surface_xyz.shape[0], 1, 1)
    surf2c = safe_l2_normalize(-rays_d, dim=-1)
    cosine = torch.clamp(torch.einsum("ijk,ik->ij", surf2l, normal), min=0.0)
    cmask = cosine > 1e-6
    vis = torch.zeros((*cmask.shape, 1), device=dev)
    ind = torch.zeros((*cmask.shape, 3), device=dev)
    vis[cmask], ind[cmask] = compute_secondary_shading_effects(
        f, surface_xyz.unsqueeze(1).expand(-1, surf2l.shape[1], -1)[cmask], surf2l[cmask],
        light_idx.view(-1, 1, 1).expand((*cmask.shape, 1))[cmask], second_nsample, second_near, second_far,
        chunk_size)
    nl = surf2l.shape[1]
    spec = ggx_specular(normal, surf2c, surf2l, roughness3, fresnel)
    brdf = albedo.unsqueeze(1).expand(-1, nl, -1) / np.pi + spec
    env = get_light_rgbs(f, dirs).to(dev)
    direct = torch.index_select(env, dim=0, index=light_idx.squeeze(-1)).to(dev)
    light = vis * direct + ind
    if sample_method == 'stratifed_sample_equal_areas':
        rgb = torch.mean(4 * torch.pi * brdf * light * cosine[:, :, None], dim=1)
    else:
        rgb = torch.sum(brdf * light * cosine[:, :, None] * area_w[None, :, None], dim=1)
    rgb = torch.clamp(rgb, min=0.0, max=1.0)
    if use_linear2srgb and rgb.shape[0] > 0:
        rgb = linear2srgb(rgb)
    return rgb


# ----------------------------------------------------------------------------------------
# primary march
# ----------------------------------------------------------------------------------------
def primary_forward(f: OracleField, rays, light_idx, white_bg=True, is_train=False, is_relight=True,
                    n_samples=-1, jitter=None, xyz_noise=None, bg_coin=None, return_aux=False):
    """TensorBase.forward, tensorBase_rotated_lights.py:868-1036 (ndc_ray=False branch).
    Random draws, in reference order: per-ray jitter (CPU rand_like, :717), xyz jitter
    (device randn_like, :937), background coin (CPU rand, :1004)."""
    viewdirs = rays[:, 3:6]
    xyz, z, valid = sample_ray(f, rays[:, :3], viewdirs, is_train, n_samples, jitter)
    dists = torch.cat((z[:, 1:] - z[:, :-1], torch.zeros_like(z[:, :1])), dim=-1)
    viewdirs = viewdirs.view(-1, 1, 3).expand(xyz.shape)
    light_idx = light_idx.view(-1, 1, 1).expand((*xyz.shape[:-1], 1))
    valid = _refine_valid(f, xyz, valid)
    dev = xyz.device
    shp2 = xyz.shape[:2]
    sigma = torch.zeros(shp2, device=dev)
    rgb = torch.zeros((*shp2, 3), device=dev)
    normal = torch.zeros((*shp2, 3), device=dev)
    albedo = torch.zeros((*shp2, 3), device=dev)
    rough = torch.zeros((*shp2, 1), device=dev)
    alb_cost = torch.zeros((*shp2, 1), device=dev)
    rough_cost = torch.zeros((*shp2, 1), device=dev)
    ndiff = torch.zeros((*shp2, 1), device=dev)
    norient = torch.zeros((*shp2, 1), device=dev)
    if valid.any():
        xyz = normalize_coord(f, xyz)
        sigma[valid] = feature2density(f, density_feature(f, xyz[valid]))
    _, weight, _ = raw2alpha(sigma, dists * f.distance_scale)
    app_mask = weight > f.weight_thres
    if app_mask.any():
        rad, intr = both_feature(f, xyz[app_mask], light_idx[app_mask])
        rgb[app_mask] = mlp_render_fea(f, f.mlp_rgb, viewdirs[app_mask], rad)
        if is_relight:
            brdf = mlp_pe_and_feature(f, f.mlp_brdf, xyz[app_mask], intr, torch.sigmoid)
            v_alb, v_rough = brdf[..., :3], (brdf[..., 3:4] * 0.9 + 0.09)
            albedo[app_mask] = v_alb
            rough[app_mask] = v_rough
            noise = torch.randn_like(xyz[app_mask]) if xyz_noise is None else xyz_noise.to(dev)
            xyz_j = xyz[app_mask] + noise * 0.01
            brdf_j = mlp_pe_and_feature(f, f.mlp_brdf, xyz_j, intrin_feature(f, xyz_j), torch.sigmoid)
            alb_cost[app_mask] = relative_smoothness(v_alb, brdf_j[..., :3])
            rough_cost[app_mask] = relative_smoothness(v_rough, brdf_j[..., 3:4] * 0.9 + 0.09)
            if f.normals_kind == "purely_predicted":
                v_n = mlp_pe_and_feature(f, f.mlp_normal, xyz[app_mask], intr, torch.tanh)
            elif f.normals_kind == "purely_derived":
                v_n = derived_normals(f, xyz[app_mask])
            elif f.normals_kind == "derived_plus_predicted":
                d_n = derived_normals(f, xyz[app_mask])
                v_n = mlp_pe_and_feature(f, f.mlp_normal, xyz[app_mask], intr, torch.tanh)
                ndiff[app_mask] = torch.sum(torch.pow(v_n - d_n, 2), dim=-1, keepdim=True)
                norient[app_mask] = torch.sum(viewdirs[app_mask] * v_n, dim=-1, keepdim=True).clamp(min=0)
            else:
                raise NotImplementedError(f.normals_kind)
            normal[app_mask] = v_n
    acc = torch.sum(weight, -1)
    depth = torch.sum(weight * z, -1)
    rgb_map = torch.sum(weight[..., None] * rgb, -2)
    aux = dict(valid=valid, app_mask=app_mask, weight=weight, z=z)

    def coin():
        if white_bg:
            return True
        if not is_train:
            return False
        c = torch.rand((1,)) if bg_coin is None else bg_coin
        return bool(c < 0.5)

    if not is_relight:
        if coin():
            depth = depth + (1. - acc) * rays[..., -1]
            rgb_map = rgb_map + (1. - acc[..., None])
        out = (rgb_map, depth, None, None, None, None, acc, None, None, None, None, None)
        return out + (aux,) if return_aux else out
    normal_map = torch.sum(weight[..., None] * normal, -2)
    ndiff_map = torch.sum(weight[..., None] * ndiff, -2)
    norient_map = torch.sum(weight[..., None] * norient, -2)
    albedo_map = torch.sum(weight[..., None] * albedo, -2)
    rough_map = torch.sum(weight[..., None] * rough, -2)
    fresnel_map = torch.zeros_like(albedo_map).fill_(f.fixed_fresnel)
    alb_loss = torch.mean(torch.sum(weight[..., None] * alb_cost, -2))
    rough_loss = torch.mean(torch.sum(weight[..., None] * rough_cost, -2))
    if coin():
        depth = depth + (1. - acc) * rays[..., -1]
        rgb_map = rgb_map + (1. - acc[..., None])
        normal_map = normal_map + (1 - acc[..., None]) * torch.tensor([0.0, 0.0, 1.0], device=dev)
        albedo_map = albedo_map + (1 - acc[..., None])
        rough_map = rough_map + (1 - acc[..., None])
        fresnel_map = fresnel_map + (1 - acc[..., None])
    rgb_map = rgb_map.clamp(0, 1)
    if rgb_map.shape[0] > 0:
        rgb_map = linear2srgb(rgb_map)
    albedo_map = albedo_map.clamp(0, 1)
    fresnel_map = fresnel_map.clamp(0, 1)
    rough_map = rough_map.clamp(0, 1)
    normal_map = safe_l2_normalize(normal_map, dim=-1)
    acc_mask = acc > 0.5
    out = (rgb_map, depth, normal_map, albedo_map, rough_map, fresnel_map, acc, ndiff_map, norient_map,
           acc_mask, alb_loss, rough_loss)
    return out + (aux,) if return_aux else out


def init_forward(f: OracleField, rays, white_bg=True, is_train=False, n_samples=-1, jitter=None, bg_coin=None):
    """TensorBase_Init.forward, tensorBase_init.py:406-462 -> (rgb_map, depth_map)."""
    viewdirs = rays[:, 3:6]
    xyz, z, valid = sample_ray(f, rays[:, :3], viewdirs, is_train, n_samples, jitter)
    dists = torch.cat((z[:, 1:] - z[:, :-1], torch.zeros_like(z[:, :1])), dim=-1)
    viewdirs = viewdirs.view(-1, 1, 3).expand(xyz.shape)
    valid = _refine_valid(f, xyz, valid)
    sigma = torch.zeros(xyz.shape[:-1], device=xyz.device)
    rgb = torch.zeros((*xyz.shape[:2], 3), device=xyz.device)
    if valid.any():
        xyz = normalize_coord(f, xyz)
        sigma[valid] = feature2density(f, density_feature(f, xyz[valid]))
    _, weight, _ = raw2alpha(sigma, dists * f.distance_scale)
    app_mask = weight > f.weight_thres
    if app_mask.any():
        rgb[app_mask] = mlp_render_fea(f, f.mlp_rgb, viewdirs[app_mask], app_feature(f, xyz[app_mask]))
    acc = torch.sum(weight, -1)
    rgb_map = torch.sum(weight[..., None] * rgb, -2)
    c = True if white_bg else (is_train and bool((torch.rand((1,)) if bg_coin is None else bg_coin) < 0.5))
    if c:
        rgb_map = rgb_map + (1. - acc[..., None])
    rgb_map = rgb_map.clamp(0, 1)
    with torch.no_grad():
        depth = torch.sum(weight * z, -1)
        depth = depth + (1. - acc) * rays[..., -1]
    return rgb_map, depth


# ----------------------------------------------------------------------------------------
# the boundary
# ----------------------------------------------------------------------------------------
def renderer_train(f: OracleField, rays, light_idx, n_samples=-1, white_bg=True, is_train=False, is_relight=True,
                   sample_method='fixed_envirmap', chunk_size=15000, second_nsample=96, second_near=0.05,
                   second_far=1.5, jitter=None, xyz_noise=None, bg_coin=None, light_jitter=None):
    """Renderer_TensoIR_train, renderer.py:57-127 -> dict of 12 maps."""
    light_idx = light_idx.to(rays.device, torch.int32)
    (rgb_map, depth, normal, albedo, rough, fresnel, acc, ndiff, norient, acc_mask, alb_loss, rough_loss) = \
        primary_forward(f, rays, light_idx, white_bg, is_train, is_relight, n_samples, jitter, xyz_noise, bg_coin)
    if is_relight:
        masked = render_with_brdf(f, depth[acc_mask], normal[acc_mask], albedo[acc_mask],
                                  rough[acc_mask].repeat(1, 3), fresnel[acc_mask], rays[acc_mask],
                                  light_idx[acc_mask], sample_method, chunk_size, second_nsample, second_near,
                                  second_far, light_jitter)
        rgb_brdf = torch.ones_like(rgb_map)
        rgb_brdf[acc_mask] = masked
    else:
        rgb_brdf = torch.ones_like(rgb_map)
    return {"rgb_map": rgb_map, "depth_map": depth, "normal_map": normal, "albedo_map": albedo, "acc_map": acc,
            "roughness_map": rough, "fresnel_map": fresnel, "rgb_with_brdf_map": rgb_brdf,
            "normals_diff_map": ndiff, "normals_orientation_loss_map": norient,
            "albedo_smoothness_loss": alb_loss, "roughness_smoothness_loss": rough_loss}


# ----------------------------------------------------------------------------------------
# field maintenance used by the scene generator (alpha mask)
# ----------------------------------------------------------------------------------------
@torch.no_grad()
def compute_alpha(f: OracleField, xyz_locs, length=1):
    """tensorBase_rotated_lights.py:819-837."""
    if f.alpha_volume is not None:
        amask = sample_alpha(f, xyz_locs) > 0
    else:
        amask = torch.ones_like(xyz_locs[:, 0], dtype=bool)
    sigma = torch.zeros(xyz_locs.shape[:-1], device=xyz_locs.device)
    if amask.any():
        sigma[amask] = feature2density(f, density_feature(f, normalize_coord(f, xyz_locs[amask])))
    return 1 - torch.exp(-sigma * length).view(xyz_locs.shape[:-1])


@torch.no_grad()
def update_alpha_mask(f: OracleField, grid_size, thres=0.001):
    """getDenseAlpha + updateAlphaMask, tensorBase_rotated_lights.py:737-779; sets
    f.alpha_volume / f.alpha_aabb and returns the tight aabb."""
    gs = list(grid_size)
    _, _, _, step, _ = f.derived()
    samples = torch.stack(torch.meshgrid(torch.linspace(0, 1, gs[0]), torch.linspace(0, 1, gs[1]),
                                         torch.linspace(0, 1, gs[2]), indexing='ij'), -1).to(f.aabb.device)
    dense = f.aabb[0] * (1 - samples) + f.aabb[1] * samples
    alpha = torch.zeros_like(dense[..., 0])
    for i in range(gs[0]):
        alpha[i] = compute_alpha(f, dense[i].view(-1, 3), step).view((gs[1], gs[2]))
    dense = dense.transpose(0, 2).contiguous()
    alpha = alpha.clamp(0, 1).transpose(0, 2).contiguous()[None, None]
    alpha = F.max_pool3d(alpha, kernel_size=3, padding=1, stride=1).view(gs[::-1])
    alpha[alpha >= thres] = 1
    alpha[alpha < thres] = 0
    f.alpha_volume = alpha.view(1, 1, *alpha.shape[-3:])
    f.alpha_aabb = f.aabb.clone()
    valid = dense[alpha > 0.5]
    return torch.stack((valid.amin(0), valid.amax(0)))


# ----------------------------------------------------------------------------------------
# relighting pass (scripts/relight_importance.py) — "next" row (f)2 of SURVEY.md §8
# ----------------------------------------------------------------------------------------
class EnvLight:
    """Environment_Light of relight_utils.py:110-205, built from arrays {name: [H,W,3] float32} instead of a
    directory of .hdr files (read_hdr, relight_utils.py:598-611, is plain cv2 I/O)."""

    def __init__(self, maps: dict, device='cpu'):
        self.hdr_rgbs, self.hdr_pdf_sample, self.hdr_pdf_return, self.hdr_dir = {}, {}, {}, {}
        for name, arr in maps.items():
            rgb = torch.as_tensor(arr).float()
            self.hdr_rgbs[name] = rgb.to(device)
            inten = torch.sum(rgb, dim=2, keepdim=True)
            H, W, _ = inten.shape
            h_int = 1.0 / H
            sin_t = torch.sin(torch.linspace(0 + 0.5 * h_int, np.pi - 0.5 * h_int, H))
            pdf = inten * sin_t.view(-1, 1, 1)
            pdf = pdf / torch.sum(pdf)
            pdf_ret = pdf * H * W / (2 * np.pi * np.pi * sin_t.view(-1, 1, 1))
            self.hdr_pdf_sample[name] = pdf.to(device)
            self.hdr_pdf_return[name] = pdf_ret.to(device)
            lat, lng = np.pi / H, 2 * np.pi / W
            phi, theta = torch.meshgrid([torch.linspace(np.pi / 2 - 0.5 * lat, -np.pi / 2 + 0.5 * lat, H),
                                         torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, W)], indexing='ij')
            dirs = torch.stack([torch.cos(theta) * torch.cos(phi), torch.sin(theta) * torch.cos(phi),
                                torch.sin(phi)], dim=-1).view(H, W, 3)
            self.hdr_dir[name] = dirs.to(device)

    @torch.no_grad()
    def sample_light(self, name, bs, num_samples, light_dir_idx=None):
        """relight_utils.py:150-188 (importance branch).  ``light_dir_idx`` [bs,num_samples] replaces the multinomial
        draw of :169 when given."""
        pdf_s = self.hdr_pdf_sample[name].view(-1).expand(bs, -1)
        pdf_r = self.hdr_pdf_return[name].view(-1).expand(bs, -1)
        dirs = self.hdr_dir[name].view(-1, 3).expand(bs, -1, -1)
        rgbs = self.hdr_rgbs[name].view(-1, 3).expand(bs, -1, -1)
        if light_dir_idx is None:
            light_dir_idx = torch.multinomial(pdf_s, num_samples, replacement=True)
        ld = dirs.gather(1, light_dir_idx.unsqueeze(-1).expand(-1, -1, 3)).view(bs, num_samples, 3)
        lr = rgbs.gather(1, light_dir_idx.unsqueeze(-1).expand(-1, -1, 3)).view(bs, num_samples, 3)
        lp = pdf_r.gather(1, light_dir_idx).unsqueeze(-1)
        return ld, lr, lp

    def get_light(self, name, incident_dir):
        """relight_utils.py:193-205."""
        env = self.hdr_rgbs[name].permute(2, 0, 1).unsqueeze(0)
        phi = torch.arccos(incident_dir[:, 2]).reshape(-1) - 1e-6
        theta = torch.atan2(incident_dir[:, 1], incident_dir[:, 0]).reshape(-1)
        qy = (phi / np.pi) * 2 - 1
        qx = -theta / np.pi
        grid = torch.stack((qx, qy)).permute(1, 0).unsqueeze(0).unsqueeze(0)
        return F.grid_sample(env, grid, align_corners=True).squeeze().permute(1, 0).reshape(-1, 3)


@torch.no_grad()
def relight_chunk(f: OracleField, env: EnvLight, name, rays, maps, rescale_value, light_dir_idx=None,
                  num_samples=512, acc_thres=0.5, vis_equation='nerv'):
    """Per-chunk body of relight(), scripts/relight_importance.py:99-181.  ``maps`` = (depth, normal, albedo,
    roughness, fresnel, acc) of the primary march for ``rays``.  -> (with_bg, without_bg) [n,3]."""
    depth, normal, albedo, rough, fresnel, acc = maps
    dev = rays.device
    relight_rgb = torch.ones((rays.shape[0], 3), device=dev)
    mask = acc > acc_thres
    rays_o, rays_d = rays[:, :3], rays[:, 3:]
    surf = (rays_o + depth.unsqueeze(-1) * rays_d)[mask]
    m_n, m_a, m_r, m_f = normal[mask], albedo[mask], rough[mask], fresnel[mask]
    surf2l, l_rgb, l_pdf = env.sample_light(name, m_n.shape[0], num_samples, light_dir_idx)
    surf2c = safe_l2_normalize(-rays_d[mask], dim=-1)
    cosine = torch.einsum("ijk,ik->ij", surf2l, m_n)
    cmask = cosine > 1e-6
    vis = torch.zeros((*cmask.shape, 1), device=dev)
    pts = surf[:, None, :].expand((*cmask.shape, 3))[cmask]
    nerv, nerf = compute_transmittance(f, pts, surf2l[cmask], 96, 0.05, 1.5)
    vis[cmask] = (nerv if vis_equation == 'nerv' else nerf).unsqueeze(-1)
    spec = ggx_specular(m_n, surf2c, surf2l, m_r, m_f)
    brdf = (m_a * rescale_value).unsqueeze(1).expand(-1, surf2l.shape[1], -1) / np.pi + spec
    contrib = brdf * (vis * l_rgb) * cosine[:, :, None] / l_pdf
    srgb = torch.clamp(torch.mean(contrib, dim=1), min=0.0, max=1.0)
    if srgb.shape[0] > 0:
        srgb = linear2srgb(srgb)
    relight_rgb[mask] = srgb
    bg = linear2srgb(torch.clamp(env.get_light(name, rays_d), min=0.0, max=1.0))
    without_bg = torch.ones_like(bg)
    without_bg[mask] = relight_rgb[mask]
    acc_t = acc[..., None].clone()
    acc_t[acc_t <= 0.9] = 0.0
    with_bg = acc_t * without_bg + (1.0 - acc_t) * bg
    return with_bg, without_bg
