"""Synthetic "lego-shaped" scene and camera rays (SURVEY.md §8d).

No dataset ships with the reference and there is no network, so every test / bench input is
generated here, seeded with the reference scripts' own seed 20211202 (train_tensoIR.py:467-470).

* Scene: aabb [-1.5,1.5]^3 (dataLoader/tensoIR_rotation_setting.py:53), near/far 2/6 (:52).
  The density field is a union of axis-aligned boxes (base plate, studs, an arch and a back
  wall => concave, self-shadowing); each box is ONE rank-1 VM component: plane_k[c] =
  A*1[footprint], line_k[c] = 1[extent], A = 30 so sigma = softplus(30-10) = 20 inside.
* Cameras: pinhole, 800x800, cam_angle_x 0.6911 (focal 1111.1), on the upper hemisphere at
  radius 4, rays built like get_ray_directions + normalise + get_rays
  (dataLoader/ray_utils.py:25-43, :67-88; tensoIR_rotation_setting.py:103-114), restated.
"""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np
import torch

SEED = 20211202
MAT_MODE = ((0, 1), (0, 2), (1, 2))
VEC_MODE = (2, 1, 0)

# (lo_xyz, hi_xyz, orientation k) ; orientation k => plane over axes MAT_MODE[k], line over VEC_MODE[k]
_BOXES: List[Tuple[Tuple[float, float, float], Tuple[float, float, float], int]] = []


def _lego_boxes():
    if _BOXES:
        return _BOXES
    b = _BOXES
    b.append(((-1.0, -1.0, -0.95), (1.0, 1.0, -0.65), 0))                     # base plate
    for ix in range(4):                                                      # 4x3 studs on the plate
        for iy in range(3):
            cx, cy = -0.75 + 0.5 * ix, -0.6 + 0.6 * iy
            b.append(((cx - 0.12, cy - 0.12, -0.65), (cx + 0.12, cy + 0.12, -0.45), 0))
    b.append(((-0.85, -0.25, -0.65), (-0.55, 0.25, 0.55), 1))                 # arch pillar L
    b.append(((0.55, -0.25, -0.65), (0.85, 0.25, 0.55), 1))                   # arch pillar R
    b.append(((-0.85, -0.25, 0.55), (0.85, 0.25, 0.85), 1))                   # arch beam
    b.append(((-1.0, 0.8, -0.65), (1.0, 1.0, 0.4), 2))                        # back wall
    b.append(((-0.2, -0.9, -0.65), (0.2, -0.6, -0.1), 2))                     # front block
    return b


def box_density_factors(grid_size: Sequence[int], aabb: torch.Tensor, n_comp: Sequence[int] = (16, 16, 16),
                        amplitude: float = 30.0, noise: float = 1e-3, generator=None):
    """Return (planes, lines) in the reference layout: plane k [1,C,G[m1],G[m0]], line k
    [1,C,G[v],1] (tensoRF_rotated_lights.py:19-29)."""
    g = torch.Generator().manual_seed(SEED + 7) if generator is None else generator
    lo, hi = aabb[0].tolist(), aabb[1].tolist()
    coords = [torch.linspace(lo[a], hi[a], int(grid_size[a])) for a in range(3)]
    planes, lines = [], []
    used = [0, 0, 0]
    for k in range(3):
        m0, m1 = MAT_MODE[k]
        v = VEC_MODE[k]
        planes.append(noise * torch.randn((1, n_comp[k], int(grid_size[m1]), int(grid_size[m0])), generator=g))
        lines.append(noise * torch.randn((1, n_comp[k], int(grid_size[v]), 1), generator=g))
    for (blo, bhi, k) in _lego_boxes():
        c = used[k]
        if c >= n_comp[k]:
            continue
        used[k] += 1
        m0, m1 = MAT_MODE[k]
        v = VEC_MODE[k]
        in0 = ((coords[m0] >= blo[m0]) & (coords[m0] <= bhi[m0])).float()
        in1 = ((coords[m1] >= blo[m1]) & (coords[m1] <= bhi[m1])).float()
        inv = ((coords[v] >= blo[v]) & (coords[v] <= bhi[v])).float()
        planes[k][0, c] = amplitude * in1[:, None] * in0[None, :]
        lines[k][0, c, :, 0] = inv
    return planes, lines


@torch.no_grad()
def install_lego_density(model, amplitude: float = 30.0):
    """Overwrite ``model.density_plane/.density_line`` (reference-layout ParameterLists) in
    place with the box scene.  Works on the reference model and on tensoir_b200's mirror."""
    gs = [int(x) for x in model.gridSize.tolist()]
    n_comp = [p.shape[1] for p in model.density_plane]
    planes, lines = box_density_factors(gs, model.aabb.detach().cpu(), n_comp, amplitude)
    for k in range(3):
        model.density_plane[k].data.copy_(planes[k].to(model.density_plane[k].device))
        model.density_line[k].data.copy_(lines[k].to(model.density_line[k].device))


def hemisphere_poses(n_views: int, radius: float = 4.0, seed: int = SEED) -> torch.Tensor:
    """n camera-to-world matrices [n,4,4] (OpenCV axes: x right, y down, z forward) on the
    upper hemisphere, looking at the origin."""
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n_views):
        az = 2 * math.pi * (i / max(n_views, 1)) + rs.uniform(-0.05, 0.05)
        el = math.radians(20.0 + 50.0 * ((i * 0.61803398875) % 1.0))
        pos = np.array([radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az),
                        radius * math.sin(el)])
        fwd = -pos / np.linalg.norm(pos)
        right = np.cross(fwd, np.array([0.0, 0.0, 1.0]))
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        c2w = np.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, pos
        out.append(c2w)
    return torch.tensor(np.stack(out), dtype=torch.float32)


def pixel_rays(c2w: torch.Tensor, pix: torch.Tensor, H: int = 800, W: int = 800,
               cam_angle_x: float = 0.6911) -> torch.Tensor:
    """Rays [n,6] for flat pixel ids ``pix`` (row-major, id = j*W+i) of one camera.
    directions = [(i+0.5-W/2)/f, (j+0.5-H/2)/f, 1] normalised, rotated by c2w[:3,:3]
    (ray_utils.py:25-43, :67-88; tensoIR_rotation_setting.py:103-114)."""
    focal = 0.5 * W / math.tan(0.5 * cam_angle_x)
    i = (pix % W).float() + 0.5
    j = (pix // W).float() + 0.5
    d = torch.stack([(i - W / 2) / focal, (j - H / 2) / focal, torch.ones_like(i)], -1)
    d = d / torch.norm(d, dim=-1, keepdim=True)
    rays_d = d @ c2w[:3, :3].T
    rays_o = c2w[:3, 3].expand(rays_d.shape)
    return torch.cat([rays_o, rays_d], 1)


def image_rays(c2w: torch.Tensor, H: int = 800, W: int = 800, crop: int = 0) -> torch.Tensor:
    """All rays of one view; ``crop`` > 0 selects the crop x crop centre window (config 1)."""
    if crop:
        j0, i0 = (H - crop) // 2, (W - crop) // 2
        jj, ii = torch.meshgrid(torch.arange(j0, j0 + crop), torch.arange(i0, i0 + crop), indexing='ij')
        pix = (jj * W + ii).reshape(-1)
    else:
        pix = torch.arange(H * W)
    return pixel_rays(c2w, pix, H, W)


def training_batch(poses: torch.Tensor, batch: int, step: int, H: int = 800, W: int = 800,
                   n_lights: int = 1, seed: int = SEED):
    """One random-ray training batch drawn from all (view, pixel) pairs like
    SimpleSampler + all_rays fancy-indexing (train_tensoIR.py:43-48, :239-242), generated on
    the fly instead of materialising the [n_views*H*W, 6] table.
    Returns rays [batch,6] fp32 and light_idx [batch,1] int32 (CPU tensors)."""
    g = torch.Generator().manual_seed(seed + 1000003 * step)
    view = torch.randint(0, poses.shape[0], (batch,), generator=g)
    pix = torch.randint(0, H * W, (batch,), generator=g)
    rays = torch.empty(batch, 6)
    for v in view.unique().tolist():
        m = view == v
        rays[m] = pixel_rays(poses[v], pix[m], H, W)
    light = torch.randint(0, n_lights, (batch, 1), generator=g, dtype=torch.int32)
    return rays, light


def training_batch_ids(n_views: int, batch: int, step: int, H: int = 800, W: int = 800, n_lights: int = 1,
                       seed: int = SEED):
    """The (view, pixel, light) ids of :func:`training_batch` without building the rays (same generator sequence):
    what the host sends per step when the rays are generated on the device (ops.generate_rays, SURVEY.md 8 f4)."""
    g = torch.Generator().manual_seed(seed + 1000003 * step)
    view = torch.randint(0, n_views, (batch,), generator=g)
    pix = torch.randint(0, H * W, (batch,), generator=g)
    light = torch.randint(0, n_lights, (batch, 1), generator=g, dtype=torch.int32)
    return view.to(torch.int32), pix.to(torch.int32), light


def make_lego_model(grid: int, device, *, lights=("000",), general=False, mask_res=None, seed: int = SEED,
                    envmap=(16, 32)):
    """The benchmark field: TensorVMSplit at ``grid``^3 on aabb +-1.5 with the lego box density installed,
    reference initialisation for everything else (appearance 0.1*N(0,1), MLPs / basis / light_line / lgtSGs at
    their default init under ``seed``), and an alpha mask from updateAlphaMask (<= 256^3, train_tensoIR.py:385-389)."""
    from .tensorf import TensorVMSplit
    torch.manual_seed(seed)
    aabb = torch.tensor([[-1.5] * 3, [1.5] * 3], device=device)
    kw = dict(density_n_comp=[16] * 3, appearance_n_comp=[48] * 3, app_dim=27, near_far=[2.0, 6.0],
              shadingMode='MLP_Fea', alphaMask_thres=0.001, density_shift=-10, distance_scale=25, pos_pe=2, view_pe=2,
              fea_pe=2, featureC=128, step_ratio=0.5, fea2denseAct='softplus', normals_kind='derived_plus_predicted',
              light_kind='sg', numLgtSGs=128, envmap_h=int(envmap[0]), envmap_w=int(envmap[1]))
    if general:
        kw["light_name_list"] = list(lights)
    else:
        kw["light_rotation"] = list(lights)
    m = TensorVMSplit(aabb, [grid] * 3, device, **kw)
    install_lego_density(m)
    r = mask_res or min(grid, 256)
    m.updateAlphaMask((r, r, r))
    return m


def n_samples_for(grid: int, step_ratio: float = 0.5, cap: int = 1000000) -> int:
    """min(args.nSamples, cal_n_samples(reso, step_ratio)) (train_tensoIR.py:161, utils.py:63-64)."""
    return min(cap, int(np.linalg.norm([grid] * 3) / step_ratio))


# per-box albedo of the synthetic test views (base plate, studs, arch, wall, block), linear RGB
_BOX_ALBEDO = ((0.70, 0.12, 0.10), (0.85, 0.75, 0.20), (0.15, 0.35, 0.75), (0.30, 0.65, 0.30), (0.55, 0.55, 0.60))


def _box_albedo(b: int) -> Tuple[float, float, float]:
    if b == 0:
        return _BOX_ALBEDO[0]
    if b <= 12:
        return _BOX_ALBEDO[1]
    if b <= 15:
        return _BOX_ALBEDO[2]
    return _BOX_ALBEDO[3] if b == 16 else _BOX_ALBEDO[4]


def trace_boxes(rays: torch.Tensor):
    """Nearest hit of each ray [n,6] with the lego boxes (slab test, fp64): (hit [n] bool, box id [n] long,
    face normal [n,3] float32, pointing against the ray)."""
    o, d = rays[:, :3].double(), rays[:, 3:6].double()
    n = rays.shape[0]
    best = torch.full((n,), float("inf"), dtype=torch.float64)
    box = torch.full((n,), -1, dtype=torch.long)
    axis = torch.zeros(n, dtype=torch.long)
    inv = 1.0 / torch.where(d == 0, torch.full_like(d, 1e-30), d)
    for b, (lo, hi, _) in enumerate(_lego_boxes()):
        t0 = (torch.tensor(lo, dtype=torch.float64) - o) * inv
        t1 = (torch.tensor(hi, dtype=torch.float64) - o) * inv
        tn = torch.minimum(t0, t1)
        t_in, ax = tn.max(dim=1)
        t_out = torch.maximum(t0, t1).min(dim=1).values
        hit = (t_in <= t_out) & (t_in > 0) & (t_in < best)
        best = torch.where(hit, t_in, best)
        box = torch.where(hit, torch.full_like(box, b), box)
        axis = torch.where(hit, ax, axis)
    found = box >= 0
    normal = torch.zeros(n, 3)
    sgn = -torch.sign(d.gather(1, axis[:, None])).float()
    normal.scatter_(1, axis[:, None], sgn)
    normal[~found] = 0.0
    return found, box, normal


class SyntheticViews:
    """Test views of the lego box scene with analytic ground truth, following the item contract of the reference's test
    dataset (dataLoader/tensoIR_rotation_setting.py:180-245).  Item i, for camera ``poses[i]``:
        rays [H*W,6], rgbs [L,H*W,3], light_idx [L,H*W,1] int32, rgbs_mask [H*W,1] bool, albedo [H*W,3],
        normals [H*W,3] (background (0,0,1)), img_wh, c2w, w2c.
    The mask, albedo and face normals come from ray-box intersection; rgb is albedo times a Lambert shading
    0.25 + 0.75 max(n.l, 0) under light l (a sun direction rotated by 360 l / L degrees about z), over white.

    With ``light_names`` the views follow the reference's relighting test set instead
    (dataLoader/tensoIR_relighting_test.py:217-228): ``split`` is 'test', ``light_names`` is the list, rgbs holds one
    ground-truth image per name, light_idx is 0 everywhere and the item gains normals_white (background (1,1,1))."""

    def __init__(self, poses: torch.Tensor, H: int, W: int, n_lights: int = 1, cam_angle_x: float = 0.6911,
                 near_far=(2.0, 6.0), light_names=None):
        if light_names is not None:
            self.split = 'test'
            self.light_names = list(light_names)
            n_lights = len(self.light_names)
        self.poses = poses.float()
        self.img_wh = (int(W), int(H))
        self.near_far = list(near_far)
        self.white_bg = True
        self.lights_probes = None
        self.n_lights = int(n_lights)
        self.cam_angle_x = cam_angle_x
        self.focal = 0.5 * W / math.tan(0.5 * cam_angle_x)

    def __len__(self):
        return int(self.poses.shape[0])

    def __getitem__(self, i):
        W, H = self.img_wh
        c2w = self.poses[i]
        focal = self.focal
        pix = torch.arange(H * W)
        u = (pix % W).float() + 0.5
        v = (pix // W).float() + 0.5
        d = torch.stack([(u - W / 2) / focal, (v - H / 2) / focal, torch.ones_like(u)], -1)
        d = d / torch.norm(d, dim=-1, keepdim=True)
        rays = torch.cat([c2w[:3, 3].expand(H * W, 3), d @ c2w[:3, :3].T], 1)
        hit, box, normal = trace_boxes(rays)
        alb_tab = torch.tensor([_box_albedo(b) for b in range(len(_lego_boxes()))])
        albedo = torch.ones(H * W, 3)
        albedo[hit] = alb_tab[box[hit]]
        normals = torch.tensor([0.0, 0.0, 1.0]).expand(H * W, 3).clone()
        normals[hit] = normal[hit]
        rgbs = []
        for l in range(self.n_lights):
            a = 2 * math.pi * l / self.n_lights
            sun = torch.tensor([0.5 * math.cos(a), 0.5 * math.sin(a), 0.8])
            sun = sun / sun.norm()
            shade = 0.25 + 0.75 * (normal @ sun).clamp(min=0.0)
            rgb = torch.ones(H * W, 3)
            rgb[hit] = albedo[hit] * shade[hit, None]
            rgbs.append(rgb)
        light_idx = torch.arange(self.n_lights, dtype=torch.int32).view(-1, 1, 1).expand(-1, H * W, 1).contiguous()
        item = {'img_wh': self.img_wh, 'light_idx': light_idx, 'rgbs': torch.stack(rgbs, 0),
                'rgbs_mask': hit.view(-1, 1), 'albedo': albedo, 'rays': rays, 'normals': normals,
                'c2w': c2w, 'w2c': torch.linalg.inv(c2w)}
        if hasattr(self, 'light_names'):
            item['light_idx'] = torch.zeros_like(light_idx)
            normals_white = torch.ones(H * W, 3)
            normals_white[hit] = normal[hit]
            item['normals_white'] = normals_white
        return item
