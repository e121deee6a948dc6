"""Host-side mirror of the reference field base class (models/tensorBase_rotated_lights.py,
models/tensorBase_general_multi_lights.py, models/tensorBase_init.py).

PyTorch owns parameters, autograd and the light model; everything per-sample (ray sampling, alpha-mask
filter, VM gathers, compositing, MLP heads on the secondary rays) runs in the CUDA kernels of
tensoir_b200/csrc through the C ABI.  Constructor arguments, attribute names, state_dict keys and
return tuples follow the reference so that train_tensoIR*.py and renderer.py callers run unchanged.
"""
from __future__ import annotations

import time

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from . import primary


def positional_encoding(positions, freqs):
    """tensorBase_rotated_lights.py:12-17 (index layout d*F+f, [sin | cos])."""
    freq_bands = 2 ** torch.arange(freqs, device=positions.device).float()
    pts = (positions[..., None] * freq_bands).reshape(positions.shape[:-1] + (freqs * positions.shape[-1],))
    return torch.cat([torch.sin(pts), torch.cos(pts)], dim=-1)


def safe_l2_normalize(x, dim=None, eps=1e-6):
    """dataLoader/ray_utils.py:278."""
    return F.normalize(x, p=2, dim=dim, eps=eps)


def raw2alpha(sigma, dist):
    """Dense reference form (tensorBase_rotated_lights.py:21-28) kept for API compatibility
    (train scripts import it); the hot path composites inside the march kernels instead."""
    alpha = 1. - torch.exp(-sigma * dist)
    T = torch.cumprod(torch.cat([torch.ones(alpha.shape[0], 1).to(alpha.device), 1. - alpha + 1e-10], -1), -1)
    return alpha, alpha * T[:, :-1], T[:, -1:]


def compute_energy(lgtSGs):
    """tensorBase_rotated_lights.py:43-47."""
    lam = torch.abs(lgtSGs[:, 3:4])
    mu = torch.abs(lgtSGs[:, 4:])
    return mu * 2.0 * np.pi / lam * (1.0 - torch.exp(-2.0 * lam))


def fibonacci_sphere(samples=1):
    """tensorBase_rotated_lights.py:49-67."""
    i = np.arange(samples, dtype=np.float64)
    z = 1 - (i / float(samples - 1)) * 2
    radius = np.sqrt(1 - z * z)
    theta = np.pi * (3. - np.sqrt(5.)) * i
    return np.stack([np.cos(theta) * radius, np.sin(theta) * radius, z], axis=-1)


def render_envmap_sg(lgtSGs, viewdirs):
    """SG mixture, tensorBase_rotated_lights.py:70-86."""
    viewdirs = viewdirs.to(lgtSGs.device).unsqueeze(-2)
    dots_sh = list(viewdirs.shape[:-2])
    M = lgtSGs.shape[0]
    sg = lgtSGs.view([1, ] * len(dots_sh) + [M, 7]).expand(dots_sh + [M, 7])
    lobes = sg[..., :3] / (torch.norm(sg[..., :3], dim=-1, keepdim=True))
    lambdas = torch.abs(sg[..., 3:4])
    mus = torch.abs(sg[..., -3:])
    rgb = mus * torch.exp(lambdas * (torch.sum(viewdirs * lobes, dim=-1, keepdim=True) - 1.))
    return torch.sum(rgb, dim=-2)


class AlphaGridMask(torch.nn.Module):
    """tensorBase_rotated_lights.py:100-119.  ``alpha_volume`` stays a float [1,1,Z,Y,X] tensor
    (checkpoint format); the kernels read the byte shadows DeviceField builds from it."""

    def __init__(self, device, aabb, alpha_volume):
        super().__init__()
        self.device = device
        self.aabb = aabb.to(self.device)
        self.aabbSize = self.aabb[1] - self.aabb[0]
        self.invgridSize = 1.0 / self.aabbSize * 2
        self.alpha_volume = alpha_volume.view(1, 1, *alpha_volume.shape[-3:])
        self.gridSize = torch.LongTensor([alpha_volume.shape[-1], alpha_volume.shape[-2],
                                          alpha_volume.shape[-3]]).to(self.device)
        self._host_geom = {"lo": self.aabb[0].tolist(), "inv": self.invgridSize.tolist()}

    def sample_alpha(self, xyz_sampled):
        """Trilinear lookup; on CUDA the >0 test of callers is served by tir_alpha_mask_points, this
        float-valued form is kept for API parity (relight_utils / user code call it)."""
        g = self.normalize_coord(xyz_sampled)
        return F.grid_sample(self.alpha_volume, g.view(1, -1, 1, 1, 3), align_corners=True).view(-1)

    def normalize_coord(self, xyz_sampled):
        return (xyz_sampled - self.aabb[0]) * self.invgridSize - 1


class _Mlp3(torch.nn.Module):
    """Shared shape of MLPRender_Fea / MLPBRDF_PEandFeature (tensorBase_rotated_lights.py:122-146,
    :182-208): Linear-ReLU-Linear-ReLU-Linear, last bias 0; state_dict keys mlp.{0,2,4}.{weight,bias}."""

    def __init__(self, in_dim, featureC, outc):
        super().__init__()
        self.in_mlpC = in_dim
        self.mlp = torch.nn.Sequential(torch.nn.Linear(in_dim, featureC), torch.nn.ReLU(inplace=True),
                                       torch.nn.Linear(featureC, featureC), torch.nn.ReLU(inplace=True),
                                       torch.nn.Linear(featureC, outc))
        torch.nn.init.constant_(self.mlp[-1].bias, 0)


class MLPRender_Fea(_Mlp3):
    def __init__(self, inChanel, viewpe=6, feape=6, featureC=128):
        super().__init__(2 * viewpe * 3 + 2 * feape * inChanel + 3 + inChanel, featureC, 3)
        self.viewpe, self.feape = viewpe, feape

    def forward(self, pts, viewdirs, features):
        indata = [features, viewdirs]
        if self.feape > 0:
            indata += [positional_encoding(features, self.feape)]
        if self.viewpe > 0:
            indata += [positional_encoding(viewdirs, self.viewpe)]
        return torch.sigmoid(self.mlp(torch.cat(indata, dim=-1)))


class MLPBRDF_PEandFeature(_Mlp3):
    def __init__(self, inChanel, pospe=6, feape=6, featureC=128, outc=1, act_net=nn.Sigmoid()):
        super().__init__(2 * pospe * 3 + 2 * feape * inChanel + 3 + inChanel, featureC, outc)
        self.pospe, self.feape, self.outc, self.act_net = pospe, feape, outc, act_net

    def forward(self, pts, features):
        indata = [features, pts]
        if self.feape > 0:
            indata += [positional_encoding(features, self.feape)]
        if self.pospe > 0:
            indata += [positional_encoding(pts, self.pospe)]
        return self.act_net(self.mlp(torch.cat(indata, dim=-1)))


class TensorBase(torch.nn.Module):
    """models/tensorBase_rotated_lights.py:343-1036 / tensorBase_general_multi_lights.py.
    ``light_name_list`` given  => general multi-light variant (one SG set per light, no rotation);
    otherwise the rotated variant (one SG set, rotated per light)."""

    def __init__(self, aabb, gridSize, device, density_n_comp=8, appearance_n_comp=24, app_dim=27,
                 shadingMode='MLP_PE', alphaMask=None, near_far=[2.0, 6.0], density_shift=-10,
                 alphaMask_thres=0.001, distance_scale=25, rayMarch_weight_thres=0.0001, pos_pe=2, view_pe=2,
                 fea_pe=2, featureC=128, step_ratio=2.0, fea2denseAct='softplus', normals_kind="purely_predicted",
                 light_rotation=['000', '120', '240'], light_name_list=None, envmap_w=32, envmap_h=16,
                 light_kind='pixel', dataset=None, numLgtSGs=128, fixed_fresnel=0.04, **kwargs):
        super().__init__()
        self.density_n_comp = density_n_comp
        self.app_n_comp = appearance_n_comp
        self.app_dim = app_dim
        self.aabb = aabb
        self.alphaMask = alphaMask
        self.device = device
        self.density_shift = density_shift
        self.alphaMask_thres = alphaMask_thres
        self.distance_scale = distance_scale
        self.rayMarch_weight_thres = rayMarch_weight_thres
        self.fea2denseAct = fea2denseAct
        self.near_far = near_far
        self.step_ratio = step_ratio
        self.shadingMode, self.normals_kind, self.pos_pe, self.view_pe, self.fea_pe, self.featureC = \
            shadingMode, normals_kind, pos_pe, view_pe, fea_pe, featureC
        self.general_lights = light_name_list is not None
        if self.general_lights:
            self.light_num = len(light_name_list)
            self.light_name_list = light_name_list
        else:
            self.light_num = len(light_rotation)
        self.light_rotation = [int(r) for r in light_rotation]
        self.envmap_w, self.envmap_h = envmap_w, envmap_h
        self.dataset = dataset
        self.light_kind = light_kind
        self.numLgtSGs = numLgtSGs
        self.fixed_fresnel = fixed_fresnel
        self.update_stepSize(gridSize)
        self.matMode = [[0, 1], [0, 2], [1, 2]]
        self.vecMode = [2, 1, 0]
        self.comp_w = [1, 1, 1]
        self.init_svd_volume(gridSize[0], device)
        self.init_render_func(shadingMode, pos_pe, view_pe, fea_pe, featureC, device)
        self.init_light()

    # ---- construction ------------------------------------------------------------------
    def init_render_func(self, shadingMode, pos_pe, view_pe, fea_pe, featureC, device):
        """tensorBase_rotated_lights.py:405-434.  Only the shipped configuration (MLP_Fea,
        configs/**: shadingMode = MLP_Fea) has kernels; other modes are out of scope (SURVEY.md §2)."""
        if shadingMode != 'MLP_Fea':
            raise NotImplementedError(f"shadingMode {shadingMode!r}: only 'MLP_Fea' is on the CUDA hot path")
        self.renderModule = MLPRender_Fea(self.app_dim, view_pe, fea_pe, featureC).to(device)
        if self.normals_kind not in ("purely_predicted", "derived_plus_predicted", "purely_derived"):
            raise NotImplementedError(f"normals_kind {self.normals_kind!r}")
        self.renderModule_normal = MLPBRDF_PEandFeature(self.app_dim, pos_pe, fea_pe, featureC, outc=3,
                                                        act_net=nn.Tanh()).to(device)
        self.renderModule_brdf = MLPBRDF_PEandFeature(self.app_dim, pos_pe, fea_pe, featureC, outc=4,
                                                      act_net=nn.Sigmoid()).to(device)

    def generate_envir_map_dir(self, envmap_h, envmap_w, is_jittor=False):
        """tensorBase_rotated_lights.py:435-453."""
        lat = np.pi / envmap_h
        lng = 2 * np.pi / envmap_w
        phi, theta = torch.meshgrid([torch.linspace(np.pi / 2 - 0.5 * lat, -np.pi / 2 + 0.5 * lat, envmap_h),
                                     torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, envmap_w)], indexing='ij')
        sin_phi = torch.sin(torch.pi / 2 - phi)
        light_area_weight = 4 * torch.pi * sin_phi / torch.sum(sin_phi)
        assert 0 not in light_area_weight, "There shouldn't be light pixel that doesn't contribute"
        light_area_weight = light_area_weight.to(torch.float32).reshape(-1)
        if is_jittor:
            phi = phi + lat * (torch.rand_like(phi) - 0.5)
            theta = theta + lng * (torch.rand_like(theta) - 0.5)
        view_dirs = torch.stack([torch.cos(theta) * torch.cos(phi), torch.sin(theta) * torch.cos(phi),
                                 torch.sin(phi)], dim=-1).view(-1, 3)
        return light_area_weight, view_dirs

    def _init_sg(self):
        """[M,7] = lobe(3) + lambda(1) + mu(3), initialised as tensorBase_rotated_lights.py:462-476."""
        sg = nn.Parameter(torch.randn(self.numLgtSGs, 7), requires_grad=True)
        sg.data[:, -2:] = sg.data[:, -3:-2].expand((-1, 2))
        sg.data[:, 3:4] = 10. + torch.abs(sg.data[:, 3:4] * 20.)
        energy = compute_energy(sg.data)
        sg.data[:, 4:] = torch.abs(sg.data[:, 4:]) / torch.sum(energy, dim=0, keepdim=True) * 2. * np.pi * 0.8
        lobes = fibonacci_sphere(self.numLgtSGs // 2).astype(np.float32)
        sg.data[:self.numLgtSGs // 2, :3] = torch.from_numpy(lobes)
        sg.data[self.numLgtSGs // 2:, :3] = torch.from_numpy(lobes)
        return sg

    def init_light(self):
        """tensorBase_rotated_lights.py:455-488 / tensorBase_general_multi_lights.py:455-479 (light_kind 'sg')."""
        self.light_area_weight, self.fixed_viewdirs = self.generate_envir_map_dir(self.envmap_h, self.envmap_w)
        if self.light_kind != 'sg':
            raise NotImplementedError("only light_kind='sg' (all shipped configs) is supported")
        if self.general_lights:
            # plain Python list, as in the reference: NOT part of state_dict (SURVEY.md §5)
            self.lgtSGs_list = [nn.Parameter(self._init_sg().data.to(self.device)) for _ in range(self.light_num)]
        else:
            self.lgtSGs = nn.Parameter(self._init_sg().data.to(self.device))
            mats = []
            for i in range(self.light_num):
                a = torch.tensor(self.light_rotation[i] / 180 * torch.pi).to(torch.float32)
                mats.append(torch.tensor([[torch.cos(a), -torch.sin(a), 0], [torch.sin(a), torch.cos(a), 0],
                                          [0, 0, 1]]).to(torch.float32))
            self.light_rotation_matrix = torch.stack(mats, dim=0).to(self.device)

    def gen_light_incident_dirs(self, sample_number=-1, method='fixed_envirmap', device='cuda'):
        """tensorBase_rotated_lights.py:492-574.  Draws stay on the host in the reference's order."""
        if method == 'fixed_envirmap':
            dirs = self.fixed_viewdirs
        elif method in ('stratified_sampling', 'stratifed_sample_equal_areas'):
            H, W = self.envmap_h, self.envmap_w
            lng = 2 * np.pi / W
            if method == 'stratified_sampling':
                lat = np.pi / H
                a_b, th_b = torch.meshgrid([torch.linspace(np.pi / 2 - 0.5 * lat, -np.pi / 2 + 0.5 * lat, H),
                                            torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, W)], indexing='ij')
                a_j, th_j = lat * (torch.rand_like(a_b) - 0.5), lng * (torch.rand_like(th_b) - 0.5)
                phi, theta = a_b + a_j, th_b + th_j
            else:
                sz = 2 / H
                a_b, th_b = torch.meshgrid([torch.linspace(1 - 0.5 * sz, -1 + 0.5 * sz, H),
                                            torch.linspace(np.pi - 0.5 * lng, -np.pi + 0.5 * lng, W)], indexing='ij')
                a_j, th_j = sz * (torch.rand_like(a_b) - 0.5), lng * (torch.rand_like(th_b) - 0.5)
                phi, theta = torch.asin(a_b + a_j), th_b + th_j
            dirs = torch.stack([torch.cos(theta) * torch.cos(phi), torch.sin(theta) * torch.cos(phi),
                                torch.sin(phi)], dim=-1)
        elif method == 'importance_sample':
            # tensorBase_rotated_lights.py:547-572: sample ``sample_number`` directions of a jittered 128x256 grid with
            # probability ~ SG-light intensity * sin(theta); returns (dirs, rgbs, pdf) instead of a direction table
            _, view_dirs = self.generate_envir_map_dir(128, 256, is_jittor=True)
            envir_map = self.get_light_rgbs(view_dirs.reshape(-1, 3).to(device), device=device)[0]
            with torch.no_grad():
                envir_map = envir_map.reshape(128, 256, 3)
                intensity = torch.sum(envir_map, dim=2, keepdim=True)
                H, W, _ = intensity.shape
                sin_theta = torch.sin(torch.linspace(0 + 0.5 / H, np.pi - 0.5 / H, H)).to(device)
                pdf = intensity * sin_theta.view(-1, 1, 1)
                pdf_to_sample = pdf / torch.sum(pdf)
                pdf_to_compute = pdf_to_sample * H * W / (2 * np.pi * np.pi * sin_theta.view(-1, 1, 1))
                idx = torch.multinomial(pdf_to_sample.view(-1), sample_number, replacement=True)
                light_dir = view_dirs.view(-1, 3).to(device).index_select(0, idx)
                light_rgb = envir_map.view(-1, 3).index_select(0, idx)
                light_pdf = pdf_to_compute.view(-1, 1).index_select(0, idx)
                return light_dir, light_rgb, light_pdf
        else:
            raise NotImplementedError(f"light sampling method {method!r}")
        return dirs.reshape(-1, 3)

    def get_light_rgbs(self, incident_light_directions=None, device='cuda'):
        """tensorBase_rotated_lights.py:577-606 (SG branch) -> [light_num, n, 3]."""
        if self.general_lights:
            d = incident_light_directions.to(device).reshape(-1, 3)
            return torch.stack([render_envmap_sg(s.to(device), d).reshape(-1, 3) for s in self.lgtSGs_list], dim=0)
        d = incident_light_directions.to(device).reshape(1, -1, 3)
        rot = self.light_rotation_matrix.to(device)
        d = torch.matmul(d, rot).reshape(-1, 3)
        return render_envmap_sg(self.lgtSGs.to(device), d).reshape(self.light_num, -1, 3)

    def update_stepSize(self, gridSize):
        """tensorBase_rotated_lights.py:608-619."""
        self.aabbSize = self.aabb[1] - self.aabb[0]
        self.invaabbSize = 2.0 / self.aabbSize
        self.gridSize = torch.LongTensor(gridSize).to(self.device)
        self.units = self.aabbSize / (self.gridSize - 1)
        # the step and the diagonal are reduced on the host: on a non-cubic grid the three units differ, and a CUDA mean
        # may round differently from the CPU one, which would move every sample position by an ulp of the step
        size_h = self.aabbSize.detach().cpu()
        step_h = torch.mean(size_h / (torch.LongTensor(gridSize) - 1)) * self.step_ratio
        self.stepSize = step_h.to(self.device)
        self.aabbDiag = torch.sqrt(torch.sum(torch.square(size_h))).to(self.device)
        self.nSamples = int((torch.sqrt(torch.sum(torch.square(size_h))) / step_h).item()) + 1
        # host copies of the (device-resident) geometry so that kernel launches never sync on .tolist()/.item();
        # every path that changes aabb / gridSize (constructor, shrink, upsample) ends in update_stepSize
        self._host_geom = {"grid": [int(g) for g in self.gridSize.tolist()], "lo": self.aabb[0].tolist(),
                           "hi": self.aabb[1].tolist(), "inv": self.invaabbSize.tolist(),
                           "step": float(self.stepSize)}

    def normalize_coord(self, xyz_sampled):
        return (xyz_sampled - self.aabb[0]) * self.invaabbSize - 1

    # ---- checkpoint (format of tensorBase_rotated_lights.py:646-692) -----------------
    def get_kwargs(self):
        kw = {'aabb': self.aabb, 'gridSize': self.gridSize.tolist(), 'density_n_comp': self.density_n_comp,
              'appearance_n_comp': self.app_n_comp, 'app_dim': self.app_dim, 'density_shift': self.density_shift,
              'alphaMask_thres': self.alphaMask_thres, 'distance_scale': self.distance_scale,
              'rayMarch_weight_thres': self.rayMarch_weight_thres, 'fea2denseAct': self.fea2denseAct,
              'near_far': self.near_far, 'step_ratio': self.step_ratio, 'shadingMode': self.shadingMode,
              'pos_pe': self.pos_pe, 'view_pe': self.view_pe, 'fea_pe': self.fea_pe, 'featureC': self.featureC,
              'normals_kind': self.normals_kind, 'light_num': self.light_num, 'light_kind': self.light_kind,
              'numLgtSGs': self.numLgtSGs}
        if self.general_lights:
            kw['light_name_list'] = self.light_name_list
        else:
            kw['light_rotation'] = self.light_rotation
        return kw

    def save(self, path):
        ckpt = {'kwargs': self.get_kwargs(), 'state_dict': self.state_dict()}
        if self.alphaMask is not None:
            alpha_volume = self.alphaMask.alpha_volume.bool().cpu().numpy()
            ckpt.update({'alphaMask.shape': alpha_volume.shape})
            ckpt.update({'alphaMask.mask': np.packbits(alpha_volume.reshape(-1))})
            ckpt.update({'alphaMask.aabb': self.alphaMask.aabb.cpu()})
        torch.save(ckpt, path)

    def load(self, ckpt):
        if 'alphaMask.aabb' in ckpt.keys():
            length = np.prod(ckpt['alphaMask.shape'])
            alpha_volume = torch.from_numpy(np.unpackbits(ckpt['alphaMask.mask'])[:length]
                                            .reshape(ckpt['alphaMask.shape']))
            self.alphaMask = AlphaGridMask(self.device, ckpt['alphaMask.aabb'].to(self.device),
                                           alpha_volume.float().to(self.device))
        self.load_state_dict(ckpt['state_dict'])

    # ---- point-wise queries (kernel-backed) ---------------------------------------------
    def feature2density(self, density_features):
        """tensorBase_rotated_lights.py:813-817."""
        if self.fea2denseAct == "softplus":
            return F.softplus(density_features + self.density_shift)
        return F.relu(density_features)

    @torch.no_grad()
    def compute_alpha(self, xyz_locs, length=1):
        """tensorBase_rotated_lights.py:819-837 via tir_alpha_mask_points + tir_density_points."""
        xyz_locs = xyz_locs.reshape(-1, 3)
        if self.alphaMask is not None:
            alpha_mask = ops.alpha_mask_points(self, xyz_locs)
        else:
            alpha_mask = torch.ones_like(xyz_locs[:, 0], dtype=bool)
        _, sigma = ops.density_points(self, self.normalize_coord(xyz_locs))
        sigma = torch.where(alpha_mask, sigma, torch.zeros_like(sigma))
        return 1 - torch.exp(-sigma * length)

    @torch.no_grad()
    def getDenseAlpha(self, gridSize=None):
        """tensorBase_rotated_lights.py:737-753 (one kernel call per slab, no Python-side masking)."""
        gridSize = self.gridSize if gridSize is None else gridSize
        gs = [int(g) for g in gridSize]
        samples = torch.stack(torch.meshgrid(torch.linspace(0, 1, gs[0]), torch.linspace(0, 1, gs[1]),
                                             torch.linspace(0, 1, gs[2]), indexing='ij'), -1).to(self.device)
        dense_xyz = self.aabb[0] * (1 - samples) + self.aabb[1] * samples
        alpha = torch.zeros_like(dense_xyz[..., 0])
        for i in range(gs[0]):
            alpha[i] = self.compute_alpha(dense_xyz[i].view(-1, 3), self.stepSize).view((gs[1], gs[2]))
        return alpha, dense_xyz

    @torch.no_grad()
    def updateAlphaMask(self, gridSize=(200, 200, 200)):
        """tensorBase_rotated_lights.py:755-779."""
        gridSize = tuple(int(g) for g in gridSize)
        alpha, dense_xyz = self.getDenseAlpha(gridSize)
        dense_xyz = dense_xyz.transpose(0, 2).contiguous()
        alpha = alpha.clamp(0, 1).transpose(0, 2).contiguous()[None, None]
        total_voxels = gridSize[0] * gridSize[1] * gridSize[2]
        alpha = F.max_pool3d(alpha, kernel_size=3, padding=1, stride=1).view(gridSize[::-1])
        alpha[alpha >= self.alphaMask_thres] = 1
        alpha[alpha < self.alphaMask_thres] = 0
        self.alphaMask = AlphaGridMask(self.device, self.aabb, alpha)
        valid_xyz = dense_xyz[alpha > 0.5]
        xyz_min, xyz_max = valid_xyz.amin(0), valid_xyz.amax(0)
        new_aabb = torch.stack((xyz_min, xyz_max))
        total = torch.sum(alpha)
        print(f"bbox: {xyz_min, xyz_max} alpha rest %%%f" % (total / total_voxels * 100))
        return new_aabb

    @torch.no_grad()
    def filtering_rays(self, all_rays, N_samples=256, chunk=10240 * 5, bbox_only=False):
        """tensorBase_rotated_lights.py:781-811."""
        print('========> filtering rays ...')
        tt = time.time()
        N = torch.tensor(all_rays.shape[:-1]).prod()
        mask_filtered = []
        for idx_chunk in torch.split(torch.arange(N), chunk):
            rays_chunk = all_rays[idx_chunk].to(self.device)
            rays_o, rays_d = rays_chunk[..., :3], rays_chunk[..., 3:6]
            if bbox_only:
                vec = torch.where(rays_d == 0, torch.full_like(rays_d, 1e-6), rays_d)
                rate_a = (self.aabb[1] - rays_o) / vec
                rate_b = (self.aabb[0] - rays_o) / vec
                t_min = torch.minimum(rate_a, rate_b).amax(-1)
                t_max = torch.maximum(rate_a, rate_b).amin(-1)
                mask_inbbox = t_max > t_min
            else:
                mask_inbbox = primary.any_sample_in_mask(self, rays_o, rays_d, N_samples)
            mask_filtered.append(mask_inbbox.cpu())
        mask_filtered = torch.cat(mask_filtered).view(all_rays.shape[:-1])
        print(f'Ray filtering done! takes {time.time() - tt} s. ray mask ratio: {torch.sum(mask_filtered) / N}')
        return all_rays[mask_filtered], mask_filtered

    def compute_relative_smoothness_loss(self, values, values_jittor):
        """tensorBase_rotated_lights.py:858-863."""
        base = torch.maximum(values, values_jittor).clip(min=1e-6)
        return torch.sum(((values - values_jittor) / base) ** 2, dim=-1, keepdim=True)

    # ---- the primary march ----------------------------------------------------------------
    def forward(self, rays_chunk, light_idx, white_bg=True, is_train=False, ndc_ray=False, is_relight=True,
                N_samples=-1):
        """TensorBase.forward (tensorBase_rotated_lights.py:868-1036) -> the reference's 12-tuple."""
        if ndc_ray:
            raise NotImplementedError("ndc_ray: no shipped TensoIR config uses NDC rays (SURVEY.md §2)")
        return primary.forward_relight(self, rays_chunk, light_idx, white_bg, is_train, is_relight, N_samples)
