"""TensorVMSplit of models/tensoRF_init.py:139-305 on TensorBase_Init (models/tensorBase_init.py:136-462):
the light-free TensoRF-heritage model used by BASELINE config 1 and OctreeRender_trilinear_fast."""
from __future__ import annotations

import torch

from . import primary, vm_autograd
from .tensorbase import MLPRender_Fea
from .tensorf import TensorVMSplit as _RelightVMSplit


class TensorVMSplit(_RelightVMSplit):
    def __init__(self, aabb, gridSize, device, density_n_comp=8, appearance_n_comp=24, app_dim=27,
                 shadingMode='MLP_PE', alphaMask=None, near_far=[2.0, 6.0], density_shift=-10,
                 alphaMask_thres=0.001, distance_scale=25, rayMarch_weight_thres=0.0001, pos_pe=6, view_pe=6,
                 fea_pe=6, featureC=128, step_ratio=2.0, fea2denseAct='softplus'):
        torch.nn.Module.__init__(self)
        self.density_n_comp, self.app_n_comp, self.app_dim = density_n_comp, appearance_n_comp, app_dim
        self.aabb, self.alphaMask, self.device = aabb, alphaMask, device
        self.density_shift, self.alphaMask_thres, self.distance_scale = density_shift, alphaMask_thres, distance_scale
        self.rayMarch_weight_thres, self.fea2denseAct = rayMarch_weight_thres, fea2denseAct
        self.near_far, self.step_ratio = near_far, step_ratio
        self.light_num = 0
        self.update_stepSize(gridSize)
        self.matMode, self.vecMode, self.comp_w = [[0, 1], [0, 2], [1, 2]], [2, 1, 0], [1, 1, 1]
        self.init_svd_volume(gridSize[0], device)
        self.shadingMode, self.pos_pe, self.view_pe, self.fea_pe, self.featureC = \
            shadingMode, pos_pe, view_pe, fea_pe, featureC
        if shadingMode != 'MLP_Fea':
            raise NotImplementedError(f"shadingMode {shadingMode!r}: only 'MLP_Fea' is on the CUDA hot path")
        self.renderModule = MLPRender_Fea(self.app_dim, view_pe, fea_pe, featureC).to(device)

    def init_svd_volume(self, res, device):
        """tensoRF_init.py:144-147 (no light_line)."""
        self.density_plane, self.density_line = self.init_one_svd(self.density_n_comp, self.gridSize, 0.1, device)
        self.app_plane, self.app_line = self.init_one_svd(self.app_n_comp, self.gridSize, 0.1, device)
        self.basis_mat = torch.nn.Linear(sum(self.app_n_comp), self.app_dim, bias=False).to(device)

    def get_kwargs(self):
        return {'aabb': self.aabb, 'gridSize': self.gridSize.tolist(), 'density_n_comp': self.density_n_comp,
                'appearance_n_comp': self.app_n_comp, 'app_dim': self.app_dim, 'density_shift': self.density_shift,
                'alphaMask_thres': self.alphaMask_thres, 'distance_scale': self.distance_scale,
                'rayMarch_weight_thres': self.rayMarch_weight_thres, 'fea2denseAct': self.fea2denseAct,
                'near_far': self.near_far, 'step_ratio': self.step_ratio, 'shadingMode': self.shadingMode,
                'pos_pe': self.pos_pe, 'view_pe': self.view_pe, 'fea_pe': self.fea_pe, 'featureC': self.featureC}

    def TV_loss_density(self, reg):
        """tensoRF_init.py:188-192 (includes the line term)."""
        total = 0
        for idx in range(len(self.density_plane)):
            total = total + reg(self.density_plane[idx]) * 1e-2 + reg(self.density_line[idx]) * 1e-3
        return total

    def TV_loss_app(self, reg):
        total = 0
        for idx in range(len(self.app_plane)):
            total = total + reg(self.app_plane[idx]) * 1e-2 + reg(self.app_line[idx]) * 1e-3
        return total

    def compute_appfeature(self, xyz_sampled, light_idx=None):
        """tensoRF_init.py:222-236."""
        return self.basis_mat(vm_autograd.app_products(self, xyz_sampled))

    def forward(self, rays_chunk, white_bg=True, is_train=False, ndc_ray=False, N_samples=-1):
        """tensorBase_init.py:406-462 -> (rgb_map, depth_map)."""
        if ndc_ray:
            raise NotImplementedError("ndc_ray is not on the TensoIR hot path")
        return primary.forward_init(self, rays_chunk, white_bg, is_train, N_samples)
