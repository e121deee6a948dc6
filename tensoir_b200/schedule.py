"""The training schedule of the reference's ``reconstruction`` loop (train_tensoIR.py:110-424), on the host.

Everything the loop decides from the iteration number alone lives here: the learning rates of every optimizer param
group (one multiplication by ``lr_factor`` per iteration, :380-381, and a reset at each upsample, :416-422), the TV
weights (decayed *before* use, :276-285, zeroed when relighting starts, :398-399), the L1 weight (:219, :393), the
relight switch (:396), the normal / BRDF loss factors (:291-292), the voxel counts of the upsamples (:209-210), the
alpha-mask resolution rule (:387-388), the ray re-filter at the second mask update (:402-407) and the logging cadence
(:337, :350, :375).  The arithmetic is restated from the reference, in the same order and in Python floats, so the host
values are bit-identical to the reference's.

Two facts of the reference are kept as they are:

* when a mask update and an upsample fall on the same iteration, the mask block runs first (:385-422);
* a mask update keeps the optimizer (even after ``shrink`` rebinds the VM factors, :391); only an upsample makes a new
  one (:421-422).

Resolutions depend on the model's aabb after ``shrink`` (:412), which only the running model knows: the caller hands it
to :meth:`TrainSchedule.upsample`.
"""
from __future__ import annotations

from typing import Callable, List, NamedTuple, Sequence

import numpy as np
import torch


def n_to_reso(n_voxels, bbox) -> List[int]:
    """Grid resolution with ``n_voxels`` cubic voxels over ``bbox`` [2,3] (utils.py:58-61)."""
    xyz_min, xyz_max = bbox
    voxel_size = ((xyz_max - xyz_min).prod() / n_voxels).pow(1 / 3)
    return ((xyz_max - xyz_min) / voxel_size).long().tolist()


def cal_n_samples(reso, step_ratio=0.5) -> int:
    """Samples per ray for a grid of ``reso`` (utils.py:63-64)."""
    return int(np.linalg.norm(reso) / step_ratio)


class SimpleSampler:
    """Batches of ray ids, a fresh ``np.random.permutation`` whenever the next batch would run past the end
    (train_tensoIR.py:36-48).  Draws from numpy's global stream, like the reference."""

    def __init__(self, total, batch):
        self.total, self.batch = int(total), int(batch)
        self.curr = self.total
        self.ids = None

    def nextids(self):
        self.curr += self.batch
        if self.curr + self.batch > self.total:
            self.ids = torch.LongTensor(np.random.permutation(self.total))
            self.curr = 0
        return self.ids[self.curr:self.curr + self.batch]


class StepWeights(NamedTuple):
    """What one training iteration uses."""
    lrs: tuple               # learning rate of every param group of the current optimizer
    tv_density: float        # weight of TV_loss_density (0: the term is not in the loss)
    tv_app: float
    l1: float                # weight of density_L1 (0: not in the loss)
    relight: bool            # phase 2: the relight step with secondary rays and the BRDF losses
    normal_factor: float     # multiplies normals_diff_weight / normals_orientation_weight (relight only)
    brdf_factor: float       # multiplies roughness / albedo smoothness weights (relight only)
    n_samples: int


class MaskUpdate(NamedTuple):
    """``updateAlphaMask(reso)``; at the first entry also ``shrink`` and the switch to relighting, at the second a
    ``filtering_rays(bbox_only=True)`` of the training rays and a new sampler."""
    reso: tuple
    shrink: bool
    refilter: bool


class Upsample(NamedTuple):
    """``upsample_volume_grid`` to ``n_voxels`` voxels (resolved by :meth:`TrainSchedule.upsample` on the model's
    aabb), then a new optimizer from ``get_optparam_groups(lr, lr_basis)``."""
    n_voxels: int
    lr: float
    lr_basis: float


class StepEnd(NamedTuple):
    """What the loop does after the optimizer step of one iteration, in the reference's order."""
    progress: bool           # print the progress line (:337)
    evaluate: bool           # evaluation_iter_TensoIR into imgs_vis/ (:350)
    save: bool               # checkpoints/{expname}_{it}.th (:375)
    grid: tuple              # MaskUpdate / Upsample events, mask block first (:385-422)


class TrainSchedule:
    """Host-only state of the reference's loop.  Call :meth:`begin` before and :meth:`end` after the step of every
    iteration 0, 1, ..., ``n_iters - 1`` in order, and :meth:`upsample` for each :class:`Upsample` that ``end``
    returns.

    ``aabb``: the scene bbox the initial resolution is computed on (:159-160).  ``group_lrs(lr, lr_basis)``: the
    learning rates of the param groups ``get_optparam_groups(lr, lr_basis)`` makes (some groups of the model have a
    fixed rate), in group order."""

    def __init__(self, args, aabb, group_lrs: Callable[[float, float], Sequence[float]]):
        self.args = args
        self.n_iters = int(args.n_iters)
        decay_iters = args.lr_decay_iters if args.lr_decay_iters > 0 else args.n_iters
        self.lr_factor = args.lr_decay_target_ratio ** (1 / decay_iters)                     # :197-201
        self.upsamp_list = list(args.upsamp_list or [])
        self.mask_list = list(args.update_AlphaMask_list or [])
        self.n_voxel_list = (torch.round(torch.exp(torch.linspace(
            np.log(args.N_voxel_init), np.log(args.N_voxel_final), len(self.upsamp_list) + 1))).long()).tolist()[1:]
        self._group_lrs = group_lrs
        self.lrs = [float(v) for v in group_lrs(args.lr_init, args.lr_basis)]              # :196
        self.reso_cur = n_to_reso(args.N_voxel_init, aabb)                                   # :160
        self.n_samples = min(args.nSamples, cal_n_samples(self.reso_cur, args.step_ratio))  # :161
        self.reso_mask = None
        self.tv_density, self.tv_app = args.TV_weight_density, args.TV_weight_app           # :221
        self.l1 = args.L1_weight_inital                                                      # :219
        self.relight = False
        self._pending = list(self.n_voxel_list)
        self._next = 0

    def begin(self, it: int) -> StepWeights:
        if it != self._next:
            raise ValueError(f"TrainSchedule.begin({it}): expected iteration {self._next}")
        a = self.args
        if self.tv_density > 0:                     # decayed before use (:276-285)
            self.tv_density *= self.lr_factor
        if self.tv_app > 0:
            self.tv_app *= self.lr_factor
        nwf = bwf = 0.0
        if self.relight:                            # :291-292
            m0 = self.mask_list[0]
            nwf = a.normals_loss_enhance_ratio ** ((it - m0) / (a.n_iters - m0))
            bwf = a.BRDF_loss_enhance_ratio ** ((it - m0) / (a.n_iters - m0))
        return StepWeights(tuple(self.lrs), self.tv_density, self.tv_app, self.l1, self.relight, nwf, bwf,
                           self.n_samples)

    def end(self, it: int) -> StepEnd:
        if it != self._next:
            raise ValueError(f"TrainSchedule.end({it}): expected iteration {self._next}")
        self._next += 1
        a = self.args
        progress = it % a.progress_refresh_rate == 0
        evaluate = it % a.vis_every == a.vis_every - 1 and a.N_vis != 0 and self.relight
        save = it % a.save_iters == 0
        self.lrs = [lr * self.lr_factor for lr in self.lrs]                                  # :380-381
        grid = []
        if it in self.mask_list:                                                             # :385-407
            if self.reso_cur[0] * self.reso_cur[1] * self.reso_cur[2] < 256 ** 3:
                self.reso_mask = self.reso_cur
            if self.reso_mask is None:
                raise ValueError(f"update_AlphaMask_list entry {it}: the grid {self.reso_cur} has 256^3 voxels or "
                                 "more and no earlier mask resolution exists")
            first = it == self.mask_list[0]
            if first:
                self.l1 = a.L1_weight_rest
                self.relight = True
                self.tv_density = self.tv_app = 0
            refilter = not a.ndc_ray and len(self.mask_list) > 1 and it == self.mask_list[1]
            grid.append(MaskUpdate(tuple(self.reso_mask), first, refilter))
        if it in self.upsamp_list:                                                           # :410-422
            n_voxels = self._pending.pop(0)
            lr_scale = 1 if a.lr_upsample_reset else a.lr_decay_target_ratio ** (it / a.n_iters)
            lr, lr_basis = a.lr_init * lr_scale, a.lr_basis * lr_scale
            self.lrs = [float(v) for v in self._group_lrs(lr, lr_basis)]
            grid.append(Upsample(n_voxels, lr, lr_basis))
        return StepEnd(progress, evaluate, save, tuple(grid))

    def upsample(self, event: Upsample, aabb) -> List[int]:
        """Resolution of ``event`` on the model's current ``aabb`` (:412-413); updates ``reso_cur`` and
        ``n_samples``."""
        self.reso_cur = n_to_reso(event.n_voxels, aabb)
        self.n_samples = min(self.args.nSamples, cal_n_samples(self.reso_cur, self.args.step_ratio))
        return self.reso_cur
