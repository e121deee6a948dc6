"""Native trainer: the reference's ``reconstruction`` loop (train_tensoIR.py:110-424) on CUDA-graph-replayed steps.

The schedule (learning rates, loss weights, grid events, logging cadence) is :class:`schedule.TrainSchedule`; the steps
are :class:`static_step.StaticTrainStep` captures: the radiance-only step (``is_relight=False``) until the first
``update_AlphaMask_list`` entry, the relight step with the loss of :262-312 after it.  Between two grid events every
iteration is one graph replay plus its input copies; nothing on the per-step path reads a device value back.

* Every value the schedule changes between replays lives in device memory: the param groups' learning rates and the
  TV / normal / BRDF weights are 0-dim views of one device vector.  The step stages each iteration's float64 host
  values into it with one host-to-device copy (``run(..., scalars=...)``), again when it redoes the iteration.  The L1
  term is folded into :class:`optim.FusedAdam` (``density_l1``).
* Batches come from the reference's :class:`schedule.SimpleSampler` on numpy's global stream, gathered on the host
  into a ring of pinned buffers.
* The host randoms of iteration ``it`` (per-ray jitter, stratified light directions) are drawn right after
  ``torch.manual_seed(SEED + it)``, in both modes (and again for a redone step), so the eager run (``graphed=False``) consumes the same host draws as
  the graphed one.  The graphed step draws the xyz noise of the smoothness terms on the device with the padded list
  shape (static_step.py), so the two runs are not one random trajectory, and neither reproduces the reference run's
  random stream.
* The loss terms of each step are copied into a device ring after each of its replays; the host flushes the step and
  reads the ring once per ``progress_refresh_rate`` iterations for the progress line and the TensorBoard scalars.  A
  step that overflowed its static lists, and every step launched after it, is a no-op replay and is redone in order on
  the same batch (static_step.py); the redo rewrites the step's ring row, so the log holds the applied replay.
* At a grid event: ``flush``, ``release``, the grid operation, a new optimizer when the reference makes one (only at an
  upsample; a mask update keeps it, :385-422), then a newly calibrated and captured step.  An evaluation or a
  checkpoint first flushes; an evaluation runs eager forwards on the model, so the step is captured again after it.

``graphed=False`` runs the same schedule with the eager ``Renderer_TensoIR_train`` and ``torch.optim.Adam``: it is the
reference the GPU tests compare the graphed run against, not a user option.

One loop serves the reference's four training scripts; ``variant`` (the names of ``evaluation._evaluate``) picks only
the model's light kwargs, the evaluation function and the final evaluation block:

* ``"full"``: train_tensoIR.py, and train_tensoIR_rotated_multi_lights.py, which is the same loop.
* ``"general"``: train_tensoIR_general_multi_lights.py.  The model gets ``light_name_list``; evaluations go through
  ``evaluation_iter_TensoIR_general_multi_lights``, whose per-view ``np.random.randint(light_num)`` draws come from the
  numpy stream the sampler permutes with, between the same two sampler calls as in the reference; the final evaluation
  runs once per light into ``imgs_test_all/{light_name}/``.
* ``"simple"``: train_tensoIR_simple.py (NeRF-synthetic scenes): ``evaluation_iter_TensoIR_simple``, no MAE or albedo
  metrics.

:func:`render_test` is the scripts' ``--render_only 1 --render_test 1`` path on a checkpoint, and :func:`main` their
``__main__`` block (mesh export, then rendering or training).
"""
from __future__ import annotations

import datetime
import gc
import os
import random
import shutil
import sys
import time

import numpy as np
import torch

from . import evaluation
from .optim import FusedAdam
from .renderer import Renderer_TensoIR_train
from .schedule import MaskUpdate, SimpleSampler, TrainSchedule, n_to_reso
from .static_step import StaticTrainStep
from .tensorf import TensorVMSplit

SEED = 20211202
RING = 8                  # pinned batch buffers: more than the lag + 1 steps a redo can reach back
# loss terms of one step, in this order, in the device log ring
TERMS = ("total", "mse_rgb", "mse_rgb_brdf", "tv_density", "tv_app", "normals_diff", "normals_orientation",
         "roughness_smoothness", "albedo_smoothness")


class TVLoss(torch.nn.Module):
    """The TV regulariser object the train loop hands to ``TV_loss_*`` (utils.py:143-162): with its
    ``TVLoss_weight`` attribute, tv.tv_planes runs the fused kernels."""

    def __init__(self, TVLoss_weight=1):
        super().__init__()
        self.TVLoss_weight = TVLoss_weight


VARIANTS = ("full", "general", "simple")


def _reject_render_path(args):
    if getattr(args, "render_path", 0):
        raise ValueError("render_path: the reference scripts have no camera-path rendering (their render_path block is "
                         "commented out); use --render_only 1 --render_test 1 to render the test views")


def check_supported(args, variant="full", train_dataset=None):
    """Reject what the native trainer does not run, before any work is done.  With ``train_dataset``, a general run's
    ``light_name_list`` must name one light per light of the training set (its ``light_num``)."""
    if variant not in VARIANTS:
        raise ValueError(f"variant {variant!r}: expected one of {VARIANTS}")
    _reject_render_path(args)
    if variant == "general":
        names = list(args.light_name_list or [])
        if not names:
            raise ValueError("the general multi-light trainer needs light_name_list (one name per training light)")
        n = getattr(train_dataset, "light_num", None)
        if train_dataset is not None and n != len(names):
            raise ValueError(f"light_name_list {names} names {len(names)} lights; the training set has "
                             f"light_num = {n}")
    if args.ndc_ray:
        raise ValueError("ndc_ray: the native trainer supports the synthetic (non-NDC) scenes only")
    if args.model_name != "TensorVMSplit" or args.shadingMode != "MLP_Fea":
        raise ValueError(f"model {args.model_name!r} / shadingMode {args.shadingMode!r}: the native trainer runs "
                         "TensorVMSplit with shadingMode MLP_Fea only")
    masks = list(args.update_AlphaMask_list or [])
    if not masks or masks[0] >= args.n_iters:
        raise ValueError(f"update_AlphaMask_list {masks}: its first entry must come before n_iters ({args.n_iters}), "
                         "where relighting starts")
    if args.Ortho_weight > 0:
        raise ValueError("Ortho_weight > 0: the native trainer has no vector_comp_diffs term")


class _Rays:
    """The filtered training rays on the host, the reference's sampler, and a ring of pinned batch buffers."""

    def __init__(self, dataset, batch):
        self.all = (dataset.all_rays, dataset.all_rgbs, dataset.all_light_idx)
        self.batch = int(batch)
        self.ring = [(torch.empty(batch, 6).pin_memory(), torch.empty(batch, 3).pin_memory(),
                      torch.empty(batch, 1, dtype=torch.int32).pin_memory()) for _ in range(RING)]
        self.k = 0

    def filter(self, model):
        """:228-231 / :404-407: keep the rays that meet the model's aabb, new sampler."""
        all_rays, all_rgbs, all_li = self.all
        self.rays, mask = model.filtering_rays(all_rays, bbox_only=True)
        self.rays = self.rays.float().contiguous()
        self.rgbs = all_rgbs[mask, :].float().contiguous()
        self.li = all_li[mask, :].to(torch.int32).contiguous()
        self.sampler = SimpleSampler(self.rays.shape[0], self.batch)

    def next(self):
        ids = self.sampler.nextids()
        rays, rgb, li = self.ring[self.k % RING]
        self.k += 1
        torch.index_select(self.rays, 0, ids, out=rays)
        torch.index_select(self.rgbs, 0, ids, out=rgb)
        torch.index_select(self.li, 0, ids, out=li)
        return rays, rgb, li

    def calibration_batches(self, n=4):
        """Random batches for sizing the static lists, drawn without touching the sampler's numpy stream."""
        g = torch.Generator().manual_seed(SEED)
        ids = [torch.randint(0, self.rays.shape[0], (self.batch,), generator=g) for _ in range(n)]
        return [(self.rays[i], self.li[i]) for i in ids]


def _load_model(path, device):
    """The checkpoint at ``path`` (:163-168); its kwargs carry the light_name_list of a general model."""
    ckpt = torch.load(path, map_location=device, weights_only=False)
    kwargs = ckpt['kwargs']
    kwargs.update({'device': device})
    model = TensorVMSplit(**kwargs)
    model.load(ckpt)
    return model


def _new_model(args, train_dataset, device, variant="full"):
    if args.ckpt is not None:                                                                # :163-168
        return _load_model(args.ckpt, device)
    aabb = train_dataset.scene_bbox.to(device)
    # the general script adds light_name_list (train_tensoIR_general_multi_lights.py:223)
    lights = {"light_name_list": args.light_name_list} if variant == "general" else {}
    return TensorVMSplit(aabb, n_to_reso(args.N_voxel_init, aabb), device,                 # :170-192
                         density_n_comp=args.n_lamb_sigma, appearance_n_comp=args.n_lamb_sh,
                         app_dim=args.data_dim_color, near_far=train_dataset.near_far, shadingMode=args.shadingMode,
                         alphaMask_thres=args.alpha_mask_thre, density_shift=args.density_shift,
                         distance_scale=args.distance_scale, pos_pe=args.pos_pe, view_pe=args.view_pe,
                         fea_pe=args.fea_pe, featureC=args.featureC, step_ratio=args.step_ratio,
                         fea2denseAct=args.fea2denseAct, normals_kind=args.normals_kind,
                         light_rotation=args.light_rotation, light_kind=args.light_kind, dataset=train_dataset,
                         numLgtSGs=args.numLgtSGs, **lights)


def _loss(args, ret, target, model, w, relight, terms):
    """:262-312 with ``w`` = (tv_density, tv_app, normal_factor, brdf_factor) as floats (eager) or 0-dim device
    tensors (graphed); the L1 term is added by the caller or folded into FusedAdam.  Sets ``terms[0]`` to the
    vector of TERMS, computed with the loss (inside the graph when captured, so every replay refreshes it)."""
    tv_d, tv_a, nwf, bwf = w
    zero = torch.zeros((), device=target.device)
    t = dict.fromkeys(TERMS[1:], zero)
    t["mse_rgb"] = torch.mean((ret['rgb_map'] - target) ** 2)
    total = t["mse_rgb"]
    if not relight:
        if args.TV_weight_density > 0:
            t["tv_density"] = model.TV_loss_density(_TV) * tv_d
            total = total + t["tv_density"]
        if args.TV_weight_app > 0:
            t["tv_app"] = model.TV_loss_app(_TV) * tv_a
            total = total + t["tv_app"]
    else:
        t["mse_rgb_brdf"] = torch.mean((ret['rgb_with_brdf_map'] - target) ** 2)
        total = total + t["mse_rgb_brdf"] * args.rgb_brdf_weight
        for key, weight, factor, value in (
                ("normals_diff", args.normals_diff_weight, nwf, lambda: ret['normals_diff_map'].mean()),
                ("normals_orientation", args.normals_orientation_weight, nwf,
                 lambda: ret['normals_orientation_loss_map'].mean()),
                ("roughness_smoothness", args.roughness_smoothness_loss_weight, bwf,
                 lambda: ret['roughness_smoothness_loss']),
                ("albedo_smoothness", args.albedo_smoothness_loss_weight, bwf, lambda: ret['albedo_smoothness_loss'])):
            if weight > 0:
                t[key] = factor * weight * value()
                total = total + t[key]
    terms[:] = [torch.stack([total] + [t[k] for k in TERMS[1:]]).detach()]
    return total


_TV = TVLoss()


def _progress_line(it, psnr_rgb, psnr_brdf, psnr_test, psnr_brdf_test, mse):
    """The reference's progress description (:338-345)."""
    return (f'Iteration {it:05d} PSNR:'
            + f' train_rgb = {float(np.mean(psnr_rgb)):.2f}'
            + f' train_rgb_brdf = {float(np.mean(psnr_brdf)):.2f}'
            + f' test_rgb = {float(np.mean(psnr_test)):.2f}'
            + f' test_rgb_brdf = {float(np.mean(psnr_brdf_test)):.2f}'
            + f' mse = {float(mse):.6f}')


def _summary_writer(logfolder):
    try:
        from torch.utils.tensorboard import SummaryWriter
    except ImportError:
        return None
    return SummaryWriter(logfolder)


class _Timer:
    def __init__(self):
        self.t = {}

    def add(self, key, seconds):
        self.t[key] = self.t.get(key, 0.0) + seconds


# the evaluation each script calls (:350-353; general :388, simple :362)
_EVAL = {"full": evaluation.evaluation_iter_TensoIR, "general": evaluation.evaluation_iter_TensoIR_general_multi_lights,
         "simple": evaluation.evaluation_iter_TensoIR_simple}


def _five(r):
    """An evaluation's result as (psnr, psnr_brdf, mae, psnr_albedo_single, psnr_albedo_three); the simple
    evaluation has no MAE or albedo metrics (None)."""
    return tuple(r) + (None,) * (5 - len(r))


def _metric_tags(variant, suffix, psnr, psnr_brdf, mae, pa1, pa3):
    """The test scalars a script logs (:366-372 / :449-453; the simple script drops MAE and the albedo PSNRs)."""
    tags = [('test/psnr_rgb', np.mean(psnr)), ('test/psnr_rgb_brdf', np.mean(psnr_brdf))]
    if variant != "simple":
        tags += [('test/mae', mae), ('test/psnr_albedo_single', pa1), ('test/psnr_albedo_three', pa3)]
    return [(t + suffix, v) for t, v in tags]


def _test_all(variant, test_dataset, model, args, savedir, device, white_bg=True):
    """The final evaluation of every test view into ``savedir`` (:433-453), once per light into
    ``{savedir}{light_name}/`` for the general model (general script :470-491) -> the 5-tuple of :func:`_five`.  For
    the general model the two PSNRs are the means over lights of the per-light means, and MAE and the albedo PSNRs are
    those of the last light, as the reference prints them."""
    kw = dict(N_samples=-1, white_bg=white_bg, ndc_ray=False, device=device, test_all=True)
    if variant != "general":
        return _five(_EVAL[variant](test_dataset, model, args, Renderer_TensoIR_train, savedir, **kw))
    psnr, psnr_brdf = [], []
    for light, name in enumerate(model.light_name_list):
        os.makedirs(f'{savedir}{name}', exist_ok=True)
        p, pb, mae, pa1, pa3 = evaluation.evaluation_iter_TensoIR_general_multi_lights(
            test_dataset, model, args, Renderer_TensoIR_train, f'{savedir}{name}/', light_idx_to_test=light, **kw)
        psnr.append(np.mean(p))
        psnr_brdf.append(np.mean(pb))
    return np.mean(psnr), np.mean(psnr_brdf), mae, pa1, pa3


def _device(args, device):
    return torch.device(device or (f"cuda:{args.local_rank}" if torch.cuda.is_available() else "cpu"))


def reconstruction(args, train_dataset, test_dataset, logfolder, *, variant="full", graphed=True, device=None,
                   out=sys.stdout):
    """Train ``args`` (the reference's option namespace, opt.config_parser) on ``train_dataset`` and evaluate on
    ``test_dataset`` (the reference's dataset contracts), writing into ``logfolder`` what the ``variant``'s script
    writes: ``checkpoints/{expname}_{it}.th``, ``imgs_vis/``, ``{expname}.th``, ``imgs_test_all/`` (with
    ``render_test``; one subfolder per light for ``general``) and TensorBoard scalars when tensorboard is importable.

    Returns a dict: ``losses`` [n_iters, len(TERMS)] (float32, read from the device ring), ``events`` (the grid, save
    and evaluation calls, in order, as ``(iteration, name, ...)``), ``redone`` / ``recaptures`` of the captured steps,
    ``psnr_test`` of the final evaluation and ``times`` (seconds per phase, per event kind, evaluation)."""
    check_supported(args, variant, train_dataset)
    if not train_dataset.white_bg:
        raise ValueError("the training step renders over a white background; this dataset has white_bg = False")
    dev = _device(args, device)
    if dev.type != "cuda":
        raise RuntimeError("the native trainer needs a CUDA device")
    os.makedirs(f'{logfolder}/imgs_vis', exist_ok=True)
    os.makedirs(f'{logfolder}/checkpoints', exist_ok=True)
    writer = _summary_writer(logfolder)
    if getattr(args, "config", None):
        shutil.copy(args.config, logfolder)

    model = _new_model(args, train_dataset, dev, variant)
    events = []
    timer = _Timer()
    sched = TrainSchedule(args, train_dataset.scene_bbox.to(dev),
                          lambda lr, lr_basis: [g['lr'] for g in model.get_optparam_groups(lr, lr_basis)])
    n_groups = len(sched.lrs)
    rays = _Rays(train_dataset, args.batch_size)
    rays.filter(model)

    # per-iteration host values -> one device vector: [lr of each group, tv_density, tv_app, normal, brdf factor]
    scal = torch.zeros(n_groups + 4, device=dev)
    w_dev = tuple(scal[n_groups + k] for k in range(4))
    ring = torch.zeros(args.progress_refresh_rate, len(TERMS), device=dev)
    losses = torch.zeros(args.n_iters, len(TERMS))
    terms = []
    # one capture stream for every step of the run: the autograd nodes that accumulate into the parameters outlive a
    # step (the graphs of captured outputs hold them) and remember the stream they were made on; a later capture's
    # backward must not wait on a different stream
    capture_stream = torch.cuda.Stream(dev)

    def optimizer(lr, lr_basis):
        groups = model.get_optparam_groups(lr, lr_basis)
        if not graphed:
            return torch.optim.Adam(groups, betas=(0.9, 0.99))
        for k, g in enumerate(groups):
            g['lr'] = scal[k]
        return FusedAdam(groups, betas=(0.9, 0.99))

    def new_step(opt, w):
        opt.density_l1(model, w.l1)
        # before the first mask update there is no alpha mask, and the appearance list grows several-fold within a few
        # steps while the density forms: the radiance-only step gets lists that cannot overflow (n_rays * n_samples)
        full = None if w.relight else args.batch_size * w.n_samples
        st = StaticTrainStep(model, opt, args.batch_size, w.n_samples, args,
                             lambda ret, m: _loss(args, ret, st.target, m, w_dev, w.relight, terms),
                             sample_method=args.light_sample_train, device=dev, is_relight=w.relight,
                             cap_valid=full, cap_app=full)
        if w.relight:
            st.calibrate(rays.calibration_batches(), headroom=4.0)
        gc.collect()                             # nothing left for the collector to free during the capture
        st._stream = capture_stream
        st.capture(warmup=1)
        return st

    opt = optimizer(args.lr_init, args.lr_basis)
    st = None
    totals = {"redone": 0, "recaptures": 0}
    relit = np.zeros(args.n_iters, dtype=bool)
    psnr_test, psnr_brdf_test = [0], [0]
    since = 0                    # first iteration of the current progress window (:323-347)
    read = 0                     # first iteration whose ring row has not been read yet
    rate = args.progress_refresh_rate

    def sync_time():
        torch.cuda.synchronize(dev)
        return time.perf_counter()

    def read_ring(upto):
        nonlocal read
        if st is not None:
            st.flush()                           # a redo rewrites its step's row
        rows = ring.cpu()                        # the one host sync of the logging path
        for i in range(read, upto + 1):
            losses[i] = rows[i % rate]
            if writer is not None:
                _write_scalars(writer, i, losses[i], relit[i])
        read = upto + 1

    def retire(where):
        """Settle the captured step's in-flight replays and drop it (grid event / end of training)."""
        nonlocal st
        st.flush()
        totals["redone"] += st.redone
        totals["recaptures"] += st.recaptures
        out.write(f"{where}: redone {st.redone}, recaptures {st.recaptures}\n")
        st.release()
        # free the graph now: the step and its loss closure form a reference cycle, and a graph destroyed by the
        # garbage collector in the middle of the next capture aborts that capture
        st.graph = st.loss_fn = None
        st = None

    phase_t0 = sync_time()
    for it in range(args.n_iters):
        w = sched.begin(it)
        relit[it] = w.relight
        timer.add("phase2_iters" if w.relight else "phase1_iters", 1)
        batch_rays, batch_rgb, batch_li = rays.next()
        if graphed:
            if st is None:
                t0 = sync_time()
                st = new_step(opt, w)
                timer.add("capture", sync_time() - t0)
                phase_t0 += time.perf_counter() - t0
            host = torch.tensor(list(w.lrs) + [w.tv_density, w.tv_app, w.normal_factor, w.brdf_factor],
                                dtype=torch.float64)
            # terms[0]: the vector of the graph captured last (re-captures included)
            st.run(batch_rays, batch_li, batch_rgb, seed=SEED + it, scalars=(scal, host),
                   after=lambda row=ring[it % rate]: row.copy_(terms[0]))
        else:
            for g, lr in zip(opt.param_groups, w.lrs):
                g['lr'] = lr
            rd, rgb, li = (t.to(dev) for t in (batch_rays, batch_rgb, batch_li))
            torch.manual_seed(SEED + it)
            ret = Renderer_TensoIR_train(rd, None, li, model, N_samples=w.n_samples, white_bg=True,
                                         ndc_ray=False, device=dev, sample_method=args.light_sample_train,
                                         chunk_size=args.relight_chunk_size, is_train=True, is_relight=w.relight,
                                         args=args)
            loss = _loss(args, ret, rgb, model, (w.tv_density, w.tv_app, w.normal_factor, w.brdf_factor),
                         w.relight, terms)
            if w.l1 > 0:
                loss = loss + w.l1 * model.density_L1()
            opt.zero_grad()
            loss.backward()
            opt.step()
            ring[it % rate].copy_(terms[0])

        end = sched.end(it)
        if (it + 1 - read == rate or end.progress or end.evaluate or end.save or end.grid
                or it == args.n_iters - 1):
            read_ring(it)
        if end.progress:
            window = losses[since:it + 1]
            psnr_rgb = [-10.0 * np.log(float(r[1])) / np.log(10.0) for r in window]
            psnr_brdf = [-10.0 * np.log(float(r[2])) / np.log(10.0) if relit[since + k] else 0.0
                         for k, r in enumerate(window)]
            out.write(_progress_line(it, psnr_rgb, psnr_brdf, psnr_test, psnr_brdf_test, losses[it, 0]) + "\n")
            since = it + 1
        if end.evaluate:                                                                     # :350-372
            t0 = sync_time()
            if st is not None:
                st.flush()
                st.release()
            # the general evaluation draws one light per view from numpy's global stream, after this iteration's
            # sampler call and before the next one's, as in the reference
            psnr_test, psnr_brdf_test, mae, pa1, pa3 = _five(_EVAL[variant](
                test_dataset, model, args, Renderer_TensoIR_train, f'{logfolder}/imgs_vis/', prtx=f'{it:06d}_',
                N_samples=w.n_samples, white_bg=True, ndc_ray=False, compute_extra_metrics=False,
                logger=writer, step=it, device=dev))
            events.append((it, "evaluation", "imgs_vis", f'{it:06d}_', int(w.n_samples), False, False))
            if writer is not None:
                for tag, v in _metric_tags(variant, '', psnr_test, psnr_brdf_test, mae, pa1, pa3):
                    writer.add_scalar(tag, v, global_step=it)
            if st is not None and not end.grid:
                st.capture(warmup=1)             # the eager forwards may have re-sized buffers the graph points into
            dt = sync_time() - t0
            timer.add("evaluation", dt)
            phase_t0 += dt                       # step times exclude evaluations and checkpoints
        if end.save:                                                                         # :375-376
            t0 = sync_time()
            if st is not None:
                st.flush()
            name = f'checkpoints/{args.expname}_{it}.th'
            model.save(f'{logfolder}/{name}')
            events.append((it, "save", name))
            dt = sync_time() - t0
            timer.add("save", dt)
            phase_t0 += dt
        if end.grid:
            if st is not None:
                retire(f"iteration {it}")
            timer.add("phase2_steps" if w.relight else "phase1_steps", sync_time() - phase_t0)
            for ev in end.grid:
                t0 = sync_time()
                if isinstance(ev, MaskUpdate):                                               # :385-407
                    new_aabb = model.updateAlphaMask(ev.reso)
                    events.append((it, "updateAlphaMask", list(ev.reso)))
                    if ev.shrink:
                        model.shrink(new_aabb)
                        events.append((it, "shrink"))
                    timer.add("mask_update", sync_time() - t0)
                    if ev.refilter:
                        t0 = sync_time()
                        rays.filter(model)
                        events.append((it, "filtering_rays", True))
                        timer.add("refilter", sync_time() - t0)
                else:                                                                        # :410-422
                    reso = sched.upsample(ev, model.aabb)
                    model.upsample_volume_grid(reso)
                    events.append((it, "upsample_volume_grid", list(reso)))
                    events.append((it, "get_optparam_groups", ev.lr, ev.lr_basis))
                    opt = optimizer(ev.lr, ev.lr_basis)
                    timer.add("upsample", sync_time() - t0)
            phase_t0 = sync_time()
    if st is not None:
        retire("end of training")
    timer.add("phase2_steps" if w.relight else "phase1_steps", sync_time() - phase_t0)
    final = f'{args.expname}.th'
    model.save(f'{logfolder}/{final}')                                                      # :424
    events.append((args.n_iters - 1, "save", final))
    res = {"losses": losses, "events": events, "psnr_test": None, "model": model, "relight": relit, **totals}
    if args.render_test:                                                                     # :433-453
        t0 = sync_time()
        os.makedirs(f'{logfolder}/imgs_test_all', exist_ok=True)
        psnr_test, psnr_brdf_test, mae, pa1, pa3 = _test_all(variant, test_dataset, model, args,
                                                             f'{logfolder}/imgs_test_all/', dev)
        events.append((args.n_iters - 1, "evaluation", "imgs_test_all", '', -1, True, True))
        res["psnr_test"] = float(np.mean(psnr_test))
        if writer is not None:
            for tag, v in _metric_tags(variant, '_all', psnr_test, psnr_brdf_test, mae, pa1, pa3):
                writer.add_scalar(tag, v, global_step=args.n_iters - 1)
        mae_part = '' if variant == "simple" else f', MAE: {mae}'
        out.write(f'======> {args.expname} test all: nvs psnr: {np.mean(psnr_test)}, nvs with brdf psnr: '
                  f'{np.mean(psnr_brdf_test)}{mae_part}  <========================\n')
        timer.add("final_evaluation", sync_time() - t0)
    if writer is not None:
        writer.close()
    res["times"] = timer.t
    return res


def render_test(args, test_dataset, logfolder, *, variant, device=None):
    """render_test(args) of the ``variant``'s script (train_tensoIR.py:65-106, general :71-127, simple :66-103): the
    checkpoint ``args.ckpt`` evaluated on every test view into ``{logfolder}/imgs_test_all/`` (one subfolder per light
    for ``general``, the lights taken from the checkpoint), with the script's printed lines.  The scripts'
    ``logfolder`` is ``{basedir}/test_{expname}-{timestamp}`` (:84).  Returns the 5-tuple of :func:`_five`, or None
    after the reference's message when the checkpoint does not exist (nothing is written then)."""
    if variant not in VARIANTS:
        raise ValueError(f"variant {variant!r}: expected one of {VARIANTS}")
    if not args.ckpt or not os.path.exists(args.ckpt):
        print('the ckpt path does not exists!!')
        return None
    dev = _device(args, device)
    model = _load_model(args.ckpt, dev)
    r = _test_all(variant, test_dataset, model, args, f'{logfolder}/imgs_test_all/', dev,
                  white_bg=test_dataset.white_bg)
    print(f'PSNRs_test: {r[0]}')
    print(f'PSNRs_rgb_brdf_test: {r[1]}')
    if variant != "simple":                  # the general script prints the last light's (:129-131)
        print(f'MAE_test: {r[2]}')
        print(f'PSNR_albedo_single: {r[3]}')
        print(f'PSNR_albedo_three: {r[4]}')
    return r


@torch.no_grad()
def export_mesh(args, device=None):
    """export_mesh(args) of the reference's scripts (train_tensoIR.py:52-61): the mesh of ``args.ckpt`` written to
    ``{ckpt[:-3]}.ply`` by mesh.export_mesh.  Returns the path."""
    from . import mesh
    path = f'{args.ckpt[:-3]}.ply'
    mesh.export_mesh(_load_model(args.ckpt, _device(args, device)), path)
    return path


def main(args, variant, datasets, render_dataset, *, device=None):
    """The ``__main__`` block of the ``variant``'s script (train_tensoIR.py:464-481): the reference's seeds, then with
    ``--export_mesh`` the mesh of ``--ckpt`` first, then :func:`render_test` when ``render_only`` and ``render_test``
    are set and :func:`reconstruction` otherwise.  ``datasets()`` returns the (train, test) datasets of the script's
    ``reconstruction``, ``render_dataset()`` the test set of its ``render_test``; each entry script builds them with its
    reference script's constructor arguments.  Returns what render_test or reconstruction returns.  A render-only run
    takes the model, and a general model's lights, from the checkpoint, so only a training run is checked against
    :func:`check_supported`; ``render_path`` is rejected in both."""
    rendering = bool(args.render_only and args.render_test)
    if rendering:
        _reject_render_path(args)
    else:
        check_supported(args, variant)
    torch.set_default_dtype(torch.float32)
    torch.manual_seed(SEED)
    torch.cuda.manual_seed_all(SEED)
    np.random.seed(SEED)
    random.seed(SEED)
    if args.export_mesh:
        export_mesh(args, device)
    stamp = datetime.datetime.now().strftime("-%Y%m%d-%H%M%S")
    if rendering:
        return render_test(args, render_dataset(), f'{args.basedir}/test_{args.expname}{stamp}', variant=variant,
                           device=device)
    train_dataset, test_dataset = datasets()
    logfolder = f'{args.basedir}/{args.expname}' + (stamp if args.add_timestamp else '')
    res = reconstruction(args, train_dataset, test_dataset, logfolder, variant=variant, device=device)
    print(f"steps redone after a list overflow: {res['redone']}, re-captures: {res['recaptures']}")
    return res


def _write_scalars(writer, it, row, relight):
    """The per-iteration scalars of :270-334 (``train/reg_l1`` is not logged: the L1 term is applied by the
    optimizer and is not part of ``total``)."""
    mse = float(row[1])
    writer.add_scalar('train/mse', float(row[0]), global_step=it)
    writer.add_scalar('train/PSNRs_rgb', -10.0 * np.log(mse) / np.log(10.0), global_step=it)
    writer.add_scalar('train/mse_rgb', mse, global_step=it)
    if not relight:
        for k, tag in ((3, 'train/reg_tv_density'), (4, 'train/reg_tv_app')):
            if float(row[k]) != 0.0:
                writer.add_scalar(tag, float(row[k]), global_step=it)
        return
    writer.add_scalar('train/PSNRs_rgb_brdf', -10.0 * np.log(float(row[2])) / np.log(10.0), global_step=it)
    writer.add_scalar('train/mse_rgb_brdf', float(row[2]), global_step=it)
    for k, tag in ((5, 'train/normals_diff_loss'), (6, 'train/normals_orientation_loss'),
                   (7, 'train/roughness_smoothness_loss'), (8, 'train/albedo_smoothness_loss')):
        writer.add_scalar(tag, float(row[k]), global_step=it)
