"""Generate tests/golden/schedule_armadillo.pt and schedule_shrunk.pt by running the reference's UNMODIFIED
train_tensoIR.py (imported from a checkout of TensoIR) on the CPU, with recording stand-ins for its model, renderer,
dataset and SummaryWriter.

    python tests/golden/make_schedule_golden.py <path to the TensoIR checkout>

The stand-ins are put first in ``sys.modules`` the way dropin/ shadows ``models.*`` / ``renderer`` on a GPU run and
tools/ref_stubs/ stands in for the third-party imports; ``opt``, ``utils`` and the script itself come from the checkout.

* The model records every call the loop makes on it: construction, ``get_optparam_groups``, ``filtering_rays``,
  ``updateAlphaMask`` (returning the fixed asymmetric ``NEW_AABB``), ``shrink`` (which takes that box as the new
  aabb), ``upsample_volume_grid`` and ``save``.  Its regularisers return float64 leaves, so after ``backward`` each
  leaf's gradient is exactly the weight the script multiplied the term by.
* The renderer returns zero maps with ``requires_grad`` and records ``N_samples`` / ``is_relight`` and the ray ids
  (the fake rays carry their own index).
* ``torch.optim.Adam`` is wrapped to record which iteration creates an optimizer and, at every ``step``, the learning
  rate of every param group and the loss weights read from the leaves' gradients.

Two configs are recorded: configs/single_light/armadillo.txt at its full 80 000 iterations (per-iteration columns kept
as a SHA-256 of their float64 bytes plus samples, to stay small), and the same config shrunk to 400 iterations with the
schedule's iterations divided by 200 (every column kept in full); the shrunk one also sets the two loss-enhance ratios
away from 1 so the exponent of :291-292 is exercised.  tests/test_train_schedule_cpu.py checks
tensoir_b200.schedule.TrainSchedule against both; tests/test_train_gpu.py trains on the shrunk one.
"""
import hashlib
import io
import os
import runpy
import shutil
import sys
import tempfile
import types
import contextlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
STUBS = os.path.join(REPO, "tools", "ref_stubs")

NEW_AABB = torch.tensor([[-0.8125, -1.0625, -0.6875], [0.9375, 0.5625, 1.1875]], dtype=torch.float32)
N_RAYS = 10000                       # fake training rays: 2 batches of 4096 per sampler epoch
N_IDS = 6                            # ray ids of the first 3 epochs
COLUMNS = ("lr0", "lr1", "lr2", "tv_density", "tv_app", "l1", "normals_diff", "normals_orientation",
           "roughness_smoothness", "albedo_smoothness", "relight", "n_samples")
SHRUNK = {"n_iters": 400, "lr_decay_iters": 400, "upsamp_list": "[50, 100, 150, 200]",
          "update_AlphaMask_list": "[50, 75, 100, 125, 150, 175]", "vis_every": 25, "save_iters": 50,
          "normals_loss_enhance_ratio": 2.5, "BRDF_loss_enhance_ratio": 0.4}


class Recorder:
    def __init__(self):
        self.it = -1                  # iteration of the renderer call in flight (-1: set-up)
        self.events = []
        self.leaves = {}
        self.rows = []
        self.ids = []
        self.render = None
        self.logfolder = None
        self.optimizers = []

    def leaf(self, name, shape=()):
        t = torch.zeros(shape, dtype=torch.float64, requires_grad=True)
        self.leaves[name] = t
        return t

    def rel(self, path):
        return os.path.relpath(path, self.logfolder)


REC = Recorder()


class TensorVMSplit(torch.nn.Module):
    def __init__(self, aabb, gridSize, device, **kw):
        super().__init__()
        REC.events.append((REC.it, "init", [int(g) for g in gridSize]))
        self.aabb = aabb.clone()
        self.p = torch.nn.ParameterList([torch.nn.Parameter(torch.zeros(1)) for _ in range(3)])

    def get_optparam_groups(self, lr_init_spatialxyz=0.02, lr_init_network=0.001):
        REC.events.append((REC.it, "get_optparam_groups", lr_init_spatialxyz, lr_init_network))
        # the three kinds of group of the real model: VM factors, networks, a fixed 0.001 (light_line / lgtSGs)
        return [{'params': [self.p[0]], 'lr': lr_init_spatialxyz}, {'params': [self.p[1]], 'lr': lr_init_network},
                {'params': [self.p[2]], 'lr': 0.001}]

    def filtering_rays(self, all_rays, N_samples=256, chunk=10240 * 5, bbox_only=False):
        REC.events.append((REC.it, "filtering_rays", bool(bbox_only)))
        mask = torch.ones(all_rays.shape[0], dtype=torch.bool)
        return all_rays[mask], mask

    def updateAlphaMask(self, gridSize=(200, 200, 200)):
        REC.events.append((REC.it, "updateAlphaMask", [int(g) for g in gridSize]))
        return NEW_AABB.clone()

    def shrink(self, new_aabb):
        REC.events.append((REC.it, "shrink"))
        self.aabb = new_aabb

    def upsample_volume_grid(self, res_target):
        REC.events.append((REC.it, "upsample_volume_grid", [int(g) for g in res_target]))

    def save(self, path):
        REC.events.append((REC.it, "save", REC.rel(path)))

    def vector_comp_diffs(self):
        return REC.leaf("ortho")

    def density_L1(self):
        return REC.leaf("l1")

    def TV_loss_density(self, reg):
        return REC.leaf("tv_density")

    def TV_loss_app(self, reg):
        return REC.leaf("tv_app")


def Renderer_TensoIR_train(rays, normal_gt, light_idx, tensoIR, N_samples=-1, is_relight=True, **kw):
    REC.it += 1
    REC.leaves = {}
    if len(REC.ids) < N_IDS:
        REC.ids.append(rays[:, 0].to(torch.int16).clone())
    REC.render = (bool(is_relight), int(N_samples))
    n = rays.shape[0]
    return {"rgb_map": REC.leaf("rgb", (n, 3)), "rgb_with_brdf_map": REC.leaf("rgb_brdf", (n, 3)),
            "normals_diff_map": REC.leaf("normals_diff", (n, 1)),
            "normals_orientation_loss_map": REC.leaf("normals_orientation", (n, 1)),
            "roughness_smoothness_loss": REC.leaf("roughness_smoothness"),
            "albedo_smoothness_loss": REC.leaf("albedo_smoothness")}


def evaluation_iter_TensoIR(test_dataset, tensoIR, args, renderer, savePath=None, prtx='', N_samples=-1,
                            white_bg=False, ndc_ray=False, compute_extra_metrics=True, device='cuda', logger=None,
                            step=None, test_all=False):
    REC.events.append((REC.it, "evaluation", REC.rel(savePath), prtx, int(N_samples), bool(test_all),
                       bool(compute_extra_metrics)))
    return [20.0], [20.0], 0.1, 20.0, 20.0


class Dataset:
    """The train / test dataset attributes the loop reads (dataLoader/tensoIR_rotation_setting.py:48-55, :86-140);
    ray i carries i in its first component."""

    def __init__(self, datadir, hdrdir=None, split='train', downsample=1.0, light_name=None, light_rotation=None,
                 **kw):
        self.white_bg, self.near_far = True, [2.0, 6.0]
        self.scene_bbox = torch.tensor([[-1.5, -1.5, -1.5], [1.5, 1.5, 1.5]]) * downsample
        self.all_rays = torch.zeros(N_RAYS, 6)
        self.all_rays[:, 0] = torch.arange(N_RAYS, dtype=torch.float32)
        self.all_rgbs = torch.full((N_RAYS, 3), 0.5)
        self.all_masks = torch.ones(N_RAYS, 1, dtype=torch.bool)
        self.all_light_idx = torch.zeros(N_RAYS, 1, dtype=torch.long)


class SummaryWriter:
    def __init__(self, logdir=None, **kw):
        REC.logfolder = logdir

    def add_scalar(self, *a, **k):
        pass

    def add_image(self, *a, **k):
        pass


class RecordingAdam(torch.optim.Adam):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        REC.events.append((REC.it, "optimizer"))

    def step(self, closure=None):
        g = {k: (None if t.grad is None else t.grad.reshape(-1)[0].item() * t.numel()) for k, t in REC.leaves.items()}
        # normals maps enter as w * map.mean(): gradient w / n per element, n a power of two here, so w is exact
        relight, n_samples = REC.render
        row = [float(grp["lr"]) for grp in self.param_groups]
        row += [g.get(k) or 0.0 for k in ("tv_density", "tv_app", "l1", "normals_diff", "normals_orientation",
                                           "roughness_smoothness", "albedo_smoothness")]
        row += [float(relight), float(n_samples)]
        REC.rows.append(row)
        return super().step(closure)


def install(ref):
    for name in ("models", "models.tensoRF_rotated_lights", "renderer", "dataLoader", "torch.utils.tensorboard"):
        sys.modules.pop(name, None)
    models = types.ModuleType("models")
    models.__path__ = []
    rot = types.ModuleType("models.tensoRF_rotated_lights")
    rot.TensorVMSplit, rot.AlphaGridMask, rot.raw2alpha = TensorVMSplit, object, None
    models.tensoRF_rotated_lights = rot
    ren = types.ModuleType("renderer")
    ren.Renderer_TensoIR_train, ren.evaluation_iter_TensoIR = Renderer_TensoIR_train, evaluation_iter_TensoIR
    ren.__all__ = ["Renderer_TensoIR_train", "evaluation_iter_TensoIR", "np", "torch", "random"]
    ren.np, ren.torch = np, torch
    import random
    ren.random = random
    dl = types.ModuleType("dataLoader")
    dl.dataset_dict = {"tensoIR_unknown_rotated_lights": Dataset}
    tb = types.ModuleType("torch.utils.tensorboard")
    tb.SummaryWriter = SummaryWriter
    sys.modules.update({"models": models, "models.tensoRF_rotated_lights": rot, "renderer": ren, "dataLoader": dl,
                        "torch.utils.tensorboard": tb})
    for p in (ref, STUBS):
        if p not in sys.path:
            sys.path.insert(0, p)
    torch.optim.Adam = RecordingAdam


def write_config(path, base, overrides):
    lines, seen = [], set()
    for line in open(base):
        key = line.split("=", 1)[0].strip()
        if key in overrides:
            line = f"{key} = {overrides[key]}\n"
            seen.add(key)
        lines.append(line)
    lines += [f"{k} = {v}\n" for k, v in overrides.items() if k not in seen]
    open(path, "w").writelines(lines)


def record(ref, cfg, basedir):
    global REC
    REC = Recorder()
    argv = sys.argv
    sys.argv = ["train_tensoIR.py", "--config", cfg, "--basedir", basedir]
    try:
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            g = runpy.run_path(os.path.join(ref, "train_tensoIR.py"), run_name="__main__")
    finally:
        sys.argv = argv
    config = {k: v for k, v in vars(g["args"]).items() if k not in ("config", "basedir", "datadir", "hdrdir")}
    cols = np.asarray(REC.rows, dtype=np.float64)
    assert cols.shape == (config["n_iters"], len(COLUMNS)), cols.shape
    return config, cols


def main(ref):
    install(ref)
    tmp = tempfile.mkdtemp(prefix="tir_schedule_")
    try:
        base = os.path.join(ref, "configs", "single_light", "armadillo.txt")
        for name, overrides in (("armadillo", {}), ("shrunk", SHRUNK)):
            cfg = os.path.join(tmp, f"{name}.txt")
            write_config(cfg, base, overrides)
            config, cols = record(ref, cfg, os.path.join(tmp, "log_" + name))
            out = {"config": config, "n_rays": N_RAYS, "new_aabb": NEW_AABB,
                   "initial_aabb": torch.tensor([[-1.5, -1.5, -1.5], [1.5, 1.5, 1.5]]), "columns": COLUMNS,
                   "events": REC.events, "ids": torch.stack(REC.ids)}
            if name == "shrunk":
                out["per_iter"] = torch.from_numpy(cols)
            else:
                events = sorted({e[0] for e in REC.events if e[0] >= 0})
                keep = sorted({i for i in range(0, cols.shape[0], 1000)} |
                              {j for e in events for j in (e - 1, e, e + 1) if 0 <= j < cols.shape[0]})
                out["sample_iters"] = torch.tensor(keep)
                out["samples"] = torch.from_numpy(cols[keep])
                out["sha256"] = [hashlib.sha256(np.ascontiguousarray(cols[:, c]).tobytes()).hexdigest()
                                 for c in range(cols.shape[1])]
            path = os.path.join(HERE, f"schedule_{name}.pt")
            torch.save(out, path)
            print(path, os.path.getsize(path) // 1024, "KiB")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    if len(sys.argv) < 2 or not os.path.isfile(os.path.join(sys.argv[1], "train_tensoIR.py")):
        raise SystemExit(__doc__)
    main(os.path.abspath(sys.argv[1]))
