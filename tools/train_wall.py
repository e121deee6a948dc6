"""Wall time of the native trainer, graphed and eager, on one GPU; prints one JSON line.

    python tools/train_wall.py [--iters 2000] [--views 30] [--res 200] [--variant full|general|simple]
                               [--filter_views 0] [--out result.json]

The schedule is configs/single_light/armadillo.txt as the reference parses it (kept in
tests/golden/schedule_armadillo.pt), with n_iters, lr_decay_iters, upsamp_list, update_AlphaMask_list, vis_every and
save_iters scaled by iters / 80000: both phases and every event type (mask updates with shrink and re-filter,
upsamples, evaluations, checkpoints).  The scene is the synthetic lego (tensoir_b200.synthetic) seen from ``views``
training cameras at ``res`` x ``res`` and 5 test cameras, batches of 4096 rays, starting from the lego density at
128^3 (the reference's random initialisation leaves the field empty after a few hundred iterations, and the mask
update then finds no occupied voxel).  Reported per run: the wall time and ms/step of each phase (evaluations and
checkpoints excluded), the time per grid-event kind, evaluation and capture times, and the card's name and power
limit read in the same run.

``--variant general`` trains the general multi-light model (train_tensoIR_general_multi_lights.py) on three lights
("sunset", "snow", "courtyard"): every training view once per light, and a final evaluation once per light;
``--variant simple`` runs train_tensoIR_simple.py's evaluations on the single-light scene.  ``--filter_views N``
additionally times, on the host, the trainer's ray filter (``filtering_rays(bbox_only=True)`` and the filtered copies of
rays, colours and light ids) on a table of N views x the variant's lights x 800 x 800 rays, the size of that script's
full training set (100 views x 3 lights: 192 M rays, 4.6 GB of rays).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.strip().split(",")]
        return name, power
    except Exception:                                   # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


LIGHTS = ("sunset", "snow", "courtyard")


def _time_filter(model, views, n_lights, res=800):
    """Host seconds of filtering_rays(bbox_only=True) and of the trainer's whole filter (train._Rays.filter: that call
    plus the filtered copies of rays, colours and light ids) on views x n_lights x res^2 rays, laid out like the
    training set (every view's rays once per light)."""
    from tensoir_b200 import train
    from tensoir_b200.synthetic import hemisphere_poses, image_rays
    per_view = [image_rays(p, res, res) for p in hemisphere_poses(views)]
    rays = torch.cat([r for r in per_view for _ in range(n_lights)])
    del per_view
    n = rays.shape[0]
    rgbs = torch.ones(n, 3)
    li = torch.arange(n_lights).repeat_interleave(res * res).repeat(views).view(-1, 1)
    t0 = time.perf_counter()
    kept, _ = model.filtering_rays(rays, bbox_only=True)
    torch.cuda.synchronize()
    t_rays = time.perf_counter() - t0
    del kept
    table = train._Rays(types.SimpleNamespace(all_rays=rays, all_rgbs=rgbs, all_light_idx=li), 4096)
    t0 = time.perf_counter()
    table.filter(model)
    torch.cuda.synchronize()
    t_all = time.perf_counter() - t0
    out = {"rays": int(n), "ray_gb": round(rays.numel() * 4 / 1e9, 2), "kept": int(table.rays.shape[0]),
           "filtering_rays_s": round(t_rays, 2), "trainer_filter_s": round(t_all, 2)}
    del table, rays, rgbs, li
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--views", type=int, default=30)
    ap.add_argument("--res", type=int, default=200)
    ap.add_argument("--variant", default="full", choices=("full", "general", "simple"))
    ap.add_argument("--filter_views", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_wall.py needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import train
    from tensoir_b200.synthetic import SyntheticTrainViews, SyntheticViews, hemisphere_poses, make_lego_model
    dev = "cuda:0"
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "schedule_armadillo.pt"), weights_only=False)
    s = a.iters / fx["config"]["n_iters"]
    general = a.variant == "general"
    lights = LIGHTS if general else ("000",)
    poses = hemisphere_poses(a.views + 5)
    train_views = SyntheticTrainViews(poses[:a.views], a.res, a.res, n_lights=len(lights))
    test_views = SyntheticViews(poses[a.views:], a.res, a.res, n_lights=len(lights))
    tmp = tempfile.mkdtemp(prefix="tir_train_wall_")
    ckpt = os.path.join(tmp, "start.th")
    m = make_lego_model(128, dev, general=general, lights=lights)
    m.alphaMask = None
    m.save(ckpt)
    card, power = _card()
    res = {"card": card, "power_limit": power, "variant": a.variant, "lights": len(lights), "iters": a.iters,
           "train_rays": int(train_views.all_rays.shape[0]), "batch": 4096, "test_views": len(test_views), "res": a.res}
    if a.filter_views:
        res["filter"] = _time_filter(m, a.filter_views, len(lights))
    del m
    for graphed in (True, False):
        args = types.SimpleNamespace(**fx["config"])
        args.n_iters = args.lr_decay_iters = a.iters
        args.upsamp_list = [int(round(v * s)) for v in args.upsamp_list]
        args.update_AlphaMask_list = [int(round(v * s)) for v in args.update_AlphaMask_list]
        args.vis_every = max(1, int(round(args.vis_every * s)))
        args.save_iters = max(1, int(round(args.save_iters * s)))
        args.progress_refresh_rate = 100
        args.expname, args.ckpt, args.config = "lego", ckpt, None
        args.light_name_list = list(LIGHTS) if general else None
        np.random.seed(20211202)
        t0 = time.perf_counter()
        out = train.reconstruction(args, train_views, test_views, os.path.join(tmp, str(graphed)), variant=a.variant,
                                   graphed=graphed, device=dev, out=sys.stderr)
        torch.cuda.synchronize()
        t = out["times"]
        r = {"wall_s": round(time.perf_counter() - t0, 3), "redone": out["redone"], "recaptures": out["recaptures"],
             "final_test_psnr": out["psnr_test"], "final_mse_rgb": float(out["losses"][-1, 1])}
        for p in ("phase1", "phase2"):
            n = int(t.get(p + "_iters", 0))
            r[p + "_iters"], r[p + "_s"] = n, round(t.get(p + "_steps", 0.0), 3)
            r[p + "_ms_per_step"] = round(1e3 * t.get(p + "_steps", 0.0) / max(n, 1), 3)
        for k in ("mask_update", "refilter", "upsample", "capture", "evaluation", "save", "final_evaluation"):
            r[k + "_s"] = round(t.get(k, 0.0), 3)
        r["events"] = {k: sum(1 for e in out["events"] if e[1] == k)
                       for k in ("updateAlphaMask", "shrink", "filtering_rays", "upsample_volume_grid", "evaluation",
                                 "save")}
        res["graphed" if graphed else "eager"] = r
        del out
        torch.cuda.empty_cache()
    res["phase_speedup"] = {p: round(res["eager"][p + "_ms_per_step"] / max(res["graphed"][p + "_ms_per_step"], 1e-9), 2)
                            for p in ("phase1", "phase2")}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
