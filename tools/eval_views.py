"""Time evaluation_iter_TensoIR on N synthetic 800x800 views of the 300^3 lego scene and print one JSON line:
seconds per view split into render, metrics (the tir_eval kernel) and image write (everything else:
uint8 conversion, host copies, PNG encoding, the per-view ratio medians), plus the wall time of the reference's metric
formulas on the CPU (oracle/eval_oracle.py: torch / numpy / scipy) on the same maps for one view.

    python tools/eval_views.py [--views 4] [--grid 300] [--size 800]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--grid", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import tensoir_b200.evaluation as E
    from oracle import eval_oracle as EO
    from tensoir_b200 import Renderer_TensoIR_train
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    assert torch.cuda.is_available(), "tools/eval_views.py measures on the GPU"
    dev = "cuda:0"
    model = make_lego_model(a.grid, dev, lights=("000", "120"))
    ds = SyntheticViews(hemisphere_poses(a.views), a.size, a.size)
    items = [ds[i] for i in range(len(ds))]                    # generated up front: not part of the timing

    class Cached:
        img_wh, near_far, white_bg, lights_probes = ds.img_wh, ds.near_far, True, None

        def __len__(self):
            return len(items)

        def __getitem__(self, i):
            return items[i]
    args = types.SimpleNamespace(N_vis=a.views, batch_size_test=4096, relight_chunk_size=160000, second_nSample=96,
                                 second_near=0.05, second_far=1.5)
    t = {"render": 0.0, "metrics": 0.0}

    def timed(key, fn):
        def run(*x, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*x, **k)
            torch.cuda.synchronize()
            t[key] += time.perf_counter() - t0
            return r
        return run
    renderer = timed("render", Renderer_TensoIR_train)
    E.view_metrics = timed("metrics", E.view_metrics)
    out = tempfile.mkdtemp()
    kw = dict(prtx="0_", N_samples=-1, white_bg=True, compute_extra_metrics=True, device=dev)
    E.evaluation_iter_TensoIR(Cached(), model, args, renderer, savePath=os.path.join(out, "warm"), **kw)  # warm-up
    t.update(render=0.0, metrics=0.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ret = E.evaluation_iter_TensoIR(Cached(), model, args, renderer, savePath=os.path.join(out, "run"), **kw)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    n = a.views
    # the reference's formulas on the CPU, for one view's maps
    maps = E._render_view(Renderer_TensoIR_train, model, items[0]["rays"].to(dev), items[0]["light_idx"][0], args, -1,
                          False, True, dev)
    c = {k: v.cpu() for k, v in maps.items()}
    it = items[0]
    s, th = EO.view_ratios(c["albedo_map"], it["albedo"], it["rgbs_mask"])
    t0 = time.perf_counter()
    EO.view_metrics(a.size, a.size, c["rgb_map"], c["rgb_with_brdf_map"], it["rgbs"][0], c["albedo_map"],
                    it["albedo"], it["rgbs_mask"], s, th, c["normal_map"], it["normals"])
    cpu = time.perf_counter() - t0
    shutil.rmtree(out)
    name, power = gpu_info()
    print(json.dumps({"tool": "eval_views", "gpu": name, "power_limit": power, "views": n, "size": a.size,
                      "grid": a.grid, "s_per_view": total / n, "render_s_per_view": t["render"] / n,
                      "metrics_s_per_view": t["metrics"] / n,
                      "image_write_s_per_view": (total - t["render"] - t["metrics"]) / n,
                      "reference_formula_metrics_cpu_s_one_view": cpu,
                      "returned": [float(x) for x in ret]}))


if __name__ == "__main__":
    main()
