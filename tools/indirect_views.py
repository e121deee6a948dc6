"""Time relighting with one bounce of indirect light on N synthetic views of the lego scene under five environment maps
and print one JSON line per K: seconds per view by phase, each phase synchronised.  K = 0 is relight()'s direct-only
path (relight_chunk_fused); K > 0 is relight_chunk_indirect with S2 light samples per secondary hit.

    python tools/indirect_views.py [--views 2] [--grid 300] [--size 800] [--batch 4096] [--ks 0,8,16,32] [--s2 32]

Phases: render (primary render), direct (direct sample + march), secondary (secondary sample + march), hits (hit
compaction + materials), light (secondary light sample + march + radiance), shade.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=2)
    ap.add_argument("--grid", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--ks", default="0,8,16,32")
    ap.add_argument("--s2", type=int, default=32)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import bench
    import tensoir_b200.indirect as I
    import tensoir_b200.relighting as R
    from eval_views import gpu_info
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    assert torch.cuda.is_available(), "tools/indirect_views.py measures on the GPU"
    dev = "cuda:0"
    names = ["bridge", "city", "fireplace", "forest", "night"]
    model = make_lego_model(a.grid, dev, lights=("000", "120"))
    env = Environment_Light({n: bench.synthetic_hdr(seed=20211202 + k) for k, n in enumerate(names)}, device=dev)
    ds = SyntheticViews(hemisphere_poses(a.views), a.size, a.size, light_names=names)
    items = [ds[i] for i in range(len(ds))]
    L, S = len(names), R.NUM_SAMPLES
    rescale = torch.tensor([1.0, 1.0, 1.0], device=dev)
    tables = R.env_tables(env, names)
    timers = {}
    stack = []                                  # time spent in nested timed calls, per open timed call

    def tick():
        torch.cuda.synchronize()
        return time.perf_counter()

    def timed(key, fn, inherit=False):
        """fn, synchronised and timed under ``key``, less the time of timed calls nested in it.  With ``inherit``, a
        call nested in another timed call counts for the outer one."""
        def run(*x, **k):
            if inherit and stack:
                return fn(*x, **k)
            t0 = tick()
            stack.append(0.0)
            try:
                return fn(*x, **k)
            finally:
                dt = tick() - t0
                nested = stack.pop()
                timers[key] = timers.get(key, 0.0) + dt - nested
                if stack:
                    stack[-1] += dt
        return run

    lib = R._lib.load()
    lib.tir_indirect_shade = timed("shade", lib.tir_indirect_shade)
    lib.tir_indirect_hits = timed("hits", lib.tir_indirect_hits)
    I.point_materials = timed("hits", I.point_materials)
    I.secondary_hits = timed("secondary", I.secondary_hits)
    I.secondary_radiance = timed("light", I.secondary_radiance)
    I.relight_visibility = timed("direct", I.relight_visibility, inherit=True)
    R.relight_visibility = timed("direct", R.relight_visibility, inherit=True)
    R.relight_shade = timed("shade", R.relight_shade)

    name, power = gpu_info()
    for K in [int(k) for k in a.ks.split(",")]:
        for rep in range(2):                                          # rep 0 warms up
            timers.clear()
            for item in items:
                rays = item["rays"].to(dev)
                n_pix = rays.shape[0]
                li = torch.zeros(n_pix, 1, dtype=torch.int32, device=dev)
                with_map = torch.empty(L, n_pix, 3, device=dev)
                without_map = torch.empty(L, n_pix, 3, device=dev)
                gen = torch.Generator(dev).manual_seed(20211202)
                for s in range(0, n_pix, a.batch):
                    e = min(s + a.batch, n_pix)
                    t0 = tick()
                    with torch.no_grad():
                        _, dep, nrm, alb, rough, fres, acc, *_ = model(rays[s:e], li[s:e], is_train=False,
                                                                       white_bg=True, ndc_ray=False, N_samples=-1)
                    timers["render"] = timers.get("render", 0.0) + tick() - t0
                    maps = (dep, nrm, alb, rough, fres, acc)
                    u = R._uniforms(L, e - s, S, dev)
                    if K == 0:
                        R.relight_chunk_fused(model, env, names, rays[s:e], maps, rescale, u, S,
                                              out=(with_map, without_map), row0=s, tables=tables)
                    else:
                        I.relight_chunk_indirect(model, env, names, rays[s:e], maps, rescale, u, gen,
                                                 indirect_samples=K, indirect_light_samples=a.s2,
                                                 out=(with_map, without_map), row0=s, tables=tables)
            torch.cuda.synchronize()
        n = len(items)
        phases = {k: timers.get(k, 0.0) / n for k in ("render", "direct", "secondary", "hits", "light", "shade")}
        print(json.dumps({"tool": "indirect_views", "gpu": name, "power_limit": power, "views": n, "size": a.size,
                          "grid": a.grid, "maps": L, "samples": S, "batch": a.batch, "K": K,
                          "S2": a.s2 if K else 0, **{f"{k}_s_per_view": v for k, v in phases.items()},
                          "total_s_per_view": sum(phases.values())}), flush=True)


if __name__ == "__main__":
    main()
