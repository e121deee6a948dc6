"""Time material editing on N synthetic views of the lego scene under five environment maps and print one JSON line per
variant count K: seconds per view by phase of relight_edited's chunk body (primary render, sample + visibility march,
edit, shade) with the original materials plus K edited variants, all sharing one visibility pass per chunk.  The last
line gives the cost of one more variant, (total(K=max) - total(K=0)) / max, against the K=0 view.

    python tools/edit_views.py [--views 2] [--grid 300] [--size 800] [--batch 4096] [--variants 0 1 4]
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


def variant_rules(k):
    """Rules of edited variant k: a box over one part of the scene gets a new albedo and roughness, the rest shinier."""
    from tensoir_b200.editing import MaterialEdit
    z = -0.65 + 0.3 * k
    return [MaterialEdit(aabb=[[-1.0, -1.0, -1.0], [1.0, 1.0, z]], albedo_set=[0.8, 0.2 + 0.1 * k, 0.1],
                         roughness_set=0.3),
            MaterialEdit(roughness_mul=0.5, fresnel_set=0.1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=2)
    ap.add_argument("--grid", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--variants", type=int, nargs="+", default=[0, 1, 4])
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import bench
    import tensoir_b200.relighting as R
    from eval_views import gpu_info
    from tensoir_b200 import _lib
    from tensoir_b200.editing import edit_materials
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    assert torch.cuda.is_available(), "tools/edit_views.py measures on the GPU"
    dev = "cuda:0"
    names = ["bridge", "city", "fireplace", "forest", "night"]
    model = make_lego_model(a.grid, dev, lights=("000", "120"))
    env = Environment_Light({n: bench.synthetic_hdr(seed=20211202 + k) for k, n in enumerate(names)}, device=dev)
    ds = SyntheticViews(hemisphere_poses(a.views), a.size, a.size, light_names=names)
    items = [ds[i] for i in range(len(ds))]
    L, S = len(names), R.NUM_SAMPLES
    assert L <= _lib.RELIGHT_MAX_LIGHTS
    envs, keep = R.env_tables(env, names)
    scale = torch.tensor([1.0, 1.0, 1.0], device=dev)
    ones = torch.ones(3, device=dev)
    gpu, power = gpu_info()

    def tick():
        torch.cuda.synchronize()
        return time.perf_counter()

    def run(K):
        runs = [[]] + [variant_rules(k) for k in range(K)]
        ph = dict(render=0.0, visibility=0.0, edit=0.0, shade=0.0)
        for item in items:
            rays_v = item["rays"].to(dev)
            n_pix = rays_v.shape[0]
            li = torch.zeros(n_pix, 1, dtype=torch.int32, device=dev)
            with_map = torch.empty(len(runs), L, n_pix, 3, device=dev)
            without_map = torch.empty(len(runs), L, n_pix, 3, device=dev)
            for s in range(0, n_pix, a.batch):
                e = min(s + a.batch, n_pix)
                t0 = tick()
                with torch.no_grad():
                    _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays_v[s:e], li[s:e], is_train=False,
                                                                              white_bg=True, ndc_ray=False, N_samples=-1)
                rays, maps = R.chunk_inputs(rays_v[s:e], (depth, normal, albedo, rough, fresnel, acc))
                depth, normal, albedo, rough, fresnel, acc = maps
                t1 = tick()
                u = R._uniforms(L, e - s, S, dev)
                vis = R.relight_visibility(model, envs, L, rays, depth, normal, acc, u, S, 0.5, 'nerv')
                t2 = tick()
                ph["render"] += t1 - t0
                ph["visibility"] += t2 - t1
                for v, rules in enumerate(runs):
                    t0 = tick()
                    a_o, r_o, f_o, _ = edit_materials(maps, rules, scale, 0.5, rays=rays)
                    t1 = tick()
                    R.relight_shade(envs, L, rays, normal, a_o, r_o, f_o, acc, S, 0.5, ones, vis, 'nerv',
                                    (with_map[v], without_map[v]), s)
                    t2 = tick()
                    ph["edit"] += t1 - t0
                    ph["shade"] += t2 - t1
        n = len(items)
        return {k: v / n for k, v in ph.items()}

    run(0)                                                            # warm-up
    totals = {}
    for K in a.variants:
        ph = run(K)
        totals[K] = sum(ph.values())
        print(json.dumps({"tool": "edit_views", "gpu": gpu, "power_limit": power, "views": len(items), "size": a.size,
                          "grid": a.grid, "maps": L, "samples": S, "batch": a.batch, "variants": K,
                          **{f"{k}_s_per_view": v for k, v in ph.items()}, "total_s_per_view": totals[K]}))
    kmax = max(a.variants)
    if 0 in totals and kmax > 0:
        per = (totals[kmax] - totals[0]) / kmax
        print(json.dumps({"tool": "edit_views", "per_variant_s_per_view": per,
                          "per_variant_fraction_of_view": per / totals[0]}))
    del keep


if __name__ == "__main__":
    main()
