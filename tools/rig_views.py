"""Time relighting under analytic lights on N synthetic views of the lego scene and print one JSON line per rig: seconds
per view by phase of relight_rig's chunk body (primary render, sample, shadow march, shade) for (a) one hard directional
light, (b) one sphere light with 64 samples, (c) a one-light-at-a-time sweep of 32 hard directional lights (32 images
per view).  Every phase ends in a synchronise; every rig runs once untimed first.

    python tools/rig_views.py [--views 2] [--grid 300] [--size 800] [--batch 4096] [--olat 32]
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
    ap.add_argument("--olat", type=int, default=32)
    a = ap.parse_args()
    from tensoir_b200 import lighting as LT
    rigs = {"hard_directional": LT.load_rig({"sun": {"lights": [
                {"type": "directional", "direction": [0.3, -0.4, 0.85], "irradiance": 3.0}]}}),
            "sphere_64": LT.load_rig({"lamp": {"lights": [
                {"type": "point", "position": [2.0, -1.5, 2.5], "intensity": 40.0, "radius": 0.3, "samples": 64}]}}),
            f"olat_{a.olat}": LT.olat_rig(a.olat)}
    if not torch.cuda.is_available():
        raise SystemExit("tools/rig_views.py measures on the GPU: no CUDA device found")
    import __graft_entry__ as g
    g.build()
    import tensoir_b200.relighting as R
    from eval_views import gpu_info
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    dev = "cuda:0"
    model = make_lego_model(a.grid, dev, lights=("000", "120"))
    ds = SyntheticViews(hemisphere_poses(a.views), a.size, a.size, light_names=["a"])
    items = [ds[i] for i in range(len(ds))]
    far = LT.default_shadow_far(model)
    z_table = LT.shadow_table(far, dev)
    scale = torch.ones(3, device=dev)
    gpu, power = gpu_info()

    def tick():
        torch.cuda.synchronize()
        return time.perf_counter()

    def run(rig, items):
        LT.check_outside(rig, model.aabb)
        ph = dict(render=0.0, sample=0.0, march=0.0, shade=0.0)
        rows = 0
        for item in items:
            rays_v, face = item["rays"].to(dev), item["normals"].to(dev)
            n_pix = rays_v.shape[0]
            li = torch.zeros(n_pix, 1, dtype=torch.int32, device=dev)
            out = tuple(torch.empty(len(rig), n_pix, 3, device=dev) for _ in range(3))
            for s in range(0, n_pix, a.batch):
                e = min(s + a.batch, n_pix)
                t0 = tick()
                with torch.no_grad():
                    _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays_v[s:e], li[s:e], is_train=False,
                                                                              white_bg=True, ndc_ray=False, N_samples=-1)
                # the scene's appearance is untrained and its predicted normals are one near-constant vector, which
                # would pass or fail the cosine test for a whole view at once: shade with the boxes' face normals
                rays, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(
                    rays_v[s:e], (depth, face[s:e], albedo, rough, fresnel, acc))
                ph["render"] += tick() - t0
                for k, setup in enumerate(rig.values()):
                    t0 = tick()
                    u = LT._uniforms((e - s) * LT.slots_per_ray(setup), dev)
                    L, falloff, pos, list_o, list_d = LT.rig_sample(setup, rays, depth, normal, acc, u, 0.5)
                    t1 = tick()
                    vis = R.march_list(model, list_o, list_d, 'nerv', z_table)
                    t2 = tick()
                    LT.rig_shade(setup, rays, normal, albedo, rough, fresnel, acc, 0.5, scale, (L, falloff, pos, vis),
                                 'nerv', tuple(o[k] for o in out), s)
                    t3 = tick()
                    ph["sample"] += t1 - t0
                    ph["march"] += t2 - t1
                    ph["shade"] += t3 - t2
                    rows += int(list_o.shape[0])
        n = len(items)
        return {k: v / n for k, v in ph.items()}, rows / n

    for rig in rigs.values():                                         # warm-up of every shape: one view
        run(rig, items[:1])
    for name, rig in rigs.items():
        ph, rows = run(rig, items)
        print(json.dumps({"tool": "rig_views", "gpu": gpu, "power_limit": power, "rig": name, "setups": len(rig),
                          "views": len(items), "size": a.size, "grid": a.grid, "batch": a.batch,
                          "shadow_far": round(far, 4), "march_samples": int(z_table.shape[0]),
                          "shadow_rays_per_view": rows, **{f"{k}_s_per_view": v for k, v in ph.items()},
                          "total_s_per_view": sum(ph.values())}))


if __name__ == "__main__":
    main()
