"""Time the light fit (tensoir_b200.light_fit) on N synthetic views of the lego scene and print one JSON line: seconds
per view by phase (primary render, transport sample, shadow march, transport build, Gram accumulation) and the solve
time, with the shadow rays per view and the card's name and power limit.  Every phase ends in a synchronise; one view
runs untimed first.  The scene's predicted normals are untrained, so it is shaded with the boxes' face normals.

    python tools/fit_views.py [--views 4] [--grid 300] [--size 800] [--pixels 65536] [--res 16x32] [--batch 4096]
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
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--grid", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--pixels", type=int, default=65536)
    ap.add_argument("--res", default="16x32")
    ap.add_argument("--batch", type=int, default=4096)
    a = ap.parse_args()
    from tensoir_b200 import light_fit as LF
    H_e, W_e = LF.parse_res(a.res)
    if not torch.cuda.is_available():
        raise SystemExit("tools/fit_views.py measures on the GPU: no CUDA device found")
    import __graft_entry__ as g
    g.build()
    import tensoir_b200.relighting as R
    from eval_views import gpu_info
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    dev = "cuda:0"
    model = make_lego_model(a.grid, dev)
    ds = SyntheticViews(hemisphere_poses(a.views + 1), a.size, a.size, light_names=["a"])
    items = [ds[i] for i in range(len(ds))]
    grid = LF.texel_tables(H_e, W_e, dev)
    K = H_e * W_e
    table = R.relight_table(dev)
    gpu, power = gpu_info()

    def tick():
        torch.cuda.synchronize()
        return time.perf_counter()

    def run(items):
        ne = LF.Normals(K, 1, dev)
        ph = dict(render=0.0, sample=0.0, march=0.0, build=0.0, gram=0.0)
        rows = pixels = 0
        gen = torch.Generator().manual_seed(LF.SEED)
        for item in items:
            pix = LF._sample_pixels(item["rgbs_mask"].reshape(-1), a.pixels, gen)
            pixels += pix.numel()
            rays_v, face = item["rays"][pix].to(dev), item["normals"][pix].to(dev)
            y = item["rgbs"][:, pix].to(dev).double()
            for s in range(0, pix.numel(), a.batch):
                e = min(s + a.batch, pix.numel())
                t0 = tick()
                li = torch.zeros(e - s, 1, dtype=torch.int32, device=dev)
                with torch.no_grad():
                    _, depth, _, albedo, rough, fresnel, acc, *_ = model(rays_v[s:e], li, is_train=False,
                                                                          white_bg=True, ndc_ray=False, N_samples=-1)
                rays, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(
                    rays_v[s:e], (depth, face[s:e], albedo, rough, fresnel, acc))
                t1 = tick()
                pos, list_o, list_d = LF.transport_sample(grid, rays, depth, normal, acc, 0.5)
                t2 = tick()
                vis = R.march_list(model, list_o, list_d, 'nerv', table)
                t3 = tick()
                T = LF.transport_build(grid, rays, normal, albedo, rough, fresnel, acc, 0.5, 1.0, pos, vis, 'nerv')
                t4 = tick()
                yc = y[:, s:e]
                ne.add(T, LF.srgb_to_linear(yc), LF.usable(yc, acc > 0.5))
                t5 = tick()
                for k, (u, v) in zip(ph, ((t0, t1), (t1, t2), (t2, t3), (t3, t4), (t4, t5))):
                    ph[k] += v - u
                rows += int(list_o.shape[0])
        t0 = tick()
        _, info = LF.solve(ne.G, ne.B, H_e, W_e)
        solve = tick() - t0
        n = len(items)
        return {k: v / n for k, v in ph.items()}, solve, rows / n, pixels / n, info[0]

    run(items[:1])                                                     # warm-up of every shape
    ph, solve, rows, pixels, info = run(items[1:])
    print(json.dumps({"tool": "fit_views", "gpu": gpu, "power_limit": power, "views": a.views, "size": a.size,
                      "grid": a.grid, "fit_res": [H_e, W_e], "pixels_per_view": pixels, "batch": a.batch,
                      "shadow_rays_per_view": rows, **{f"{k}_s_per_view": v for k, v in ph.items()},
                      "total_s_per_view": sum(ph.values()), "solve_s": solve, "solve_iterations": info["iterations"]}))


if __name__ == "__main__":
    main()
