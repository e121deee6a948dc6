"""Time the relighting evaluation on N synthetic views of the lego scene under five environment maps and print one JSON
line: seconds per view by phase (primary render, sample + visibility list, visibility march, shade, metrics, PNG
writing), and on the same chunks and the same sample indices the eager relight_chunk (tensoir_b200/relight.py) with the
largest difference between the two.  With ``--sampling mis`` the chunks go through mis.relight_chunk_mis (S_b =
``--brdf_samples`` BRDF samples and 512 - S_b light samples per (map, hit)) and the eager comparison is skipped.  Both
modes report the shadow rays marched per view and a noise figure: on the middle chunk of every view, the RMSE of the
linear estimate against the mean of 16 MIS passes (S_b = 128), over the hit pixels of every map whose reference is
below 0.98 (the default estimator's linear value is its sRGB output inverted, on pixels below the clamp).

    python tools/relight_views.py [--views 2] [--grid 300] [--size 800] [--batch 4096] [--sampling light|mis]
                                  [--brdf_samples 128]
"""
import argparse
import json
import os
import sys
import tempfile
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
    ap.add_argument("--sampling", choices=("light", "mis"), default="light")
    ap.add_argument("--brdf_samples", type=int, default=128)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import bench
    import tensoir_b200.mis as MIS
    import tensoir_b200.relighting as R
    from eval_views import gpu_info
    from tensoir_b200 import ops
    from tensoir_b200.relight import Environment_Light, relight_chunk
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    assert torch.cuda.is_available(), "tools/relight_views.py measures on the GPU"
    dev = "cuda:0"
    names = ["bridge", "city", "fireplace", "forest", "night"]
    model = make_lego_model(a.grid, dev, lights=("000", "120"))
    env = Environment_Light({n: bench.synthetic_hdr(seed=20211202 + k) for k, n in enumerate(names)}, device=dev)
    ds = SyntheticViews(hemisphere_poses(a.views), a.size, a.size, light_names=names)
    items = [ds[i] for i in range(len(ds))]
    L, S, H, W = len(names), R.NUM_SAMPLES, a.size, a.size
    rescale = torch.tensor([1.0, 1.0, 1.0], device=dev)
    phases = dict(render=0.0, sample=0.0, march=0.0, shade=0.0, metrics=0.0, write=0.0, eager=0.0, eager_march=0.0)

    def tick():
        torch.cuda.synchronize()
        return time.perf_counter()

    # phase timing: the two relighting kernels and the march are timed through the same wrappers relight() calls
    lib = R._lib.load()
    timers = {}
    for key, fn_name in (("sample", "tir_relight_sample"), ("shade", "tir_relight_shade"),
                         ("sample", "tir_relight_mis_sample"), ("shade", "tir_relight_mis_shade")):
        fn = getattr(lib, fn_name)

        def timed(*x, _fn=fn, _key=key):
            t0 = tick()
            r = _fn(*x)
            timers[_key] = timers.get(_key, 0.0) + tick() - t0
            return r
        timers[key] = 0.0
        setattr(lib, fn_name, timed)
    # the density march is shared by both paths: it is timed under "march" inside the fused chunk and under
    # "eager_march" inside the eager one, so that the two shading figures can be compared on their own
    march = ops.march_density
    march_key = [None]
    shadow_rays = [0]

    def timed_march(*x, **k):
        t0 = tick()
        r = march(*x, **k)
        timers[march_key[0]] = timers.get(march_key[0], 0.0) + tick() - t0
        if march_key[0] == "march":
            shadow_rays[0] += int(x[1].shape[0])
        return r
    ops.march_density = timed_march

    def with_march_key(key, fn):
        def run(*x, **k):
            march_key[0] = key
            try:
                return fn(*x, **k)
            finally:
                march_key[0] = None
        return run
    relight_chunk_fused = with_march_key("march", R.relight_chunk_fused)
    relight_chunk_mis = with_march_key("march", MIS.relight_chunk_mis)
    S_b = a.brdf_samples if a.sampling == "mis" else 0
    relight_chunk = with_march_key("eager_march", relight_chunk)
    tables = R.env_tables(env, names)
    max_diff = 0.0
    out_dir = tempfile.mkdtemp()
    for rep in range(2):                                              # rep 0 warms up
        timers.clear()
        shadow_rays[0] = 0
        for k in phases:
            phases[k] = 0.0
        for v, item in enumerate(items):
            rays = item["rays"].to(dev)
            n_pix = rays.shape[0]
            li = torch.zeros(n_pix, 1, dtype=torch.int32, device=dev)
            with_map = torch.empty(L, n_pix, 3, device=dev)
            without_map = torch.empty(L, n_pix, 3, device=dev)
            for s in range(0, n_pix, a.batch):
                e = min(s + a.batch, n_pix)
                t0 = tick()
                with torch.no_grad():
                    _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays[s:e], li[s:e], is_train=False,
                                                                              white_bg=True, ndc_ray=False, N_samples=-1)
                phases["render"] += tick() - t0
                maps = (depth, normal, albedo, rough, fresnel, acc)
                if a.sampling == "mis":
                    u_l, u_b = MIS.mis_uniforms(L, e - s, S - S_b, S_b, dev)
                    relight_chunk_mis(model, env, names, rays[s:e], maps, rescale, u_l, u_b,
                                      out=(with_map, without_map), row0=s, tables=tables)
                    continue
                u = R._uniforms(L, e - s, S, dev)
                relight_chunk_fused(model, env, names, rays[s:e], maps, rescale, u, S, out=(with_map, without_map),
                                    row0=s, tables=tables)
                t0 = tick()
                hit = acc > 0.5
                for k, name in enumerate(names):
                    cdf = env._cdf[name]
                    idx = torch.searchsorted(cdf, u[k][hit], right=True).clamp_(max=cdf.numel() - 1)
                    w, wo = relight_chunk(model, env, name, rays[s:e], maps, rescale, idx, S)
                    max_diff = max(max_diff, float((wo - without_map[k, s:e]).abs().max()),
                                   float((w - with_map[k, s:e]).abs().max()))
                phases["eager"] += tick() - t0
            gt = item["rgbs"].to(dev)
            t0 = tick()
            R.pair_metrics(without_map, gt, H, W).cpu()
            phases["metrics"] += tick() - t0
            t0 = tick()
            u8 = (without_map * 255).to(torch.uint8).reshape(L, H, W, 3).cpu().numpy()
            u8w = (with_map * 255).to(torch.uint8).reshape(L, H, W, 3).cpu().numpy()
            for k, name in enumerate(names):
                R._imwrite(os.path.join(out_dir, f"{v}_{name}_without.png"), u8[k])
                R._imwrite(os.path.join(out_dir, f"{v}_{name}_with.png"), u8w[k])
            phases["write"] += tick() - t0
        for k in ("sample", "march", "shade", "eager_march"):
            phases[k] = timers.get(k, 0.0)
    n = len(items)
    rays_per_view = shadow_rays[0] / n
    # noise figure on the middle chunk of every view, which holds the object (not timed)
    sq, cnt = 0.0, 0
    for item in items:
        mid = (item["rays"].shape[0] - a.batch) // 2
        rays = item["rays"].to(dev)[mid:mid + a.batch]
        m = rays.shape[0]
        li = torch.zeros(m, 1, dtype=torch.int32, device=dev)
        with torch.no_grad():
            _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays, li, is_train=False, white_bg=True,
                                                                      ndc_ray=False, N_samples=-1)
        maps = (depth, normal, albedo, rough, fresnel, acc)

        def mis_linear(sb):
            lin = torch.zeros(L, m, 3, device=dev)
            u_l, u_b = MIS.mis_uniforms(L, m, S - sb, sb, dev)
            MIS.relight_chunk_mis(model, env, names, rays, maps, rescale, u_l, u_b, tables=tables, linear_out=lin)
            return lin
        ref = sum(mis_linear(128) for _ in range(16)) / 16
        mask = (acc.reshape(-1) > 0.5)[None, :, None] & (ref < 0.98)
        if a.sampling == "mis":
            est = mis_linear(S_b)
        else:
            _, wo = R.relight_chunk_fused(model, env, names, rays, maps, rescale, R._uniforms(L, m, S, dev), S,
                                          tables=tables)
            est = torch.where(wo <= 0.0031308 * 12.92, wo / 12.92, ((wo + 0.055) / 1.055) ** 2.4 - 1e-6)
            mask = mask & (wo < 0.999)
        sq += float(((est - ref) ** 2)[mask].sum())
        cnt += int(mask.sum())
    name, power = gpu_info()
    print(json.dumps({"tool": "relight_views", "gpu": name, "power_limit": power, "views": n, "size": a.size,
                      "grid": a.grid, "maps": L, "samples": S, "batch": a.batch, "sampling": a.sampling,
                      "brdf_samples": S_b, "shadow_rays_per_view": rays_per_view,
                      "linear_rmse_middle_chunk": (sq / max(cnt, 1)) ** 0.5,
                      **{f"{k}_s_per_view": v / n for k, v in phases.items() if k not in ("eager", "eager_march")},
                      "fused_relight_s_per_view": (phases["sample"] + phases["march"] + phases["shade"]) / n,
                      "fused_without_march_s_per_view": (phases["sample"] + phases["shade"]) / n,
                      "eager_relight_chunk_s_per_view": phases["eager"] / n,
                      "eager_march_s_per_view": phases["eager_march"] / n,
                      "eager_without_march_s_per_view": (phases["eager"] - phases["eager_march"]) / n,
                      "max_abs_diff_fused_vs_eager": max_diff}))


if __name__ == "__main__":
    main()
