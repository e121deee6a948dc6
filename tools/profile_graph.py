"""Kernel-time breakdown of the CUDA-graph replayed training step that bench.py times (config 2).

The step is built as ``bench.measure`` builds it: ``tensoir_b200.optim.FusedAdam`` over ``lr_tensors`` groups with the
density L1 term folded into the optimiser, the lean march counters, the static lists reserved at 4x the warm-up's
longest.  Prints the step time (CUDA events, profiler off), one row per kernel (device time per replay and its share of
the summed kernel time, torch.profiler over ``--replays`` replays), the device-side list lengths of the last replay and,
for the VM-factor gradient scatters, how many consecutive list rows hit the same tap texel (the runs that the scatters
sum in registers before their atomics).

    python tools/profile_graph.py [--replays 10] [--json FILE]
"""
import argparse, json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
import __graft_entry__ as g

# kernel names of this build and of the build before it (the two can be compared with TIR_LIB)
SCATTERS = ("density_bwd_kernel", "app_products_bwd_kernel", "density_grad_bwd_kernel", "app_scatter_kernel")
MERGE_ROWS = (1, 4, 8, 16, 32)


def tap_keys(xn, grid, k):
    """Texel index and weight of the 4 plane taps and 2 line taps of orientation k (zero-padding sampler, the
    arithmetic of bilinear_setup / linear_setup in tir_device.cuh)."""
    m0, m1, v = ((0, 1, 2), (0, 2, 1), (1, 2, 0))[k]
    W, H, D = grid[m0], grid[m1], grid[v]

    def axis(c, n):
        i = (c + 1.0) * 0.5 * (n - 1)
        f = torch.floor(i)
        i0 = f.long()
        w1, w0 = i - f, f + 1.0 - i
        ok0, ok1 = (i0 >= 0) & (i0 < n), (i0 + 1 >= 0) & (i0 + 1 < n)
        return i0.clamp(0, n - 1), (i0 + 1).clamp(0, n - 1), torch.where(ok0, w0, 0.0), torch.where(ok1, w1, 0.0)

    x0, x1, wx0, wx1 = axis(xn[:, m0], W)
    y0, y1, wy0, wy1 = axis(xn[:, m1], H)
    l0, l1, wl0, wl1 = axis(xn[:, v], D)
    plane = [(y0 * W + x0, wx0 * wy0), (y0 * W + x1, wx1 * wy0), (y1 * W + x0, wx0 * wy1), (y1 * W + x1, wx1 * wy1)]
    return plane, [(l0, wl0), (l1, wl1)]


def run_stats(xn, grid, active=None):
    """Atomics per tap for merge blocks of B consecutive rows (B = 1: one per row, as an unmerged scatter issues them):
    a row adds to the open run of its tap when the texel is the one the previous active row of the block hit."""
    rows = torch.arange(xn.shape[0], device=xn.device)
    out = {"plane": {B: 0 for B in MERGE_ROWS}, "line": {B: 0 for B in MERGE_ROWS}}
    hist = {"plane": torch.zeros(6, dtype=torch.int64), "line": torch.zeros(6, dtype=torch.int64)}
    for k in range(3):
        plane, line = tap_keys(xn, grid, k)
        for kind, taps in (("plane", plane), ("line", line)):
            for key, w in taps:
                on = w != 0
                if active is not None:
                    on &= active
                idx, key = rows[on], key[on]
                if idx.numel() == 0:
                    continue
                same = torch.zeros_like(key, dtype=torch.bool)
                same[1:] = key[1:] == key[:-1]
                for B in MERGE_ROWS:
                    blk = idx // B
                    cont = same.clone()
                    cont[1:] &= blk[1:] == blk[:-1]
                    out[kind][B] += int((~cont).sum())
                # unbounded run lengths (B = infinity): 1, 2, 3, 4, 5-8, 9+
                starts = torch.nonzero(~same).flatten()
                lens = torch.diff(torch.cat([starts, starts.new_tensor([key.numel()])]))
                edges = lens.new_tensor([1, 2, 3, 4, 5, 9])
                hist[kind] += torch.bincount(torch.bucketize(lens, edges, right=True) - 1, minlength=6)[:6].cpu()
    return out, {kind: h.tolist() for kind, h in hist.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    g.build()
    from tensoir_b200 import ops
    from tensoir_b200.optim import FusedAdam
    from tensoir_b200.static_step import StaticTrainStep, lr_tensors
    from tensoir_b200.synthetic import make_lego_model, hemisphere_poses, training_batch, n_samples_for
    from torch.profiler import profile, ProfilerActivity
    grid, batch = 300, 4096
    dev = torch.device("cuda", 0)
    model = make_lego_model(grid, dev)
    opt = FusedAdam(lr_tensors(model.get_optparam_groups(0.02, 0.001), dev), betas=(0.9, 0.99))
    opt.density_l1(model, bench.L1_WEIGHT)
    model.__dict__["_tir_counters"] = ops.new_counters(dev)
    model.__dict__["_tir_lean"] = True
    poses = hemisphere_poses(100)
    hb = [(r.to(dev), l.to(dev)) for r, l in (training_batch(poses, batch, i) for i in range(8 + 2 * a.replays + 8))]
    target = torch.full((batch, 3), 0.5, device=dev)
    st = StaticTrainStep(model, opt, batch, n_samples_for(grid), bench.Args,
                         lambda r, m: bench.loss_of(r, target, m, l1_in_optimizer=True), device=dev)
    st.calibrate(hb[:8])
    st.capture(warmup=3)
    it = iter(hb[8:])
    for _ in range(3):
        st.run(*next(it))
    st.reserve(4.0)
    for _ in range(3):
        st.run(*next(it))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.replays):
        st.run(*next(it))
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.replays
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.replays):
            st.run(*next(it))
        torch.cuda.synchronize()
    st.flush()
    kernels = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", 0.0)
        if us > 0:
            kernels[e.key] = kernels.get(e.key, 0.0) + us / a.replays
    total = sum(kernels.values())
    gpu = torch.cuda.get_device_name(0)
    print(f"{gpu}; step {step_ms:.3f} ms (CUDA events, {a.replays} replays, profiler off); "
          f"kernels {total / 1e3:.3f} ms per replay under the profiler")
    print(f"{'us/replay':>10} {'share':>6}  kernel")
    for name, us in sorted(kernels.items(), key=lambda kv: -kv[1]):
        print(f"{us:10.1f} {100 * us / total:5.1f}%  {name[:110]}")
    sc = sum(us for name, us in kernels.items() if any(s in name for s in SCATTERS))
    print(f"VM-factor gradient scatters: {sc:.1f} us per replay ({100 * sc / total:.1f}% of the kernel time)")
    stats = [int(v) for v in st.static["stats"].tolist()]
    print(f"lists of the last replay: valid {stats[0]}, appearance {stats[1]}, secondary appearance {stats[3]}; "
          f"capacities {st.capacities()}")
    ws = model.__dict__["_tir_primary_ws"]
    gs = [int(v) for v in model._host_geom["grid"]]
    n_valid, n_app = stats[0], stats[1]
    runs = {}
    for name, xn, act in (("valid v_xn (density_bwd, g_feat != 0)", ws.t["v_xn"][:n_valid], ws.t["g_feat"][:n_valid] != 0),
                          ("appearance a_xn", ws.t["a_xn"][:n_app], None),
                          ("appearance a_xj", ws.t["a_xj"][:n_app], None)):
        atom, hist = run_stats(xn, gs, act)
        runs[name] = {"atomics": atom, "run_length_hist": hist}
        print(f"{name}: tap atomics per step for merge blocks of B rows (runs cut at block ends)")
        for kind in ("plane", "line"):
            base = atom[kind][1]
            cells = ", ".join(f"B={B}: {n} ({base / max(n, 1):.2f}x fewer)" for B, n in atom[kind].items())
            print(f"  {kind}: {cells}")
            print(f"  {kind} run lengths (1, 2, 3, 4, 5-8, 9+): {hist[kind]}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"gpu": gpu, "step_ms": step_ms, "kernels_us": kernels, "scatters_us": sc, "stats": stats,
                       "runs": runs}, fh, indent=1)


if __name__ == "__main__":
    main()
