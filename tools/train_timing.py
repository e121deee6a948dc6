"""Time the phase-1 (radiance-only, is_relight=False) training step and print one JSON line.

    python tools/train_timing.py [--grid 128] [--rays 4096] [--steps 100] [--warmup 10]

The bench scene at ``grid``^3 without an alpha mask (the state of a fresh training run before
update_AlphaMask_list[0]), batches of ``rays`` training rays, loss mse(rgb_map, 0.5), fused torch Adam.  Three forms of
the same step, each from the same initial model on the same batches and the same per-ray jitter:

  modular_eager  the per-op path (march + fused_head + segment sums, torch autograd, host syncs in torch.nonzero)
  fused_eager    the fused radiance node (tir_primary_radiance / _backward), eager
  fused_graph    the fused node captured with the loss, backward and Adam in one CUDA graph (StaticTrainStep)

Times are host wall clock around ``steps`` steps ending in a device synchronise, after ``warmup`` steps.  Every form's
per-step losses are compared with fused_eager's (max relative difference; the script exits non-zero above 2e-3 or if
a replay had to be redone), and the card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=128)
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_timing.py needs a CUDA device")
    import contextlib
    import io
    from tensoir_b200 import Renderer_TensoIR_train, _lib
    from tensoir_b200.static_step import StaticTrainStep
    from tensoir_b200.synthetic import make_lego_model, hemisphere_poses, training_batch, n_samples_for
    dev = "cuda:0"
    _lib.load()
    n_s = n_samples_for(a.grid)
    total = a.warmup + a.steps
    poses = hemisphere_poses(100)
    batches = [tuple(t.to(dev) for t in training_batch(poses, a.rays, it)) for it in range(total)]
    target = torch.full((a.rays, 3), 0.5, device=dev)

    def loss_of(ret):
        return ((ret["rgb_map"] - target) ** 2).mean()

    def model():
        with contextlib.redirect_stdout(io.StringIO()):
            m = make_lego_model(a.grid, dev)
        m.alphaMask = None
        return m

    def eager(modular):
        m = model()
        m.__dict__["_tir_modular"] = modular
        opt = torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), betas=(0.9, 0.99), fused=True)

        def step(it):
            rays, li = batches[it]
            torch.manual_seed(1000 + it)            # the per-ray jitter of step `it`, drawn inside the forward
            ret = Renderer_TensoIR_train(rays, None, li, m, N_samples=n_s, white_bg=True, is_train=True,
                                         is_relight=False, device=dev)
            loss = loss_of(ret)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            return loss.detach()
        return step, m

    def graphed(caps):
        m = model()
        opt = torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), betas=(0.9, 0.99), fused=True, capturable=True)
        # the appearance list grows ~20x while the density forms: the lists are sized by the eager run of the same
        # steps (its workspace grew to fit all of them), so no timed replay overflows and every loss is its step's
        st = StaticTrainStep(m, opt, a.rays, n_s, None, lambda ret, mm: loss_of(ret), device=dev, is_relight=False,
                             cap_valid=caps[0], cap_app=caps[1])
        it_box = [0]
        orig = st._stage_host_randoms

        def stage(slot):
            torch.manual_seed(1000 + it_box[0])      # the same jitter as the eager forms
            orig(slot)
        st._stage_host_randoms = stage
        st.capture(warmup=2)

        def step(it):
            it_box[0] = it
            rays, li = batches[it]
            return st.run(rays, li).detach().clone()
        return step, st

    res = {}
    losses = {}
    caps = None
    for name in ("modular_eager", "fused_eager", "fused_graph"):
        st = m = None
        if name == "fused_graph":
            step, st = graphed(caps)
        else:
            step, m = eager(name == "modular_eager")
        out = [step(it) for it in range(a.warmup)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out += [step(it) for it in range(a.warmup, total)]
        torch.cuda.synchronize()
        res[name + "_ms"] = round((time.perf_counter() - t0) * 1e3 / a.steps, 4)
        if name == "fused_eager":
            ws = m.__dict__["_tir_radiance_ws"]
            caps = (ws.cap_valid, ws.cap_app)
        if st is not None:
            st.flush()
            res["graph_redone"], res["graph_recaptures"] = st.redone, st.recaptures
            res["graph_launches_per_replay"] = st.launches_per_replay
            st.release()
        losses[name] = torch.stack(out).float().cpu()
    ref = losses["fused_eager"]
    for name in ("modular_eager", "fused_graph"):
        res[name + "_loss_max_rel_diff"] = float(((losses[name] - ref).abs() / ref.abs().clamp_min(1e-6)).max())
    res["loss_first_last"] = [float(ref[0]), float(ref[-1])]
    card, power = _card()
    res.update(card=card, power_limit=power, grid=a.grid, rays=a.rays, n_samples=n_s, steps=a.steps,
               warmup=a.warmup, alpha_mask=None)
    print(json.dumps(res))
    # the three forms must compute the same training run at the timed size, or their times are not comparable
    bad = {k: v for k, v in res.items() if k.endswith("_loss_max_rel_diff") and not v < 2e-3}
    if bad or res.get("graph_redone", 0):
        raise SystemExit(f"outputs disagree with fused_eager (limit 2e-3 relative per step) or a replay was redone: "
                         f"{bad}, redone {res.get('graph_redone')}")


if __name__ == "__main__":
    main()
