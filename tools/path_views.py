"""Time camera-path frames on the lego scene and print one JSON line per setting: seconds per frame by phase of
camera_path.render_frame (rays, primary render, object sample + march, object shade, ground sample + march (with the
ground's march timed on its own), composite) and the PNG write, for one environment map with the ground off and then
on.  Each setting renders one untimed frame, then ``--frames`` timed frames of an orbit with the map turning.  Every
phase ends in a synchronise.  The card's name and power limit are printed with the numbers.  ``--rig`` times
camera_path.render_rig_frame instead, the same phases under two rigs turning with the orbit, one hard directional light
and one sphere light of 64 samples, with the ground off and then on.

    python tools/path_views.py [--grid 300] [--size 800] [--frames 3] [--batch 4096] [--rig]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=300)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--rig", action="store_true", help="time frames under analytic light rigs instead of a map")
    a = ap.parse_args()
    if a.frames < 3:
        raise SystemExit("--frames: at least 3 timed frames")
    if not torch.cuda.is_available():
        raise SystemExit("tools/path_views.py measures on the GPU: no CUDA device found")
    import __graft_entry__ as g
    g.build()
    from eval_views import gpu_info
    from tensoir_b200 import camera_path as P
    from tensoir_b200 import lighting as LT
    from tensoir_b200 import relighting as R
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    dev = "cuda:0"
    model = make_lego_model(a.grid, dev, lights=("000", "120"))
    rng = np.random.default_rng(5)
    env = Environment_Light({"sky": (0.3 + rng.uniform(0, 1, (64, 128, 3)) ** 4 * 4).astype(np.float32)}, device=dev)
    ds = SyntheticViews(hemisphere_poses(1), a.size, a.size, light_names=["a"])
    centre = model.aabb.detach().double().mean(0).cpu().numpy()
    r, el, az = P.orbit_of(ds.poses[0], centre)
    n_frames = a.frames + 1
    poses = P.orbit_poses(n_frames, r, el, centre, start_deg=az)
    angles = P.frame_angles(n_frames, (0.0, 360.0))
    gpu, power = gpu_info()
    scale = torch.ones(3, device=dev)
    gen = torch.Generator(dev)

    state = {}

    def tick(phase=None):
        torch.cuda.synchronize()
        t = time.perf_counter()
        if phase is not None:
            state["ph"][phase] = state["ph"].get(phase, 0.0) + t - state["t"]
        state["t"] = t

    march = R.march_list

    def timed_march(*args, **kw):
        tick("ground_sample" if state.get("in_ground") else "object_sample")
        out = march(*args, **kw)
        tick("ground_march" if state.get("in_ground") else "object_march")
        return out

    def timed_ground(fn):
        def run(*args, **kw):
            state["in_ground"] = True
            try:
                return fn(*args, **kw)
            finally:
                state["in_ground"] = False
        return run

    R.march_list = timed_march
    P.ground_visibility = timed_ground(P.ground_visibility)
    P.ground_lights_visibility = timed_ground(P.ground_lights_visibility)
    if a.rig:
        rigs = {"hard_directional": LT.load_rig({"sun": {"lights": [
                    {"type": "directional", "direction": [0.3, -0.4, 0.85], "irradiance": 3.0}]}}),
                "sphere_64": LT.load_rig({"lamp": {"lights": [
                    {"type": "point", "position": [2.0, -1.5, 2.5], "intensity": 40.0, "radius": 0.3,
                     "samples": 64}]}})}
        z_obj = LT.shadow_table(LT.default_shadow_far(model), dev)
        settings = [(name, ground) for name in rigs for ground in (None, P.default_ground_z(model))]
    else:
        settings = [("sky", ground) for ground in (None, P.default_ground_z(model))]
    for name, ground in settings:
        if a.rig:
            frames_rig = P.frame_rigs(rigs[name], angles, model.aabb)
            names = list(rigs[name])
        else:
            names = ["sky"]
        with tempfile.TemporaryDirectory() as out:
            totals = {}
            for f in range(n_frames):
                state["ph"] = {}
                tick()
                rays = P.frame_rays(poses[f], a.size, a.size, ds.focal, dev)
                tick("rays")
                if a.rig:
                    wb, wo, _ = P.render_rig_frame(model, frames_rig[f], rays, scale, a.batch, gen, 20211202, ground,
                                                   shadow_table_z=z_obj, timer=tick)
                else:
                    wb, wo, _ = P.render_frame(model, env, ["sky"], rays, angles[f], scale, a.batch, gen, 20211202,
                                               ground, timer=tick)
                tick()
                P._write_frame(out, names, f, a.size, a.size, wb, wo)
                tick("png_write")
                if f > 0:                                            # frame 0 is the untimed warm-up
                    for k, v in state["ph"].items():
                        totals[k] = totals.get(k, 0.0) + v
        per = {k: v / a.frames for k, v in totals.items()}
        # render_frame's own phases end after the march: what is left of them after it belongs to the sample
        per["object_sample"] = per.get("object_sample", 0.0) + per.pop("object_visibility", 0.0)
        if ground is not None:
            per["ground_sample"] = per.get("ground_sample", 0.0) + per.pop("ground", 0.0)
        light = (dict(rig=name, samples=LT.slots_per_ray(rigs[name][names[0]])) if a.rig else
                 dict(maps=1, samples=P.NUM_SAMPLES))
        print(json.dumps(dict(gpu=gpu, power_limit=power, grid=a.grid, size=a.size, batch=a.batch, **light,
                              ground="off" if ground is None else f"z={ground:.4f}",
                              frames=a.frames, seconds_per_frame={k: round(v, 4) for k, v in sorted(per.items())},
                              total=round(sum(per.values()), 4))))


if __name__ == "__main__":
    main()
