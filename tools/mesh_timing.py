"""Time the native mesh export on the 300^3 synthetic lego scene and print one JSON line.

    python tools/mesh_timing.py [--grid 300] [--reps 20] [--host] [--asset] [--glb]

Reports getDenseAlpha, the marching-cubes calls (tir_marching_cubes_count + _emit, CUDA events over repeated
launches after warm-up, outputs preallocated: the calls are issued back to back, so host launch overhead can show in
these figures and they are an upper bound on the kernels' time), the device time of each kernel those calls launch
(torch.profiler, same launches), the device-to-host copy of the PLY body, the PLY write, V and F, the
achieved read bandwidth against the volume's X*Y*Z*4 bytes, and the card name and power limit read in the same run.
--host also times the host build of the same C ABI (tests/host_mesh.cpp, g++ -O2, one thread) on the same volume: our
CPU build, not the reference (whose skimage path is not measured here).  --asset also times the steps of
mesh.export_asset on the same model, three runs after a warm-up, each step synchronised, wall clock, with each run's
total: the surface (getDenseAlpha and the two marching-cubes calls), the derived normals at the vertices, the probe
forward, the record packing with its device-to-host copy, the PLY write, the environment maps with their .hdr writes;
plus V and the unprobed count.  --glb times gltf.export_asset_glb's steps the same way (T = 4096, one warm-up and
three timed runs): the surface, then summed over the texel chunks the texels, their derived normals, the probe forward
and the encode, then the corners, the device-to-host copy, the PNG encode and the .glb write; plus F, the texel count,
the unprobed count and the file size.  Compiled artefacts and written files go to a temporary directory.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

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


def _events(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def _kernel_times(fn, reps):
    """device time per call of every kernel / memset ``fn`` launches (torch.profiler), without host launch overhead"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us > 0:                      # names cut to 80 characters: instantiations that share a prefix add up
            out[e.key[:80]] = out.get(e.key[:80], 0.0) + us / reps / 1e3
    return {k: round(v, 4) for k, v in out.items()}


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, round((time.perf_counter() - t0) * 1e3, 3)


def _asset_timing(model, tmp, runs=3):
    """mesh.export_asset's steps in its order, as it runs them (the PLY written without fsync), after one warm-up run:
    per timed run the wall time of each step (synchronised before and after) and of the whole run, so that the steps of
    a run add up to its total"""
    from tensoir_b200 import mesh
    from tensoir_b200.relight import write_hdr
    path = os.path.join(tmp, "lego_asset.ply")

    def write():
        with open(path, "wb") as f:
            f.write(data)

    def envmaps():
        for q, rgb in zip(mesh.envmap_paths(path, model.light_num), mesh.light_envmaps(model).cpu().numpy()):
            write_hdr(q, rgb)
    out = []
    for _ in range(runs + 1):
        t = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        (pts, faces, v), t["surface_ms"] = _wall(lambda: mesh.asset_surface(model))
        n, t["normals_ms"] = _wall(lambda: mesh.vertex_normals(model, v))
        p, t["probe_forward_ms"] = _wall(lambda: mesh.probe(model, v, n))
        data, t["pack_and_d2h_ms"] = _wall(lambda: mesh.asset_ply_bytes(pts, faces, p["normal"], p["albedo"],
                                                                      p["roughness"], p["probed"]))
        _, t["ply_write_ms"] = _wall(write)
        _, t["envmaps_ms"] = _wall(envmaps)
        t["total_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
        out.append(t)
    return dict(runs=out[1:], V=int(pts.shape[0]), rays=int(mesh.has_normal(n).sum()),
                unprobed=int(pts.shape[0] - p["probed"].sum()), asset_ply_bytes=len(data),
                probe_offset=mesh.probe_offset(model))


def _glb_timing(model, tmp, T=4096, runs=3):
    """gltf.export_asset_glb's steps in its order (the .glb written without fsync, no .hdr files: --asset times
    those), after one warm-up run: per timed run the wall time of each step, each synchronised before and after, the
    per-chunk steps summed over the chunks, and of the whole run"""
    from tensoir_b200 import gltf, mesh
    path = os.path.join(tmp, "lego_asset.glb")
    out = []
    for _ in range(runs + 1):
        t = dict.fromkeys(("texels_ms", "texel_normals_ms", "probe_forward_ms", "encode_ms"), 0.0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        (_, faces, v), t["surface_ms"] = _wall(lambda: mesh.asset_surface(model))
        F = int(faces.shape[0])
        s = gltf.atlas_cell_size(F, T)
        total, unprobed = gltf.texel_count(F, s), 0
        images = gltf.new_images(T, v.device)
        for first in range(0, total, gltf.TEXEL_CHUNK):
            n = min(gltf.TEXEL_CHUNK, total - first)
            (_, pos), dt = _wall(lambda: gltf.atlas_texels(faces, v, T, s, first, n))
            t["texels_ms"] += dt
            nrm, dt = _wall(lambda: mesh.vertex_normals(model, pos))
            t["texel_normals_ms"] += dt
            p, dt = _wall(lambda: mesh.probe(model, pos, nrm))
            t["probe_forward_ms"] += dt
            _, dt = _wall(lambda: gltf.atlas_encode(faces, v, T, s, first, p["albedo"], p["roughness"], p["normal"],
                                                    p["probed"], images))
            t["encode_ms"] += dt
            unprobed += n - int(p["probed"].sum())
        corners, t["corners_ms"] = _wall(lambda: gltf.atlas_corners(faces, v, T, s))
        (host, imgs), t["d2h_ms"] = _wall(lambda: ({k: c.cpu().numpy() for k, c in corners.items()},
                                                   images.cpu().numpy()))
        pngs, t["png_encode_ms"] = _wall(lambda: [gltf.png_bytes(im) for im in imgs])

        def write():
            with open(path, "wb") as f:
                f.write(gltf.glb_bytes(host, pngs))
        _, t["glb_write_ms"] = _wall(write)
        for k in ("texels_ms", "texel_normals_ms", "probe_forward_ms", "encode_ms"):
            t[k] = round(t[k], 3)
        t["total_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
        out.append(t)
    return dict(runs=out[1:], texture_size=T, cell=s, F=F, texels=total, unprobed=unprobed,
                glb_bytes=os.path.getsize(path), png_bytes=[len(q) for q in pngs])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=300)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--asset", action="store_true")
    ap.add_argument("--glb", action="store_true")
    a = ap.parse_args()
    from tensoir_b200 import _lib, mesh
    from tensoir_b200.synthetic import make_lego_model
    lib = _lib.load()
    dev = torch.device("cuda")
    model = make_lego_model(a.grid, dev)
    model.getDenseAlpha()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    alpha, _ = model.getDenseAlpha()
    torch.cuda.synchronize()
    t_alpha = (time.perf_counter() - t0) * 1e3
    vol = alpha.contiguous()
    X, Y, Z = vol.shape
    level = 0.005
    sp = [float(v) for v in mesh.ply_spacing(tuple(vol.shape), model.aabb)]
    nbytes = C.c_int64(0)
    _lib.check(lib.tir_marching_cubes_work_size(X, Y, Z, C.byref(nbytes)), "work_size")
    work = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    st = _lib.stream_ptr()

    def count():
        _lib.check(lib.tir_marching_cubes_count(_lib.dptr(vol), X, Y, Z, level, _lib.dptr(work, torch.uint8),
                                                nbytes.value, _lib.dptr(totals, torch.int64), st), "count")
    count()
    V, F = (int(t) for t in totals.tolist())
    verts = torch.empty(V, 3, device=dev)
    faces = torch.empty(F, 3, dtype=torch.int32, device=dev)

    def emit():
        _lib.check(lib.tir_marching_cubes_emit(_lib.dptr(vol), X, Y, Z, level, sp[0], sp[1], sp[2],
                                               _lib.dptr(work, torch.uint8), nbytes.value, V, F, _lib.dptr(verts),
                                               _lib.dptr(faces, torch.int32), st), "emit")
    for _ in range(3):
        count()
        emit()
    t_count = _events(count, a.reps)
    t_emit = _events(emit, a.reps)
    t_both = _events(lambda: (count(), emit()), a.reps)
    kernels = _kernel_times(lambda: (count(), emit()), a.reps)
    # the PLY body: records built on the device, one device-to-host copy, then the write
    body_dev = mesh.ply_bytes(verts, faces, model.aabb)       # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    body_dev = mesh.ply_bytes(verts, faces, model.aabb)
    t_copy = (time.perf_counter() - t0) * 1e3
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "lego.ply")
        t0 = time.perf_counter()
        with open(path, "wb") as f:
            f.write(body_dev)
            f.flush()
            os.fsync(f.fileno())
        t_write = (time.perf_counter() - t0) * 1e3
        host_ms = None
        if a.host:
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            from mesh_helpers import build_host_lib, host_marching_cubes
            hl = build_host_lib(tmp)
            v_np = vol.cpu().numpy()
            t0 = time.perf_counter()
            hv, hf = host_marching_cubes(hl, v_np, level, sp)
            host_ms = (time.perf_counter() - t0) * 1e3
            assert torch.equal(torch.from_numpy(hv), verts.cpu()) and torch.equal(torch.from_numpy(hf), faces.cpu())
        asset = _asset_timing(model, tmp) if a.asset else None
        glb = _glb_timing(model, tmp) if a.glb else None
    name, power = _card()
    vol_bytes = X * Y * Z * 4
    print(json.dumps(dict(
        grid=[X, Y, Z], level=level, V=V, F=F, card=name, power_limit=power,
        dense_alpha_ms=round(t_alpha, 3), mc_count_ms=round(t_count, 4), mc_emit_ms=round(t_emit, 4),
        mc_total_ms=round(t_both, 4), d2h_and_pack_ms=round(t_copy, 3), ply_write_ms=round(t_write, 3),
        ply_bytes=len(body_dev), volume_bytes=vol_bytes,
        mc_volume_read_GBps=round(vol_bytes / (t_both * 1e-3) / 1e9, 1),
        mc_kernels_ms=kernels, mc_kernels_total_ms=round(sum(kernels.values()), 4),
        host_build_ms=None if host_ms is None else round(host_ms, 1), asset=asset, glb=glb)))


if __name__ == "__main__":
    main()
