"""Camera-path frames on the H100: the lego box model at a small grid, 64x64 views.

The primary render composites with float atomics, so where two frames are compared to the bit the model's forward of
the first is replayed in the second (test_material_edit_gpu.Replay); everything after it (rays, draws, the visibility
lists in slot order, their marches, shading and the composite) runs again.  The background lookup uses acosf / atan2f,
whose device and host results may differ in the last bit, so device frames agree with the host build to rounding; the
shadow ratio, which uses only correctly rounded operations, agrees to the bit."""
import math
import os
import types

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from test_material_edit_gpu import Replay

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GRID, HW = 64, 64


@pytest.fixture(scope="module")
def model():
    import __graft_entry__ as g
    g.build()
    from tensoir_b200.synthetic import make_lego_model
    return make_lego_model(GRID, DEV, lights=("000", "090"))


def views(n=2, size=HW):
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    return SyntheticViews(hemisphere_poses(n), size, size, light_names=["a"])


def one_texel(H, W, row, col, rgb=(40.0, 36.0, 30.0)):
    arr = np.zeros((H, W, 3), np.float32)
    arr[row, col] = rgb
    return arr


def smooth_map(H=16, W=32, seed=3):
    g = np.random.default_rng(seed)
    return (0.2 + g.uniform(0, 1, (H, W, 3)) ** 3 * 2).astype(np.float32)


def frame(m, env, names, rays, angle, ground_z=None, S=64, shadow=False, box=None):
    from tensoir_b200 import camera_path as P
    gen = torch.Generator(DEV)
    return P.render_frame(m, env, names, rays, angle, torch.ones(3, device=DEV), 1500, gen, 7, ground_z, box, S,
                          shadow=shadow)


def rays_of(ds, i):
    from tensoir_b200 import camera_path as P
    W, H = ds.img_wh
    return P.frame_rays(ds.poses[i], W, H, ds.focal, DEV)


def test_generate_rays_reproduce_the_dataset(model):
    ds = views(3, 48)
    for i in range(len(ds)):
        assert (rays_of(ds, i).cpu() - ds[i]["rays"]).abs().max() < 1e-6


def test_identity_is_relight_shade(model):
    """Rotation 0, no ground: the frame is relight_visibility(ordered=True) + relight_shade on the same rays and
    draws, to the bit."""
    from tensoir_b200 import relighting as R
    from tensoir_b200.relight import Environment_Light
    env = Environment_Light({"s": smooth_map()}, device=DEV)
    rays = rays_of(views(), 0)
    rep = Replay(model)
    try:
        wb, wo, _ = frame(model, env, ["s"], rays, 0.0)
        rep.i = 0
        envs, keep = R.env_tables(env, ["s"])
        gen = torch.Generator(DEV).manual_seed(7)
        want = (torch.empty_like(wb), torch.empty_like(wo))
        for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(model, rays, 1500):
            r, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(rays[s:e], (depth, normal, albedo, rough,
                                                                                         fresnel, acc))
            u = torch.rand(1, e - s, 64, device=DEV, dtype=torch.float64, generator=gen)
            vis = R.relight_visibility(model, envs, 1, r, depth, normal, acc, u, 64, 0.5, "nerv", ordered=True)
            R.relight_shade(envs, 1, r, normal, albedo, rough, fresnel, acc, 64, 0.5, torch.ones(3, device=DEV), vis,
                            "nerv", want, s)
    finally:
        model.forward = rep.fwd
    assert torch.equal(wb, want[0]) and torch.equal(wo, want[1])
    assert (wo < 1).any() and (wb != wo).any()


def test_rotation_is_a_column_roll(model):
    """A one-texel map rotated by 360 k / W lights the object as the map rolled by k columns does at rotation 0 (the
    texel of E(w @ R(a)) at texel centre w is k columns on), except where the two visibilities differ (the rotated
    direction is rounded differently).  The background is get_light at d @ R(a); a rolled map is not the same
    lookup there, since get_light spreads W - 1 columns over the full turn (align_corners)."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200 import relighting as R
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.relight_utils import linear2srgb_torch
    H, W, k = 16, 32, 5
    a = 360.0 * k / W
    bright = one_texel(H, W, 4, 9)
    env = Environment_Light({"rot": bright, "roll": np.roll(bright, -k, axis=1).copy()}, device=DEV)
    rays = rays_of(views(), 1)
    rep = Replay(model)
    try:
        _, wo_rot, _ = frame(model, env, ["rot"], rays, a)
        rep.i = 0
        _, wo_roll, _ = frame(model, env, ["roll"], rays, 0.0)
        # per-pixel visibility of both, from the same primary maps
        rep.i = 0
        hit = torch.zeros(rays.shape[0], dtype=torch.bool, device=DEV)
        dv = torch.zeros(rays.shape[0], device=DEV)
        for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(model, rays, 1500):
            r, (depth, normal, _, _, _, acc) = R.chunk_inputs(rays[s:e], (depth, normal, albedo, rough, fresnel, acc))
            u = torch.rand(1, e - s, 8, device=DEV, dtype=torch.float64)
            mv = []
            for tables in (P.rotated_env_tables(env, ["rot"], a), R.env_tables(env, ["roll"])):
                _, pos, vis = R.relight_visibility(model, tables[0], 1, r, depth, normal, acc, u, 8, 0.5, "nerv",
                                                   ordered=True)
                mv.append(torch.where(pos[0] >= 0, vis[pos[0].clamp(min=0).long()], torch.zeros_like(vis[:1])).mean(1))
            dv[s:e] = (mv[0] - mv[1]).abs()
            hit[s:e] = acc > 0.5
    finally:
        model.forward = rep.fwd
    boundary = dv > 1e-3
    assert hit.sum() > 200 and (wo_rot[0][hit] < 1).any()
    assert boundary[hit].float().mean() < 0.01
    assert (wo_rot[0] - wo_roll[0])[~boundary].abs().max() < 2e-5
    # the background at d @ R(a), on the pixels the object leaves
    env2 = Environment_Light({"s": smooth_map()}, device=DEV)
    wb, _, _ = frame(model, env2, ["s"], rays, 73.0)
    rep_acc = torch.cat([c[1][6].reshape(-1) for c in rep.calls]) if rep.calls else None
    d = rays[:, 3:] @ P.rotation_matrix(73.0).to(DEV)
    want = linear2srgb_torch(env2.get_light("s", d).clamp(0, 1))
    bg = rep_acc <= 0.9
    assert bg.sum() > 500 and (wb[0][bg] - want[bg]).abs().max() < 1e-5


def test_convention_matches_light_rotation(model):
    """light_envmaps(model)[1] (the reference's '090' light) is light_envmaps(model)[0] looked up through the path's
    rotation by 90 degrees: 128 columns at 512 wide; and the object lit by map 0 rotated by 90 sees map 1's
    radiance from every texel direction."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200.mesh import light_envmaps
    maps = light_envmaps(model)
    Hm, Wm = maps.shape[1:3]
    _, dirs = model.generate_envir_map_dir(Hm, Wm)
    rot = P.rotation_matrix(90.0)
    d = dirs.reshape(-1, 3) @ rot                                          # w @ R(a): where map 0 is read
    theta = torch.atan2(d[:, 1], d[:, 0])
    col = torch.round((math.pi - theta) / (2 * math.pi / Wm) - 0.5).long() % Wm
    row = torch.arange(Hm).repeat_interleave(Wm)
    own = torch.arange(Wm).repeat(Hm)
    assert torch.equal((col - own) % Wm, torch.full_like(col, (Wm - 128) % Wm)) or \
        torch.equal((col - own) % Wm, torch.full_like(col, 128))
    looked = maps[0].reshape(Hm, Wm, 3)[row, col].reshape(Hm, Wm, 3)
    assert (looked - maps[1]).abs().max() < 1e-5
    # through the rotated direction table: texel k of map 0 arrives from dir_k @ R^T, where light 1 shines texel k
    from tensoir_b200.relight import Environment_Light
    env = Environment_Light({"l0": maps[0].cpu().numpy()}, device=DEV)
    _, keep = P.rotated_env_tables(env, ["l0"], 90.0)
    lit = model.get_light_rgbs(keep[-1], device=DEV)[1].clamp(min=0)
    assert (lit - maps[0].reshape(-1, 3)).abs().max() < 1e-5


def test_empty_field(model):
    """No density anywhere: every shadow ratio is exactly 1 and the frame is its rotated background."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.synthetic import make_lego_model
    m = make_lego_model(GRID, DEV)
    with torch.no_grad():
        for p in list(m.density_plane) + list(m.density_line):
            p.zero_()
    m.density_shift = -1e4                                                 # softplus(-1e4) is 0 in fp32
    env = Environment_Light({"s": smooth_map()}, device=DEV)
    rays = rays_of(views(), 0)
    z = P.default_ground_z(m)
    wb, wo, r = frame(m, env, ["s"], rays, 40.0, z, shadow=True)
    bg, _, _ = frame(m, env, ["s"], rays, 40.0)
    assert (r == 1).all() and (wo == 1).all()
    assert torch.equal(wb, bg)


def test_sun_shadow_on_the_ground(model):
    """A one-texel sun at 45 degrees elevation: ground points whose sun ray meets a lego box are dark, points more than
    two voxels from the shadow's edge whose ray misses are lit (synthetic.trace_boxes, float64)."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, trace_boxes
    H, W = 18, 36                                                           # row 4 is at 45 degrees elevation
    env = Environment_Light({"sun": one_texel(H, W, 4, 7)}, device=DEV)
    sun = env.hdr_dir["sun"].reshape(-1, 3)[4 * W + 7].double().cpu()
    assert abs(math.degrees(math.asin(sun[2])) - 45) < 1e-4
    z = P.default_ground_z(model)
    ds = SyntheticViews(hemisphere_poses(3, radius=5.0), 96, 96, light_names=["a"])
    vox = 3.0 / (GRID - 1)
    far_hit = far_miss = 0
    for i in range(len(ds)):
        rays = rays_of(ds, i)
        _, _, r = frame(model, env, ["sun"], rays, 0.0, z, S=4, shadow=True)
        rc = rays.double().cpu()
        t = (z - rc[:, 2]) / rc[:, 5]
        ground = (rc[:, 5] < 0) & (t > 0)
        p = rc[:, :3] + t[:, None] * rc[:, 3:]
        offs = [(0, 0)] + [(2 * vox * math.cos(q), 2 * vox * math.sin(q)) for q in np.linspace(0, 2 * math.pi, 16,
                                                                                                 endpoint=False)]
        hits = []
        for dx, dy in offs:
            q = p + torch.tensor([dx, dy, 0.0], dtype=torch.float64)
            hits.append(trace_boxes(torch.cat([q, sun.expand_as(q)], 1).float())[0])
        hits = torch.stack(hits)
        # the primary ray itself must reach the ground: not hidden behind the object
        seen = ground & ~trace_boxes(rays.cpu())[0]
        rr = r[0].cpu().mean(1)
        sure_hit = seen & hits.all(0)
        sure_miss = seen & ~hits.any(0)
        assert (rr[sure_hit] < 0.01).all() and (rr[sure_miss] > 0.99).all()
        far_hit += int(sure_hit.sum())
        far_miss += int(sure_miss.sum())
    assert far_hit >= 10 and far_miss > 1000


def test_device_matches_host_build(model, tmp_path, monkeypatch):
    from tensoir_b200 import camera_path as P
    from tensoir_b200.relight import Environment_Light
    arr = smooth_map(16, 32, 5)
    env_d = Environment_Light({"s": arr}, device=DEV)
    env_h = Environment_Light({"s": arr}, device="cpu")
    rays = rays_of(views(), 1)[:3000].contiguous()
    n, S, a = rays.shape[0], 64, 25.0
    z = P.default_ground_z(model)
    box = P.ground_box(model)
    u = torch.rand(1, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    envs, keep = P.rotated_env_tables(env_d, ["s"], a)
    table = P.ground_table(box, DEV)
    bins, pos, vis = P.ground_visibility(model, envs, 1, rays, z, box, u.to(DEV), S, "nerv", table)
    acc = torch.rand(n, device=DEV)
    wo = torch.rand(1, n, 3, device=DEV)
    wb, sh = torch.empty(1, n, 3, device=DEV), torch.empty(1, n, 3, device=DEV)
    P.path_composite(envs, 1, rays, acc, a, z, (bins, pos, vis), S, "nerv", (wb, wo), 0, sh)
    assert (pos >= 0).any() and (pos == -2).any() and (sh < 0.99).any()
    host = build_host_lib(tmp_path, "host_relight.cpp", "host_path.cpp")
    use_host(monkeypatch, host, lambda *a_, **k: (_ for _ in ()).throw(AssertionError("host march")))
    envs_h, keep_h = P.rotated_env_tables(env_h, ["s"], a)
    # the sample kernel: the same bins and pos codes, the list the host's in slot order
    hb, hp = torch.empty(1, n, S, dtype=torch.int32), torch.empty(1, n, S, dtype=torch.int32)
    lo, ld = torch.empty(n * S, 3), torch.empty(n * S, 3)
    cnt = torch.zeros(1, dtype=torch.int64)
    import ctypes as C
    f3 = lambda v: (C.c_float * 3)(*v)                                    # noqa: E731
    rays_h = rays.cpu()
    assert host.tir_ground_sample(envs_h, 1, C.c_void_p(rays_h.data_ptr()), n, z, f3(box[0]), f3(box[1]), S,
                                  C.c_void_p(u.data_ptr()), C.c_void_p(hb.data_ptr()), C.c_void_p(hp.data_ptr()),
                                  C.c_void_p(lo.data_ptr()), C.c_void_p(ld.data_ptr()), n * S,
                                  C.c_void_p(cnt.data_ptr()), None) == 0
    assert torch.equal(bins.cpu(), hb) and torch.equal(pos.cpu(), hp)          # slot order on both
    # the composite on the same bins, pos and vis
    hwb, hsh = torch.empty(1, n, 3), torch.empty(1, n, 3)
    P.path_composite(envs_h, 1, rays.cpu(), acc.cpu(), a, z, (hb, hp, vis.cpu()), S, "nerv", (hwb, wo.cpu()), 0, hsh)
    assert torch.equal(sh.cpu(), hsh)
    # acosf / atan2f may differ in the last bit between the builds; the bilinear weights carry that (times the map's
    # texel contrast) and sRGB's slope, up to 12.92, multiplies it
    assert (wb.cpu() - hwb).abs().max() < 1e-5
    del keep, keep_h


def test_frames_are_reproducible(model):
    from tensoir_b200 import camera_path as P
    from tensoir_b200.relight import Environment_Light
    env = Environment_Light({"s": smooth_map(), "t": smooth_map(seed=9)}, device=DEV)
    rays = rays_of(views(), 0)
    z = P.default_ground_z(model)
    rep = Replay(model)
    try:
        a = frame(model, env, ["s", "t"], rays, 17.0, z, shadow=True)
        rep.i = 0
        b = frame(model, env, ["s", "t"], rays, 17.0, z, shadow=True)
    finally:
        model.forward = rep.fwd
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert (a[2] < 0.9).any()


def test_render_path_end_to_end(model, tmp_path):
    """An 8-frame turntable under the model's learned lights with the ground: 8 frames per map and side."""
    from tensoir_b200 import camera_path as P
    ds = views(1, 48)
    centre = model.aabb.detach().double().mean(0).cpu().numpy()
    r, el, az = P.orbit_of(ds.poses[0], centre)
    poses = P.orbit_poses(8, r, el, centre, start_deg=az)
    args = types.SimpleNamespace(out=str(tmp_path), batch_size=2048, light="learned")
    P.render_path(ds, args, poses, P.frame_angles(8, (0.0, 360.0)), tensoIR=model, ground_z=True)
    for name in ("learned_000", "learned_090"):
        for sub in ("with_bg", "without_bg"):
            assert sorted(os.listdir(tmp_path / name / sub)) == [f"{f:04d}.png" for f in range(8)]
    try:
        import imageio  # noqa: F401
        assert (tmp_path / "learned_000.mp4").exists()
    except ImportError:
        pass


def test_rejections(model, tmp_path):
    from tensoir_b200 import camera_path as P
    from tensoir_b200.synthetic import make_lego_model
    ds = views(1, 16)
    poses = ds.poses[:1]
    base = dict(out=str(tmp_path), batch_size=1024, light="learned")
    for extra in (dict(sampling="mis"), dict(indirect_samples=2)):
        with pytest.raises(ValueError):
            P.render_path(ds, types.SimpleNamespace(**base, **extra), poses, [0.0], tensoIR=model)
    general = make_lego_model(32, DEV, lights=("a", "b"), general=True)
    with pytest.raises(ValueError, match="fit_lights"):
        P.render_path(ds, types.SimpleNamespace(**base), poses, [0.0], tensoIR=general)
    assert not os.listdir(tmp_path)
