"""Camera-path frames under analytic light rigs on the H100: the lego box model at a small grid, 64x64 views.

As in test_camera_path_gpu, where two frames are compared to the bit the model's forward of the first is replayed in
the second (test_material_edit_gpu.Replay).  The ground's weights, codes and shadow ratio use only correctly rounded
operations and agree with the host build to the bit; the darkened background goes through powf and agrees to
rounding."""
import ctypes as C
import math
import os
import types

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from test_camera_path_gpu import GRID, frame, one_texel, rays_of, views
from test_lighting_gpu import first_hit
from test_material_edit_gpu import Replay

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def model():
    import __graft_entry__ as g
    g.build()
    from tensoir_b200.synthetic import make_lego_model
    return make_lego_model(GRID, DEV, lights=("000", "090"))


def mixed_setup():
    """One light of each kind, all outside the aabb (+-1.5), the point light soft."""
    from tensoir_b200 import lighting
    from tensoir_b200.lighting import Light, Setup
    return Setup((Light("directional", (2.0, 2.0, 1.8), direction=lighting._unit((0.4, -0.3, 1.0), "")),
                  Light("point", (30.0, 28.0, 25.0), position=(2.2, 0.5, 0.4), extent=0.2, samples=12),
                  Light("spot", (50.0, 50.0, 50.0), position=(-1.0, -2.5, 2.5),
                        direction=lighting._unit((1.0, 2.5, -3.4), ""), cos_inner=math.cos(math.radians(20)),
                        cos_outer=math.cos(math.radians(35)))), background=(0.7, 0.6, 0.5))


def rig_frame(m, rig, rays, ground_z=None, shadow=False, z_obj=None):
    from tensoir_b200 import camera_path as P
    return P.render_rig_frame(m, rig, rays, torch.ones(3, device=DEV), 1500, torch.Generator(DEV), 7, ground_z,
                              shadow=shadow, shadow_table_z=z_obj)


def test_device_matches_host_build(model, tmp_path, monkeypatch):
    from tensoir_b200 import camera_path as P
    from tensoir_b200 import lighting, ops
    setup = mixed_setup()
    rays = rays_of(views(), 1)[:3000].contiguous()
    n = rays.shape[0]
    slots = n * lighting.slots_per_ray(setup)
    z = P.default_ground_z(model)
    box = P.rig_ground_box(model)
    u = torch.rand(slots, 2, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    seen, march = {}, ops.march_density

    def recording(m, o, d, **kw):
        seen.update(o=o.clone(), d=d.clone())
        return march(m, o, d, **kw)

    monkeypatch.setattr(ops, "march_density", recording)
    g, pos, vis = P.ground_lights_visibility(model, setup, rays, z, box, u.to(DEV), "nerv", P.ground_table(box, DEV))
    monkeypatch.setattr(ops, "march_density", march)
    acc = torch.rand(n, device=DEV)
    wo = torch.rand(n, 3, device=DEV)
    wb, sh = torch.empty(n, 3, device=DEV), torch.empty(n, 3, device=DEV)
    P.path_lights_composite(setup, rays, acc, z, (g, pos, vis), "nerv", (wb, wo), 0, sh)
    assert (pos >= 0).any() and (pos == -2).any() and (sh < 0.99).any()
    host = build_host_lib(tmp_path, "host_relight.cpp", "host_lights.cpp", "host_path.cpp", "host_path_lights.cpp")
    use_host(monkeypatch, host, lambda *a_, **k: (_ for _ in ()).throw(AssertionError("host march")))
    hg, hp = torch.empty(slots), torch.empty(slots, dtype=torch.int32)
    lo, ld = torch.empty(slots, 3), torch.empty(slots, 3)
    cnt = torch.zeros(1, dtype=torch.int64)
    f3 = lambda v: (C.c_float * 3)(*v)                                    # noqa: E731
    rays_h = rays.cpu()
    assert host.tir_ground_lights_sample(lighting.light_table(setup), len(setup.lights), C.c_void_p(rays_h.data_ptr()),
                                         n, z, f3(box[0]), f3(box[1]), C.c_void_p(u.data_ptr()),
                                         C.c_void_p(hg.data_ptr()), C.c_void_p(hp.data_ptr()),
                                         C.c_void_p(lo.data_ptr()), C.c_void_p(ld.data_ptr()), slots,
                                         C.c_void_p(cnt.data_ptr()), None) == 0
    # the same weights and codes, and the device's list put in slot order is the host's
    assert torch.equal(g.cpu(), hg) and torch.equal(pos.cpu(), hp)
    m = int(cnt)
    assert torch.equal(seen["o"].cpu(), lo[:m]) and torch.equal(seen["d"].cpu(), ld[:m])
    # the composite on the same g, pos and vis
    hwb, hsh = torch.empty(n, 3), torch.empty(n, 3)
    P.path_lights_composite(setup, rays_h, acc.cpu(), z, (hg, hp, vis.cpu()), "nerv", (hwb, wo.cpu()), 0, hsh)
    assert torch.equal(sh.cpu(), hsh)
    assert (wb.cpu() - hwb).abs().max() < 1e-5                              # powf in the tone map


def test_no_ground_rotation_zero_is_rig_shade(model):
    """No ground, no rotation: a rig frame is rig_visibility (slot order) + rig_shade on the same rays and draws, to
    the bit, for every setup."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200 import lighting
    from tensoir_b200 import relighting as R
    rig = {"mixed": mixed_setup(), "key": lighting.load_rig(
        {"key": {"lights": [{"type": "directional", "direction": [-0.3, 0.6, 0.8], "irradiance": 3.0,
                             "angular_radius_deg": 4.0, "samples": 6}]}})["key"]}
    rays = rays_of(views(), 0)
    rep = Replay(model)
    try:
        wb, wo, _ = rig_frame(model, {k: P.rotated_setup(s, 0.0) for k, s in rig.items()}, rays)
        rep.i = 0
        gen = torch.Generator(DEV).manual_seed(7)
        z = lighting.shadow_table(lighting.default_shadow_far(model), DEV)
        want = (torch.empty_like(wb), torch.empty_like(wo))
        for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(model, rays, 1500):
            r, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(rays[s:e], (depth, normal, albedo, rough,
                                                                                         fresnel, acc))
            for k, setup in enumerate(rig.values()):
                u = torch.rand((e - s) * lighting.slots_per_ray(setup), 2, device=DEV, dtype=torch.float64,
                               generator=gen)
                vis = lighting.rig_visibility(model, setup, r, depth, normal, acc, u, 0.5, "nerv", z, ordered=True)
                lighting.rig_shade(setup, r, normal, albedo, rough, fresnel, acc, 0.5, torch.ones(3, device=DEV), vis,
                                   "nerv", (want[0][k], want[1][k], None), s)
    finally:
        model.forward = rep.fwd
    assert torch.equal(wb, want[0]) and torch.equal(wo, want[1])
    assert (wo < 1).any() and (wb != wo).any()


def _ground_points(rays, z):
    rc = rays.double().cpu()
    t = (z - rc[:, 2]) / rc[:, 5]
    ground = (rc[:, 5] < 0) & (t > 0)
    return ground, rc[:, :3] + t[:, None] * rc[:, 3:]


def longest_chord(o, d, far):
    """The longest run of the segments o + t d, 0 < t < far, inside one lego box (slab test, float64)."""
    from tensoir_b200.synthetic import _lego_boxes
    o, d = o.double(), d.double().expand_as(o)
    inv = 1.0 / torch.where(d == 0, torch.full_like(d, 1e-30), d)
    best = torch.zeros(o.shape[0], dtype=torch.float64)
    for lo, hi, _ in _lego_boxes():
        t0 = (torch.tensor(lo, dtype=torch.float64) - o) * inv
        t1 = (torch.tensor(hi, dtype=torch.float64) - o) * inv
        t_in = torch.minimum(t0, t1).max(dim=1).values.clamp(min=0)
        t_out = torch.minimum(torch.maximum(t0, t1).min(dim=1).values, torch.as_tensor(far, dtype=torch.float64))
        best = torch.maximum(best, (t_out - t_in).clamp(min=0))
    return best


def _offsets(vox):
    """The segment itself and its copies moved by two voxels: 16 ways sideways, up and down."""
    return [(0.0, 0.0, 0.0)] + [(2 * vox * math.cos(q), 2 * vox * math.sin(q), 0.0)
                                for q in np.linspace(0, 2 * math.pi, 16, endpoint=False)] + \
        [(0.0, 0.0, 2 * vox), (0.0, 0.0, -2 * vox)]


def test_shadows_where_the_geometry_says(model):
    """Ground points more than two voxels from a shadow's edge: those whose ray to the light, moved by two voxels in
    any of 18 directions, still crosses at least four voxels of a lego box are dark; those whose ray so moved still
    misses every box are lit (synthetic boxes, float64; a ray that only clips a box's corner crosses too little of the
    64^3 field to be opaque, and one that grazes a face sees the field's blur).  For the point lights the ray is the
    segment to the light.  The low point light beside the object has ground points whose ray passes the light before it
    meets a box: they must be lit (the distance cull)."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200.lighting import Light, Setup
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, trace_boxes
    z = P.default_ground_z(model)
    el = math.radians(45.0)
    sun_dir = (math.cos(el) * math.cos(0.6), math.cos(el) * math.sin(0.6), math.sin(el))
    cases = {"sun": Light("directional", (3.0, 3.0, 3.0), direction=sun_dir),
             "lamp": Light("point", (40.0, 40.0, 40.0), position=(0.6, -0.4, 2.4)),
             "low": Light("point", (40.0, 40.0, 40.0), position=(2.1, 0.3, z + 0.6))}
    rig = {k: Setup((l,)) for k, l in cases.items()}
    ds = SyntheticViews(hemisphere_poses(3, radius=5.0), 96, 96, light_names=["a"])
    vox = 3.0 / (GRID - 1)
    counts = {k: [0, 0] for k in cases}
    passed_light = 0
    for i in range(len(ds)):
        rays = rays_of(ds, i)
        _, _, r = rig_frame(model, rig, rays, z, shadow=True)
        ground, p = _ground_points(rays, z)
        seen = ground & ~trace_boxes(rays.cpu())[0]                         # the primary ray reaches the ground
        for k, (name, l) in enumerate(cases.items()):
            if l.kind == "directional":
                d, dist = torch.tensor(l.direction, dtype=torch.float64).expand_as(p), math.inf
            else:
                to = torch.tensor(l.position, dtype=torch.float64) - p
                dist = to.norm(dim=1)
                d = to / dist[:, None]
            hits, through = [], []
            for off in _offsets(vox):
                q = p + torch.tensor(off, dtype=torch.float64)
                hits.append(first_hit(q, d) < dist)
                through.append(longest_chord(q, d, dist) >= 4 * vox)
            hits, through = torch.stack(hits), torch.stack(through)
            rr = r[k].cpu().mean(1)
            sure_hit, sure_miss = seen & through.all(0), seen & ~hits.any(0)
            assert (rr[sure_hit] < 0.01).all(), (name, float(rr[sure_hit].max()))
            # the low light's rays graze the boxes' tops for long stretches, where the 64^3 field is faint but not
            # empty; a point lit through the distance cull would otherwise be dark (< 0.01)
            assert (rr[sure_miss] > (0.95 if name == "low" else 0.99)).all(), (name, float(rr[sure_miss].min()))
            counts[name][0] += int(sure_hit.sum())
            counts[name][1] += int(sure_miss.sum())
            if name == "low":
                # lit points whose ray, continued past the light, meets a box
                to = torch.tensor(l.position, dtype=torch.float64) - p
                beyond = first_hit(p, to / to.norm(dim=1, keepdim=True)) < math.inf
                passed_light += int((sure_miss & beyond).sum())
    for name, (h, m_) in counts.items():
        assert h >= 10 and m_ > 1000, (name, h, m_)
    assert passed_light > 50


def test_rotation_convention_matches_the_maps(model):
    """A hard directional light at the direction of a one-texel map's texel, with the irradiance that texel delivers,
    turned with the map by 90 degrees: the light's turned direction is the map's rotated table entry, and the object
    is shaded as under that map's path frame (shadow march to 1.5, relight()'s table, for both)."""
    from tensoir_b200 import camera_path as P
    from tensoir_b200 import lighting
    from tensoir_b200.lighting import Light, Setup
    from tensoir_b200.relight import Environment_Light
    H, W, b = 16, 32, 4 * 32 + 9
    env = Environment_Light({"one": one_texel(H, W, 4, 9, (90.0, 80.0, 70.0))}, device=DEV)
    pdf = env.hdr_pdf_return["one"].reshape(-1)[b]
    light = Light("directional", tuple((env.hdr_rgbs["one"].reshape(-1, 3)[b] / pdf).tolist()),
                  direction=tuple(env.hdr_dir["one"].reshape(-1, 3)[b].tolist()))
    turned = P.rotated_setup(Setup((light,)), 90.0)
    table = P.rotated_env_tables(env, ["one"], 90.0)[1][-1]
    assert torch.equal(torch.tensor(lighting.light_table(turned)[0].dir[:]), table[b].cpu())
    rays = rays_of(views(), 1)
    rep = Replay(model)
    try:
        _, wo_map, _ = frame(model, env, ["one"], rays, 90.0, S=4)
        rep.i = 0
        _, wo_rig, _ = rig_frame(model, {"one": turned}, rays, z_obj=lighting.shadow_table(1.5, DEV))
    finally:
        model.forward = rep.fwd
    hit = torch.cat([c[1][6].reshape(-1) for c in rep.calls]) > 0.5
    assert (wo_rig[0] - wo_map[0]).abs().max() < 1e-5
    assert hit.sum() > 200 and ((wo_rig[0] < 1) & (wo_rig[0] > 0))[hit].any()


def test_frames_are_reproducible(model):
    from tensoir_b200 import camera_path as P
    rig = {"a": P.rotated_setup(mixed_setup(), 33.0)}
    rays = rays_of(views(), 0)
    z = P.default_ground_z(model)
    rep = Replay(model)
    try:
        a = rig_frame(model, rig, rays, z, shadow=True)
        rep.i = 0
        b = rig_frame(model, rig, rays, z, shadow=True)
    finally:
        model.forward = rep.fwd
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert (a[2] < 0.9).any()


def test_render_path_with_a_rig_end_to_end(model, tmp_path):
    """An 8-frame turntable under a two-setup rig with the ground: 8 frames per setup and side, and the videos."""
    from tensoir_b200 import camera_path as P
    ds = views(1, 48)
    centre = model.aabb.detach().double().mean(0).cpu().numpy()
    r, el, az = P.orbit_of(ds.poses[0], centre)
    poses = P.orbit_poses(8, r, el, centre, start_deg=az)
    rig = {"studio": {"background": [0.9, 0.9, 0.9],
                      "lights": [{"type": "directional", "direction": [0.3, -0.4, 1.0], "irradiance": 2.5},
                                 {"type": "point", "position": [-2.0, 2.0, 2.0], "intensity": 20, "radius": 0.2,
                                  "samples": 8}]},
           "spot": {"lights": [{"type": "spot", "position": [0, -2.5, 2.5], "target": [0, 0, 0], "intensity": 60,
                                "inner_deg": 15, "outer_deg": 30}]}}
    args = types.SimpleNamespace(out=str(tmp_path), batch_size=2048, shadow_far=3.0)
    P.render_path(ds, args, poses, P.frame_angles(8, (0.0, 360.0)), tensoIR=model, ground_z=True, rig=rig)
    for name in rig:
        for sub in ("with_bg", "without_bg"):
            assert sorted(os.listdir(tmp_path / name / sub)) == [f"{f:04d}.png" for f in range(8)]
    try:
        import imageio  # noqa: F401
        assert (tmp_path / "studio.mp4").exists() and (tmp_path / "spot.mp4").exists()
    except ImportError:
        pass
    with pytest.raises(ValueError):
        P.render_path(ds, types.SimpleNamespace(out=str(tmp_path / "x"), batch_size=2048, light="learned"), poses[:1],
                      [0.0], tensoIR=model, rig=rig)
    assert not (tmp_path / "x").exists()
