"""Relighting under analytic lights on the H100: the tir_lights kernels against their host build and float64, a
directional light against the environment-map pass it is a special case of, shadows on the lego scene against ray-box
intersection, and relight_rig end to end.

The primary render composites with float atomics and the density march's result for a ray can change in its last bits
with the ray's place in the list, which an atomic append fills; where a test compares two runs to the byte, the forward
and the visibility of the first run are replayed in the second (as in test_material_edit_gpu.py).  The GGX terms
(csrc/tir_ggx.h) are shared with the training kernels and contracted into FMAs by the device compiler, so the shaded
images agree with the host build to rounding, not to the bit; everything the sample kernel writes does to the bit."""
import math
import os
import types

import numpy as np
import pytest
import torch

from gpu_helpers import load_fixture, model_from_fixture
from helpers import build_host_lib, use_host
from test_lighting_cpu import MIXED, check_against_float64, random_chunk, reference64, run_chunk
from test_material_edit_gpu import Replay

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def fx():
    import __graft_entry__ as g
    g.build()
    return load_fixture("rotated_g24.pt")


@pytest.mark.parametrize("stride,vis_kind", [(1, 0), (3, 1)])
def test_kernels_match_host_build(fx, tmp_path, monkeypatch, stride, vis_kind):
    from tensoir_b200 import lighting
    n = 6000
    ch = random_chunk(40 + stride, n, stride)
    u = torch.rand(n * lighting.slots_per_ray(MIXED), 2, dtype=torch.float64,
                   generator=torch.Generator().manual_seed(12))
    rescale = [1.2, 0.9, 1.05]
    dch = {k: v.to(DEV) for k, v in ch.items()}
    got = {k: v.cpu() for k, v in run_chunk(MIXED, dch, u.to(DEV), vis_kind, rescale, seed=3).items()}
    again = run_chunk(MIXED, dch, u.to(DEV), vis_kind, rescale, seed=3)
    assert torch.equal(got["L"], again["L"].cpu()) and torch.equal(got["falloff"], again["falloff"].cpu())
    assert torch.equal(got["pos"] >= 0, again["pos"].cpu() >= 0)

    use_host(monkeypatch, build_host_lib(tmp_path, "host_lights.cpp"))
    want = run_chunk(MIXED, ch, u, vis_kind, rescale, seed=3)
    assert torch.equal(got["L"], want["L"]) and torch.equal(got["falloff"], want["falloff"])
    joined = want["pos"] >= 0
    assert torch.equal(got["pos"] >= 0, joined) and got["list_o"].shape == want["list_o"].shape
    rows_g, rows_w = got["pos"][joined].long(), want["pos"][joined].long()
    assert torch.equal(rows_g.sort().values, torch.arange(rows_g.numel()))  # the append order differs, the set does not
    assert torch.equal(got["list_o"][rows_g], want["list_o"][rows_w])
    assert torch.equal(got["list_d"][rows_g], want["list_d"][rows_w])
    # the same visibility per slot for both builds: the kernel's list is the host's, permuted
    vis = torch.empty_like(want["vis"])
    vis[rows_g] = want["vis"][rows_w]
    out = tuple(torch.full((n + 3, 3), -7.0, device=DEV) for _ in range(3))
    monkeypatch.undo()
    lighting.rig_shade(MIXED, dch["rays"], dch["normal"], dch["albedo"], dch["rough"], dch["fresnel"], dch["acc"], 0.5,
                       rescale, tuple(got[k].to(DEV) for k in ("L", "falloff", "pos")) + (vis.to(DEV),),
                       'nerfactor' if vis_kind else 'nerv', out, 2)
    res = dict(got, vis=vis, with_bg=out[0].cpu(), without_bg=out[1].cpu(), linear=out[2].cpu())
    out2 = tuple(torch.full((n + 3, 3), -7.0, device=DEV) for _ in range(3))
    lighting.rig_shade(MIXED, dch["rays"], dch["normal"], dch["albedo"], dch["rough"], dch["fresnel"], dch["acc"], 0.5,
                       rescale, tuple(got[k].to(DEV) for k in ("L", "falloff", "pos")) + (vis.to(DEV),),
                       'nerfactor' if vis_kind else 'nerv', out2, 2)
    assert all(torch.equal(a, b) for a, b in zip(out, out2))                # fixed-order sums: bit-identical reruns
    check_against_float64(MIXED, ch, u, res, vis_kind, rescale, slot_order=False)
    # both builds lie within the fp32 bound of the float64 result, so within twice the bound of each other
    _, bound, _, _ = reference64(MIXED, ch, u, res, vis_kind, rescale)
    lin_g, lin_w = res["linear"][2:2 + n].double(), want["linear"][2:2 + n].double()
    assert ((lin_g - lin_w).abs() <= 2 * bound + 1e-30).all()
    for k in ("without_bg", "with_bg"):
        assert ((res[k][2:2 + n] - want[k][2:2 + n]).abs() <= 2 * 12.92 * bound + 1e-6).all()


def test_directional_light_is_a_one_pixel_environment(fx):
    """An environment map whose only non-zero pixel is bin b with radiance R shades every hit with
    f vis R cos / pdf_return[b]; so does a hard directional light along hdr_dir[b] with irradiance R / pdf_return[b]."""
    from tensoir_b200 import lighting, relighting
    from tensoir_b200.lighting import Light, Setup
    from tensoir_b200.relight import Environment_Light
    m = model_from_fixture(fx, DEV)
    maps = tuple(t.to(DEV) for t in fx["relight_maps"])
    rays = fx["rays"].to(DEV)
    n = rays.shape[0]
    H, W = 16, 32
    probe = Environment_Light({"p": np.ones((H, W, 3), np.float32)}, device=DEV)
    hit = maps[5].reshape(-1) > 0.5
    b = int(((maps[1][hit] @ probe.hdr_dir["p"].reshape(-1, 3).T) > 0.2).sum(0).argmax())
    arr = np.zeros((H * W, 3), np.float32)
    arr[b] = (90.0, 80.0, 70.0)
    env = Environment_Light({"one": arr.reshape(H, W, 3)}, device=DEV)
    pdf = env.hdr_pdf_return["one"].reshape(-1)[b]
    direction = env.hdr_dir["one"].reshape(-1, 3)[b]
    setup = Setup((Light("directional", tuple((env.hdr_rgbs["one"].reshape(-1, 3)[b] / pdf).tolist()),
                         direction=tuple(direction.tolist())),))
    for vis_equation in ("nerv", "nerfactor"):
        S = 4
        u_env = torch.rand(1, n, S, dtype=torch.float64, device=DEV)
        w, wo = relighting.relight_chunk_fused(m, env, ["one"], rays, maps, 1.3, u_env, S, vis_equation=vis_equation)
        u = torch.zeros(n, 2, dtype=torch.float64, device=DEV)
        rw, rwo, rlin = lighting.relight_chunk_rig(m, setup, rays, maps, 1.3, u, vis_equation=vis_equation,
                                                   shadow_far=1.5)
        assert (rwo - wo[0]).abs().max() < 1e-5
        lit = (rlin.sum(-1) > 0)
        assert lit.sum() > 0.2 * hit.sum() and bool(((rwo < 1) & (rwo > 0))[lit].any())
    # the shadow-ray list is the environment pass's visibility list (one sample per hit), to the bit
    r, (depth, normal, _, _, _, acc) = relighting.chunk_inputs(rays, maps)
    L, falloff, pos, list_o, list_d = lighting.rig_sample(setup, r, depth, normal, acc, u, 0.5)
    envs, keep = relighting.env_tables(env, ["one"])
    seen = {}
    monkey = pytest.MonkeyPatch()
    monkey.setattr(relighting.ops, "march_density",
                   lambda model, o, d, **kw: seen.update(o=o.clone(), d=d.clone(), table=kw["table"]) or
                   (torch.ones(o.shape[0], device=DEV),) * 3)
    try:
        _, epos, _ = relighting.relight_visibility(m, envs, 1, r, depth, normal, acc, u_env[:, :, :1].contiguous(), 1,
                                                   0.5, 'nerv')
    finally:
        monkey.undo()
    epos = epos.reshape(-1)
    joined = pos >= 0
    assert torch.equal(epos >= 0, joined) and int(joined.sum()) == seen["o"].shape[0] > 0
    assert torch.equal(seen["o"][epos[joined].long()], list_o[pos[joined].long()])
    assert torch.equal(seen["d"][epos[joined].long()], list_d[pos[joined].long()])
    assert torch.equal(seen["table"], lighting.shadow_table(1.5, DEV))


# ---- shadows on the lego scene ----------------------------------------------------------------------------------------

def look_at_origin(pos):
    """Camera-to-world matrix at ``pos`` looking at the origin, built like synthetic.hemisphere_poses."""
    pos = np.asarray(pos, dtype=np.float64)
    fwd = -pos / np.linalg.norm(pos)
    right = np.cross(fwd, np.array([0.0, 0.0, 1.0]))
    right /= np.linalg.norm(right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, np.cross(fwd, right), fwd, pos
    return torch.tensor(c2w[None], dtype=torch.float32)


def first_hit(o, d):
    """Distance to the nearest lego box along the rays o + t d (slab test, float64), inf without one."""
    from tensoir_b200.synthetic import _lego_boxes
    o, d = o.double(), d.double().expand_as(o)
    inv = 1.0 / torch.where(d == 0, torch.full_like(d, 1e-30), d)
    best = torch.full((o.shape[0],), float("inf"), dtype=torch.float64)
    for lo, hi, _ in _lego_boxes():
        t0 = (torch.tensor(lo, dtype=torch.float64) - o) * inv
        t1 = (torch.tensor(hi, dtype=torch.float64) - o) * inv
        t_in, t_out = torch.minimum(t0, t1).max(dim=1).values, torch.maximum(t0, t1).min(dim=1).values
        best = torch.where((t_in <= t_out) & (t_in > 0) & (t_in < best), t_in, best)
    return best


def occluder_range(p, d, margin):
    """(nearest, furthest) first-hit distance over the plate point and its four neighbours at +-margin in x and y."""
    dist = []
    for dx, dy in ((0, 0), (margin, 0), (-margin, 0), (0, margin), (0, -margin)):
        dist.append(first_hit(p + torch.tensor([dx, dy, 0.02], dtype=p.dtype), d))
    dist = torch.stack(dist)
    return dist.min(0).values, dist.max(0).values


@pytest.fixture(scope="module")
def lego_view():
    """One 160x160 view of the lego scene from the front, above the open side of the arch: the model, the rays, the
    primary maps (with the boxes' face normals), the surface points and the mask of pixels on the top of the base
    plate."""
    import __graft_entry__ as g
    g.build()
    from tensoir_b200.synthetic import SyntheticViews, make_lego_model
    m = make_lego_model(96, DEV)
    ds = SyntheticViews(look_at_origin((0.0, -2.2, 3.2)), 160, 160, light_names=["a"])
    rays = ds[0]["rays"].to(DEV)
    li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        _, depth, normal, albedo, rough, fresnel, acc, *_ = m(rays, li, is_train=False, white_bg=True, ndc_ray=False,
                                                              N_samples=-1)
    # the scene's appearance is untrained, so its predicted normals mean nothing: shade with the boxes' face normals
    face = ds[0]["normals"]
    maps = tuple(t.detach() for t in (depth, face.to(DEV), albedo, rough, fresnel, acc))
    p = (rays[:, :3] + depth.reshape(-1, 1) * rays[:, 3:]).cpu()
    plate = (acc.reshape(-1).cpu() > 0.9) & ((p[:, 2] + 0.65).abs() < 0.03) & (face[:, 2] == 1) & \
        (p[:, :2].abs().max(dim=1).values < 0.97)
    assert plate.sum() > 2000
    return m, rays, maps, p, plate


def _linear(m, rays, maps, light, **kw):
    from tensoir_b200 import lighting
    setup = lighting.Setup((light,))
    u = torch.rand(rays.shape[0] * light.samples, 2, dtype=torch.float64, device=DEV,
                   generator=torch.Generator(DEV).manual_seed(1))
    return lighting.relight_chunk_rig(m, setup, rays, maps, 1.0, u, **kw)[2].cpu()


def dark(x):
    """Nearly every pixel of a shadow is black: a shadow ray may still clip a caster's soft, one-voxel edge."""
    return x.numel() > 0 and (x < 1e-3).float().mean() > 0.95 and x.median() < 1e-4


def lit(x):
    return x.numel() > 0 and (x > 1e-2).float().mean() > 0.95


ABOVE = (0.0, 0.0, 1.0)
OPEN_SIDE = (0.0, -0.5 / math.hypot(0.5, 0.85), 0.85 / math.hypot(0.5, 0.85))


def test_shadows_are_where_the_geometry_says(lego_view):
    from tensoir_b200 import lighting
    from tensoir_b200.lighting import Light
    m, rays, maps, p, plate = lego_view
    white = (3.0, 3.0, 3.0)
    lin, near, far = {}, {}, {}
    for name, d in (("above", ABOVE), ("side", OPEN_SIDE)):
        lin[name] = _linear(m, rays, maps, Light("directional", white, direction=d)).sum(-1)
        near[name], far[name] = occluder_range(p, torch.tensor(d), 0.06)
    shadowed = {k: plate & torch.isfinite(far[k]) for k in lin}           # the point and its neighbours all occluded
    open_ = {k: plate & torch.isinf(near[k]) for k in lin}                 # none occluded
    under_arch = shadowed["above"] & (p[:, :2].abs() < torch.tensor([0.5, 0.25])).all(1)
    assert under_arch.sum() > 30 and (under_arch & open_["side"]).sum() > 10
    assert lin["above"][under_arch].max() < 1e-4                           # the beam's shadow
    assert lit(lin["side"][under_arch & open_["side"]])                    # lit through the arch's open side
    clear = open_["above"] & open_["side"]
    assert clear.sum() > 100 and lit(lin["above"][clear]) and lit(lin["side"][clear])
    for k in lin:
        assert dark(lin[k][shadowed[k]]) and shadowed[k].sum() > 30

    # a 5 degree disc: partial visibility along the shadow edge; 64 samples of a light without extent are one sample
    soft = Light("directional", white, direction=ABOVE, extent=math.tan(math.radians(5.0)), samples=64)
    r, (depth, normal, _, _, _, acc) = __import__("tensoir_b200").relighting.chunk_inputs(rays, maps)
    u = torch.rand(rays.shape[0] * 64, 2, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(2))
    L, falloff, pos, vis = lighting.rig_visibility(m, lighting.Setup((soft,)), r, depth, normal, acc, u, 0.5, 'nerv',
                                                   lighting.shadow_table(lighting.default_shadow_far(m), DEV))
    v = torch.where(pos >= 0, vis[pos.clamp(min=0).long()], torch.zeros((), device=DEV)).reshape(-1, 64).mean(1).cpu()
    penumbra = plate & (v > 0.1) & (v < 0.9)
    assert penumbra.sum() > 20
    assert (v[under_arch & (p[:, :2].abs() < torch.tensor([0.3, 0.1])).all(1)] < 0.05).all()
    assert (v[clear & (near["above"] == float("inf"))] > 0.5).float().mean() > 0.9
    many = _linear(m, rays, maps, Light("directional", white, direction=ABOVE, samples=64))
    assert (many.sum(-1) - lin["above"]).abs().max() < 3e-6 and many.shape == (rays.shape[0], 3)


def test_shadow_far(lego_view):
    """Low light from behind the back wall: the wall's shadow reaches the front end of the plate from more than 1.5
    away.  Marched to 1.5 as relight() marches, that shadow is missing; marched across the box it is there."""
    from tensoir_b200.lighting import Light
    m, rays, maps, p, plate = lego_view
    d = (0.0, 0.906, 0.423)
    d = tuple(c / math.sqrt(sum(x * x for x in d)) for c in d)
    light = Light("directional", (3.0, 3.0, 3.0), direction=d)
    near, far = occluder_range(p, torch.tensor(d), 0.04)
    distant = plate & torch.isfinite(far) & (near > 1.65)
    assert distant.sum() > 10
    short = _linear(m, rays, maps, light, shadow_far=1.5).sum(-1)
    full = _linear(m, rays, maps, light).sum(-1)
    assert lit(short[distant]) and dark(full[distant])
    close = plate & (far < 1.3)
    assert close.sum() > 30 and dark(short[close]) and dark(full[close])


# ---- relight_rig end to end -------------------------------------------------------------------------------------------

class ReplayCalls:
    """A module function recorded on the first pass and its results replayed, in call order, on later passes."""

    def __init__(self, monkeypatch, module, name):
        self.fn, self.calls, self.i = getattr(module, name), [], None
        monkeypatch.setattr(module, name, self)

    def __call__(self, *a, **k):
        if self.i is None:
            self.calls.append(self.fn(*a, **k))
            return self.calls[-1]
        self.i += 1
        return self.calls[self.i - 1]


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs
                  if not f.endswith(".mp4"))


def test_relight_rig_end_to_end(fx, tmp_path, monkeypatch):
    """Two setups on two 32x24 views, batch_size 300 (three chunks per view): the file list, identical bytes from a
    second run with the same seed, and a light inside the aabb refused."""
    from tensoir_b200 import lighting
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    m = model_from_fixture(fx, DEV)
    H, W, B = 24, 32, 300
    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=["a"])
    rig = {"noon": {"lights": [{"type": "directional", "direction": [0.2, 0.1, 1.0], "irradiance": [3.0, 3.0, 2.8],
                                "angular_radius_deg": 2.0, "samples": 16}]},
           "lamp": {"background": [0.0, 0.1, 0.2],
                    "lights": [{"type": "point", "position": [2.5, 0.0, 2.0], "intensity": [40, 36, 30],
                                "radius": 0.15, "samples": 8},
                               {"type": "spot", "position": [-3, -3, 3], "target": [0, 0, 0], "intensity": 60,
                                "inner_deg": 10, "outer_deg": 18}]}}
    rep = Replay(m)
    rv = ReplayCalls(monkeypatch, lighting, "rig_visibility")
    outs = []
    for run in ("a", "b"):
        out = tmp_path / run
        lighting.relight_rig(ds, types.SimpleNamespace(geo_buffer_path=str(out), batch_size=B, seed=7, save_linear=1),
                             rig, tensoIR=m)
        rep.i = rv.i = 0
        outs.append(out)
    assert len(rv.calls) == len(ds) * -(-H * W // B) * len(rig)
    want = [f"test_{i:03d}/relighting_{sub}/{s}.{ext}" for i in range(len(ds)) for s in rig
            for sub, ext in (("with_bg", "png"), ("without_bg", "png"), ("linear", "hdr"))]
    assert _files(outs[0]) == sorted(want) == _files(outs[1])
    for f in want:
        assert (outs[0] / f).read_bytes() == (outs[1] / f).read_bytes(), f
    import cv2
    lamp = cv2.imread(str(outs[0] / "test_000/relighting_with_bg/lamp.png"))[..., ::-1]
    bare = cv2.imread(str(outs[0] / "test_000/relighting_without_bg/lamp.png"))[..., ::-1]
    bg = (bare == 255).all(-1)
    assert bg[0, 0] and not bg.all()                                    # the corner ray misses the object
    assert (lamp[0, 0] == (np.array([0.0, 0.1, 0.2], np.float32) * 255).astype(np.uint8)).all()
    assert len(np.unique(bare[~bg])) > 10
    no_linear = tmp_path / "c"
    rep.i = rv.i = 0
    lighting.relight_rig(ds, types.SimpleNamespace(geo_buffer_path=str(no_linear), batch_size=B, seed=7), rig, tensoIR=m)
    assert _files(no_linear) == sorted(f for f in want if f.endswith(".png"))
    inside = {"bad": {"lights": [{"type": "point", "position": [0.5, 0.0, 0.0], "intensity": 1.0}]}}
    with pytest.raises(ValueError, match=r"setup 'bad' light 0"):
        lighting.relight_rig(ds, types.SimpleNamespace(geo_buffer_path=str(tmp_path / "d"), batch_size=B), inside,
                             tensoIR=m)


def test_olat_images_add_up(fx, tmp_path, monkeypatch):
    """A one-light-at-a-time sweep of four lights: its four un-toned images sum to the image of one setup holding the
    four lights."""
    import tensoir_b200.relight as RL
    from tensoir_b200 import lighting
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    m = model_from_fixture(fx, DEV)
    ds = SyntheticViews(hemisphere_poses(1), 24, 32, light_names=["a"])
    written = {}
    monkeypatch.setattr(RL, "write_hdr", lambda path, rgb: written.__setitem__(os.path.basename(path), rgb.copy()))
    rep = Replay(m)
    olat = lighting.olat_rig(4)
    args = lambda d: types.SimpleNamespace(geo_buffer_path=str(tmp_path / d), batch_size=500, save_linear=True)  # noqa: E731
    lighting.relight_rig(ds, args("olat"), olat, tensoIR=m)
    rep.i = 0
    lighting.relight_rig(ds, args("all"), {"all": lighting.Setup(tuple(s.lights[0] for s in olat.values()))}, tensoIR=m)
    assert sorted(written) == ["all.hdr"] + [f"olat_{k:03d}.hdr" for k in range(4)]
    total = sum(written[f"olat_{k:03d}.hdr"].astype(np.float64) for k in range(4))
    assert np.abs(total - written["all.hdr"]).max() < 1e-5 and written["all.hdr"].max() > 1e-3
    assert sum(written[f"olat_{k:03d}.hdr"].max() > 0 for k in range(4)) >= 2
