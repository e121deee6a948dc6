"""Relighting under analytic lights on the CPU.

tir_lights_sample and tir_lights_shade are built for the host (tests/host_lights.cpp: the same C ABI, argument checks
and per-slot math of csrc/tir_lights_body.h, loops instead of kernels) and driven through the real ctypes wrapper
tensoir_b200.lighting.  They are compared with a float64 restatement of the definitions in include/tensoir_b200.h,
written here with torch and relight_utils.GGX_specular."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from tensoir_b200 import _lib, lighting
from tensoir_b200.lighting import Light, Setup
from tensoir_b200.relight_utils import GGX_specular, linear2srgb_torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
EPS = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_lights"), "host_lights.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


# ---- 1. the rig file ----------------------------------------------------------------------------------------------

RIG = {"noon": {"lights": [{"type": "directional", "direction": [0.2, 0.1, 1.0], "irradiance": [3.0, 3.0, 2.8],
                            "angular_radius_deg": 0.27, "samples": 16}]},
       "lamp": {"background": [0.0, 0.0, 0.0],
                "lights": [{"type": "point", "position": [2.5, 0.0, 2.0], "intensity": [40, 36, 30], "radius": 0.15,
                            "samples": 64},
                           {"type": "spot", "position": [-3, -3, 3], "target": [0, 0, 0], "intensity": 60,
                            "inner_deg": 10, "outer_deg": 18}]}}


def test_load_rig_fields(tmp_path):
    p = tmp_path / "rig.json"
    p.write_text(json.dumps(RIG))
    rig = lighting.load_rig(str(p))
    assert rig == lighting.load_rig(json.dumps(RIG)) == lighting.load_rig(RIG) == lighting.load_rig(rig)
    assert list(rig) == ["noon", "lamp"]
    sun, = rig["noon"].lights
    n = math.sqrt(0.2 ** 2 + 0.1 ** 2 + 1)
    assert sun.kind == "directional" and sun.direction == pytest.approx((0.2 / n, 0.1 / n, 1 / n))
    assert sun.power == (3.0, 3.0, 2.8) and sun.samples == 16
    assert sun.extent == pytest.approx(math.tan(math.radians(0.27)))
    assert rig["noon"].background == (1.0, 1.0, 1.0) and rig["lamp"].background == (0.0, 0.0, 0.0)
    lamp, spot = rig["lamp"].lights
    assert (lamp.kind, lamp.position, lamp.power, lamp.extent, lamp.samples) == \
        ("point", (2.5, 0.0, 2.0), (40.0, 36.0, 30.0), 0.15, 64)
    s3 = 1 / math.sqrt(3)
    assert spot.kind == "spot" and spot.power == (60.0,) * 3 and spot.direction == pytest.approx((s3, s3, -s3))
    assert spot.cos_inner == pytest.approx(math.cos(math.radians(10)))
    assert spot.cos_outer == pytest.approx(math.cos(math.radians(18)))
    assert spot.extent == 0.0 and spot.samples == 1
    # samples is forced to 1, without an error, when the light has no extent
    hard = lighting.load_rig({"a": {"lights": [{"type": "directional", "direction": [0, 0, 1], "irradiance": 1,
                                                "samples": 64},
                                               {"type": "point", "position": [3, 0, 0], "intensity": 1,
                                                "samples": 9}]}})
    assert [l.samples for l in hard["a"].lights] == [1, 1]
    t = lighting.light_table(rig["lamp"])
    assert (t[0].type, t[0].n_samples, t[1].type, t[1].n_samples) == (_lib.LIGHT_POINT, 64, _lib.LIGHT_SPOT, 1)
    assert list(t[0].pos) == [2.5, 0.0, 2.0] and t[1].cos_outer == pytest.approx(math.cos(math.radians(18)))
    olat = lighting.olat_rig(4)
    assert list(olat) == ["olat_000", "olat_001", "olat_002", "olat_003"]
    assert olat["olat_000"].lights[0].direction == pytest.approx((0, 0, 1)) and olat["olat_002"].lights[0].samples == 1


_SUN = {"type": "directional", "direction": [0, 0, 1], "irradiance": 1.0}
_LAMP = {"type": "point", "position": [3, 0, 0], "intensity": 1.0}
_SPOT = {"type": "spot", "position": [3, 0, 0], "target": [0, 0, 0], "intensity": 1.0, "inner_deg": 5, "outer_deg": 9}


@pytest.mark.parametrize("light", [
    {**_SUN, "colour": 1},                                           # unknown key
    {**_SUN, "position": [3, 0, 0]},                                 # a key of another type
    {**_SUN, "type": "area"},
    {"direction": [0, 0, 1], "irradiance": 1.0},                     # no type
    {**_SUN, "direction": [0, 0, 0]},                                # zero length
    {**_SUN, "direction": [0, 1]},                                   # wrong shapes
    {**_SUN, "irradiance": [1, 1]},
    {**_SUN, "irradiance": -1.0},                                    # negative, non-finite
    {**_SUN, "irradiance": [1, float("nan"), 1]},
    {**_SUN, "angular_radius_deg": 31},
    {**_SUN, "angular_radius_deg": -1},
    {**_SUN, "samples": 0},
    {**_SUN, "samples": 1025},
    {**_SUN, "samples": 2.5},
    {"type": "directional", "direction": [0, 0, 1]},                 # missing irradiance
    {**_LAMP, "radius": -0.1},
    {**_LAMP, "position": [float("inf"), 0, 0]},
    {**_LAMP, "intensity": "bright"},
    {**_LAMP, "target": [0, 0, 0]},
    {"type": "point", "intensity": 1.0},
    {**_SPOT, "inner_deg": 10},                                      # inner above outer
    {**_SPOT, "outer_deg": 90},
    {**_SPOT, "inner_deg": -1},
    {**_SPOT, "target": [3, 0, 0]},                                  # no axis
    {k: v for k, v in _SPOT.items() if k != "target"},
    "sun",
])
def test_load_rig_names_setup_and_light(light):
    with pytest.raises(ValueError, match=r"setup 'key' light 1"):
        lighting.load_rig({"key": {"lights": [_SUN, light]}})


@pytest.mark.parametrize("bad", [
    {"v": {"lights": []}},
    {"v": {"lights": [_SUN] * 17}},
    {"v": {}},
    {"v": {"lights": [_SUN], "ambient": 0.1}},
    {"v": [_SUN]},
    {"v": {"lights": [_SUN], "background": [0, 0]}},
    {"v": {"lights": [_SUN], "background": [0, 0, 1.5]}},
    {"../x": {"lights": [_SUN]}},
    {"a/b": {"lights": [_SUN]}},
    {"": {"lights": [_SUN]}},
    {"..": {"lights": [_SUN]}},
    {},
    [_SUN],
])
def test_load_rig_rejects(bad):
    with pytest.raises(ValueError):
        lighting.load_rig(bad)
    if isinstance(bad, dict) and "v" in bad:
        with pytest.raises(ValueError, match="'v'"):
            lighting.load_rig(bad)


def test_lights_must_clear_the_aabb():
    aabb = torch.tensor([[-1.5, -1.5, -1.5], [1.5, 1.5, 1.5]])
    rig = lambda **kw: lighting.load_rig({"s": {"lights": [_SUN, {**_LAMP, **kw}]}})  # noqa: E731
    lighting.check_outside(rig(position=[1.6, 0, 0]), aabb)
    lighting.check_outside(rig(position=[2.0, 2.0, 0], radius=0.7), aabb)           # corner gap 0.707
    lighting.check_outside(lighting.load_rig({"s": {"lights": [_SUN]}}), aabb)      # directional: no position
    for kw in (dict(position=[0, 0, 0]), dict(position=[1.5, 0, 0]), dict(position=[1.75, 0, 0], radius=0.25),
               dict(position=[2.0, 2.0, 0], radius=0.71), dict(position=[1.4, 9, 9], radius=20)):
        with pytest.raises(ValueError, match=r"setup 's' light 1"):
            lighting.check_outside(rig(**kw), aabb)


def test_shadow_table_keeps_the_reference_spacing():
    from tensoir_b200 import ops
    t = lighting.shadow_table(1.5, "cpu")
    assert torch.equal(t, ops.equal_z_table(96, 0.05, 1.5, "cpu"))
    far = math.sqrt(27.0)
    t = lighting.shadow_table(far, "cpu")
    n = t.shape[0]
    assert n == math.ceil((far - 0.05) / lighting.SHADOW_STEP) + 1 and t[-1] >= far > t[-2]
    assert torch.allclose(t[1:] - t[:-1], torch.full((n - 1,), lighting.SHADOW_STEP), atol=1e-6)
    with pytest.raises(ValueError):
        lighting.shadow_table(0.05, "cpu")


# ---- 2. the host twin against float64 -----------------------------------------------------------------------------

def random_chunk(seed, n, stride):
    """Seeded maps of n primary rays: cameras at radius 4 looking at points of the [-1, 1] box, normals roughly towards
    the camera (raw length 0.8 .. 1.2), albedo, roughness and fresnel in the model's ranges, a fifth of acc below the
    threshold."""
    g = np.random.default_rng(seed)
    pts = g.uniform(-1, 1, (n, 3))
    cam = g.normal(size=(n, 3))
    cam = 4 * cam / np.linalg.norm(cam, axis=1, keepdims=True)
    d = pts - cam
    depth = np.linalg.norm(d, axis=1)
    d /= depth[:, None]
    normal = -d + 0.5 * g.normal(size=(n, 3))
    normal *= (g.uniform(0.8, 1.2, n) / np.linalg.norm(normal, axis=1))[:, None]
    acc = np.where(g.uniform(size=n) < 0.2, g.uniform(0, 0.5, n), g.uniform(0.5, 1, n))
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))  # noqa: E731
    return dict(rays=f(np.concatenate([cam, d], 1)), depth=f(depth), normal=f(normal), albedo=f(g.uniform(0, 1, (n, 3))),
                rough=f(g.uniform(0.09, 0.99, (n, stride))), fresnel=f(g.uniform(0.02, 0.1, (n, 3))), acc=f(acc))


def run_chunk(setup, ch, u, vis_kind, rescale, seed=0, vis_one=False):
    """rig_sample + a seeded random visibility list + rig_shade through whatever library _lib.load() gives."""
    dev = ch["rays"].device
    L, falloff, pos, list_o, list_d = lighting.rig_sample(setup, ch["rays"], ch["depth"], ch["normal"], ch["acc"], u, 0.5)
    m = list_o.shape[0]
    vis = torch.rand(max(m, 1), generator=torch.Generator().manual_seed(seed))
    if vis_one:
        vis = torch.full_like(vis, 0.0 if vis_kind else 1.0)
    vis = vis.to(dev)
    n = ch["rays"].shape[0]
    out = tuple(torch.full((n + 3, 3), -7.0, device=dev) for _ in range(3))
    lighting.rig_shade(setup, ch["rays"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"], 0.5,
                       rescale, (L, falloff, pos, vis), 'nerfactor' if vis_kind else 'nerv', out, 2)
    return dict(L=L, falloff=falloff, pos=pos, list_o=list_o, list_d=list_d, vis=vis, with_bg=out[0],
                without_bg=out[1], linear=out[2])


def _frame64(w):
    """The disc axes of csrc/tir_lights_body.h (Duff et al.'s orthonormal basis around w), in float64."""
    s = torch.where(w[..., 2] >= 0, 1.0, -1.0).double()
    a = -1.0 / (s + w[..., 2])
    b = w[..., 0] * w[..., 1] * a
    t1 = torch.stack([1.0 + s * w[..., 0] ** 2 * a, s * b, -s * w[..., 0]], -1)
    t2 = torch.stack([b, s + w[..., 1] ** 2 * a, -w[..., 1]], -1)
    return t1, t2


def _disc64(u):
    a, b = 2 * u[..., 0] - 1, 2 * u[..., 1] - 1
    wide = a.abs() > b.abs()
    r = torch.where(wide, a, b)
    phi = torch.where(wide, (math.pi / 4) * b / torch.where(a == 0, 1.0, a),
                      math.pi / 2 - (math.pi / 4) * a / torch.where(b == 0, 1.0, b))
    return r * torch.cos(phi), r * torch.sin(phi)


def reference64(setup, ch, u, res, vis_kind, rescale, thr=0.5):
    """The definitions of include/tensoir_b200.h in float64, per light [n, K]: direction, falloff, the cosine test, and
    the linear sum with the visibility the host build's pos selects.  Also the bound on |linear32 - linear64|.

    Bound.  A slot's term is T = (a/pi + S) v f c with S = frac/nom the GGX term, v the visibility, f the falloff and
    c = L.n.  In fp32 every factor is a chain of at most ~30 rounded operations on well-conditioned inputs, each adding
    a relative error <= eps, except two: (i) nom0 = NoH^2 (alpha^2 - 1) + 1 cancels near a highlight, where an absolute
    error of ~4 eps in NoH^2 becomes the relative error 4 eps / nom0, and nom holds nom0 squared; (ii) c carries the
    absolute error of the fp32 direction, <= 4 eps |n|.  So |dT| <= eps (32 |T| + 16 |S v f c| / nom0 + 8 B v f |n|)
    with B = a/pi + S, and the light sums and the mean add the same relative eps per addition, covered by the 32.
    A spot adds (iii): its cone is a smoothstep (slope <= 1.5) of (cos - cos_outer) / (cos_inner - cos_outer), where cos
    carries an absolute error <= 8 eps, so |df| <= 12 eps / (cos_inner - cos_outer) / d^2 and |dT| grows by B v |c| |df|."""
    t = lambda x: x.double()  # noqa: E731
    rays, depth, normal, acc = t(ch["rays"]), t(ch["depth"]), t(ch["normal"]), t(ch["acc"])
    albedo = t(ch["albedo"]) * torch.as_tensor(rescale, dtype=torch.float64).reshape(-1).expand(3)
    rough, fresnel = t(ch["rough"]), t(ch["fresnel"])
    n = rays.shape[0]
    p = rays[:, :3] + depth[:, None] * rays[:, 3:]
    hit = acc > thr
    linear, bound = torch.zeros(n, 3, dtype=torch.float64), torch.zeros(n, 3, dtype=torch.float64)
    per_light, k0 = [], 0
    for l in setup.lights:
        K = l.samples
        sl = slice(n * k0, n * (k0 + K))
        k0 += K
        uu = t(u[sl]).reshape(n, K, 2)
        centre = K == 1 or not l.extent > 0
        x, y = (torch.zeros(n, K, dtype=torch.float64),) * 2 if centre else _disc64(uu)
        power = torch.tensor(l.power, dtype=torch.float64)
        axis = torch.tensor(l.direction, dtype=torch.float64)
        if l.kind == "directional":
            t1, t2 = _frame64(axis)
            q = axis + l.extent * (x[..., None] * t1 + y[..., None] * t2)
            Ld = q / q.norm(dim=-1, keepdim=True)
            fall = torch.ones(n, K, dtype=torch.float64)
            dfall = torch.zeros(n, K, dtype=torch.float64)
        else:
            c = torch.tensor(l.position, dtype=torch.float64)
            w = (c - p) / (c - p).norm(dim=-1, keepdim=True)
            t1, t2 = _frame64(w)
            q = c + l.extent * (x[..., None] * t1[:, None] + y[..., None] * t2[:, None])
            to = q - p[:, None]
            d = to.norm(dim=-1)
            Ld = to / d[..., None]
            cone = torch.ones(n, K, dtype=torch.float64)
            if l.kind == "spot":
                cs = -(Ld * axis).sum(-1)
                s = ((cs - l.cos_outer) / max(l.cos_inner - l.cos_outer, 1e-300)).clamp(0, 1)
                cone = torch.where(cs >= l.cos_inner, 1.0, torch.where(cs <= l.cos_outer, 0.0, s * s * (3 - 2 * s)))
            fall = cone / d ** 2
            dfall = torch.zeros_like(fall)
            if l.kind == "spot" and l.cos_inner > l.cos_outer:
                dfall = 12 * EPS / (l.cos_inner - l.cos_outer) / d ** 2
        cos = (Ld * normal[:, None]).sum(-1)
        joins = hit[:, None] & (cos > 1e-6) & (fall > 0)
        pos = res["pos"][sl].reshape(n, K).long()
        v = res["vis"].double()[pos.clamp(min=0)]
        v = torch.where(pos >= 0, 1 - v if vis_kind else v, 0.0)
        spec = GGX_specular(normal, -rays[:, 3:], Ld, rough, fresnel)                  # [n, K, 3]
        B = albedo[:, None] / math.pi + spec
        T = B * (v * fall * cos)[..., None]
        V = torch.nn.functional.normalize(-rays[:, 3:], dim=-1)
        N = torch.nn.functional.normalize(normal, dim=-1)
        N = N * (V * N).sum(-1, keepdim=True).sign()
        H = torch.nn.functional.normalize(Ld + V[:, None], dim=-1)
        NoH = (N[:, None] * H).sum(-1, keepdim=True).clamp(1e-6, 1)
        nom0 = NoH * NoH * ((rough ** 4)[:, None] - 1) + 1
        dT = EPS * (32 * T.abs() + 16 * (spec * (v * fall * cos)[..., None]).abs() / nom0
                    + 8 * B * (v * fall)[..., None] * normal.norm(dim=-1)[:, None, None]
                    + B * (v * cos.abs() * dfall)[..., None] / EPS)
        linear += torch.where(hit[:, None], power * T.mean(1), 0.0)
        bound += torch.where(hit[:, None], power * dT.mean(1), 0.0)
        per_light.append(dict(L=Ld, falloff=fall, dfall=dfall, joins=joins, cos=cos))
    return linear, bound, per_light, hit


MIXED = Setup((Light("directional", (3.0, 3.0, 2.8), direction=lighting._unit((0.2, 0.1, 1.0), ""),
                     extent=math.tan(math.radians(5.0)), samples=8),
               Light("point", (40.0, 36.0, 30.0), position=(2.5, 0.0, 2.0), extent=0.15, samples=40),
               Light("spot", (60.0, 60.0, 60.0), position=(-3.0, -3.0, 3.0), direction=(3 ** -0.5, 3 ** -0.5, -3 ** -0.5),
                     cos_inner=math.cos(math.radians(10)), cos_outer=math.cos(math.radians(18))),
               Light("spot", (20.0, 10.0, 5.0), position=(0.0, 3.0, 2.0),
                     direction=lighting._unit((0.0, -3.0, -2.0), ""), extent=0.2, samples=5,
                     cos_inner=math.cos(math.radians(12)), cos_outer=math.cos(math.radians(25))),
               Light("directional", (0.5, 0.6, 0.7), direction=(0.0, 0.6, 0.8)),
               Light("point", (9.0, 9.0, 9.0), position=(0.0, 0.0, -2.5))), background=(0.1, 0.2, 0.3))


def check_against_float64(setup, ch, u, res, vis_kind, rescale, slot_order=True):
    n = ch["rays"].shape[0]
    linear, bound, per_light, hit = reference64(setup, ch, u, res, vis_kind, rescale)
    k0, expect_pos, sure = 0, [], []
    for l, ref in zip(setup.lights, per_light):
        K = l.samples
        sl = slice(n * k0, n * (k0 + K))
        k0 += K
        L, fall = res["L"][sl].reshape(n, K, 3).double(), res["falloff"][sl].reshape(n, K).double()
        assert (L - ref["L"])[hit].abs().max() < 8 * EPS
        assert ((fall - ref["falloff"])[hit].abs() <= 16 * EPS * ref["falloff"][hit] + ref["dfall"][hit] + 1e-9).all()
        assert not L[~hit].any() and not fall[~hit].any()
        expect_pos.append(ref["joins"].reshape(-1))
        # slots whose membership no rounding can change: the cosine away from 1e-6, the cone away from its edge
        sure.append((((ref["cos"] - 1e-6).abs() > 1e-5) & ((ref["falloff"] > 1e-6) | (ref["falloff"] == 0)))
                    .reshape(-1))
    joins, sure = torch.cat(expect_pos), torch.cat(sure)
    assert sure.float().mean() > 0.99
    got = res["pos"] >= 0
    assert torch.equal(got[sure], joins[sure])
    # one list row per joining slot (in slot order for the host build), holding the fp32 surface point and the slot's
    # own direction
    rows = res["pos"][got].long()
    assert torch.equal(rows if slot_order else rows.sort().values, torch.arange(int(got.sum())))
    assert res["list_o"].shape[0] == int(got.sum())
    ray_of = torch.cat([torch.arange(n).repeat_interleave(l.samples) for l in setup.lights])
    p32 = ch["rays"][:, :3] + ch["depth"][:, None] * ch["rays"][:, 3:]
    assert torch.equal(res["list_o"][rows], p32[ray_of[got]]) and torch.equal(res["list_d"][rows], res["L"][got])
    lin = res["linear"][2:2 + n].double()
    assert ((lin - linear).abs() <= bound + 1e-30).all(), float(((lin - linear).abs() / (bound + 1e-30)).max())
    assert float(((lin - linear).abs() / (bound + 1e-30)).max()) > 1e-3              # the bound is not vacuous
    assert (linear[hit].sum(-1) > 0).float().mean() > 0.5 and not lin[~hit].any()
    wo = res["without_bg"][2:2 + n].double()
    want = torch.where(hit[:, None], linear2srgb_torch(linear), 1.0)
    slope = 12.92                                                                     # steepest part of the tone curve
    assert ((wo - want).abs() <= slope * bound + 8 * EPS).all()
    acc_t = torch.where(ch["acc"] > 0.9, ch["acc"], 0.0).double()[:, None]
    wb = acc_t * wo + (1 - acc_t) * torch.tensor(setup.background, dtype=torch.float64)
    assert (res["with_bg"][2:2 + n].double() - wb).abs().max() < 4 * EPS
    for k in ("with_bg", "without_bg", "linear"):                                      # rows outside [row0, row0 + n)
        assert (res[k][:2] == -7).all() and (res[k][2 + n:] == -7).all()


@pytest.mark.parametrize("stride,vis_kind", [(1, 0), (3, 1)])
def test_host_build_matches_float64(host_lib, stride, vis_kind):
    n = 1500
    ch = random_chunk(7 + stride, n, stride)
    u = torch.rand(n * lighting.slots_per_ray(MIXED), 2, dtype=torch.float64,
                   generator=torch.Generator().manual_seed(11))
    rescale = [1.2, 0.9, 1.05]
    res = run_chunk(MIXED, ch, u, vis_kind, rescale, seed=stride)
    check_against_float64(MIXED, ch, u, res, vis_kind, rescale)
    again = run_chunk(MIXED, ch, u, vis_kind, rescale, seed=stride)
    assert all(torch.equal(res[k], again[k]) for k in res)
    # each light alone, K = 1 and K > 1, sums to the setup's image
    total = torch.zeros(n, 3, dtype=torch.float64)
    for l in MIXED.lights:
        one = Setup((l,))
        k0 = sum(m.samples for m in MIXED.lights[:MIXED.lights.index(l)])
        r1 = run_chunk(one, ch, u[n * k0:n * (k0 + l.samples)].contiguous(), vis_kind, rescale, vis_one=True)
        total += r1["linear"][2:2 + n].double()
    full = run_chunk(MIXED, ch, u, vis_kind, rescale, vis_one=True)["linear"][2:2 + n].double()
    assert torch.allclose(full, total, rtol=1e-5, atol=1e-7)


# ---- 3. inverse square and the cone -------------------------------------------------------------------------------

def test_inverse_square(host_lib):
    """Every surface point at the origin: a point light moved from distance d to 2d along its direction quarters the
    image where nothing shadows it."""
    n = 400
    g = np.random.default_rng(5)
    ch = random_chunk(21, n, 1)
    d = ch["rays"][:, 3:]
    ch["rays"] = torch.cat([-4 * d, d], 1).contiguous()
    ch["depth"] = torch.full((n,), 4.0)
    to = torch.tensor(g.normal(size=3), dtype=torch.float32)
    to = to / to.norm()
    u = torch.zeros(n, 2, dtype=torch.float64)
    lin = []
    for dist in (3.0, 6.0):
        s = Setup((Light("point", (10.0, 20.0, 30.0), position=tuple((to * dist).tolist())),))
        lin.append(run_chunk(s, ch, u, 0, 1.0, vis_one=True)["linear"][2:2 + n])
    lit = lin[0].sum(-1) > 0
    assert lit.float().mean() > 0.2
    assert torch.allclose(lin[1], lin[0] / 4, rtol=2e-5, atol=0)


def test_spot_cone(host_lib):
    n = 3000
    ch = random_chunk(31, n, 3)
    u = torch.zeros(n, 2, dtype=torch.float64)
    pos, inner, outer = (0.0, 0.0, 4.0), 10.0, 18.0
    point = Setup((Light("point", (50.0, 50.0, 50.0), position=pos),))
    spot = Setup((Light("spot", (50.0, 50.0, 50.0), position=pos, direction=(0.0, 0.0, -1.0),
                        cos_inner=math.cos(math.radians(inner)), cos_outer=math.cos(math.radians(outer))),))
    a = run_chunk(point, ch, u, 0, 1.0, vis_one=True)
    b = run_chunk(spot, ch, u, 0, 1.0, vis_one=True)
    p = (ch["rays"][:, :3] + ch["depth"][:, None] * ch["rays"][:, 3:]).double()
    ang = torch.rad2deg(torch.atan2(p[:, :2].norm(dim=-1), 4.0 - p[:, 2]))
    la, lb = a["linear"][2:2 + n], b["linear"][2:2 + n]
    lit = la.sum(-1) > 0
    inside, outside, between = ang < inner - 0.01, ang > outer + 0.01, (ang > inner + 0.01) & (ang < outer - 0.01)
    assert (inside & lit).sum() > 20 and (outside & lit).sum() > 20 and (between & lit).sum() > 20
    assert torch.equal(lb[inside], la[inside])
    assert not lb[outside].any() and (b["pos"][outside] < 0).all()
    m = between & lit
    assert (lb[m] > 0).all() and (lb[m] < la[m]).all()
    s = ((torch.cos(torch.deg2rad(ang[m])) - spot.lights[0].cos_outer)
         / (spot.lights[0].cos_inner - spot.lights[0].cos_outer))
    assert torch.allclose((lb[m] / la[m]).double(), (s * s * (3 - 2 * s))[:, None].expand(-1, 3), atol=2e-4)


# ---- 4. argument checks ---------------------------------------------------------------------------------------------

def test_lights_arguments(host_so):
    lib = host_so
    lights = (_lib.TirLight * 17)()
    for l in lights:
        l.n_samples = 1
    buf = (C.c_float * 256)()
    ibuf = (C.c_int32 * 64)()
    dbuf = (C.c_double * 64)()
    cnt = (C.c_int64 * 1)()

    def sample(tab=lights, k=1, n=4, rays=buf, cap=8, lo=buf, cnt_=cnt):
        return lib.tir_lights_sample(tab, k, rays, buf, buf, buf, n, 0.5, dbuf, buf, buf, ibuf, lo, buf, cap, cnt_, None)

    def shade(tab=lights, k=1, n=4, stride=1, vis_kind=0, rows=4, row0=0, alb=buf, linear=buf, bg=buf):
        return lib.tir_lights_shade(tab, k, buf, buf, alb, buf, stride, buf, buf, n, 0.5, buf, bg, buf, buf, ibuf, buf,
                                    vis_kind, buf, buf, linear, rows, row0, None)
    assert sample() == 0 and shade() == 0 and shade(stride=3) == 0 and shade(linear=None) == 0
    assert sample(k=0, tab=None) == 0 and shade(k=0, tab=None) == 0 and sample(n=0) == 0 and shade(n=0) == 0
    for call in (sample, shade):
        assert call(n=-1) == -2 and call(k=-1) == -2 and call(k=17) == -2
        assert call(tab=None) == -1
        for bad in (0, -3, 1025):
            lights[0].n_samples = bad
            assert call() == -2 and call(n=0) == -2                  # checked before the empty early-out
        lights[0].n_samples = 1
        for bad in (3, -1):
            lights[0].type = bad
            assert call() == -3 and call(n=0) == -3
        lights[0].type = 0
    lights[0].n_samples, lights[1].n_samples = 1024, 1024
    assert sample(k=2, n=1 << 21) == -2 and shade(k=2, n=1 << 21, rows=1 << 21) == -2       # more than INT32_MAX slots
    lights[0].n_samples = lights[1].n_samples = 1
    assert sample(rays=None) == -1 and sample(cnt_=None) == -1 and sample(lo=None) == -1
    assert sample(cap=0, lo=None) == 0 and sample(cap=-1) == -2
    assert shade(stride=2) == -2 and shade(rows=3) == -2 and shade(row0=-1) == -2 and shade(rows=5, row0=2) == -2
    assert shade(vis_kind=2) == -3 and shade(vis_kind=-1) == -3
    assert shade(alb=None) == -1 and shade(bg=None) == -1


def test_light_struct_layout(tmp_path):
    src = tmp_path / "sz.c"
    names = ["type", "n_samples", "dir", "pos", "power", "extent", "cos_inner", "cos_outer"]
    offs = ",".join(f"offsetof(TirLight,{k})" for k in names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tensoir_b200.h"\n'
                   f'int main(void){{printf("%zu{" %zu" * len(names)} %d %d %d %d %d\\n",sizeof(TirLight),{offs},'
                   'TIR_LIGHTS_MAX,TIR_LIGHT_SAMPLES_MAX,TIR_LIGHT_DIRECTIONAL,TIR_LIGHT_POINT,TIR_LIGHT_SPOT);'
                   'return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    T = _lib.TirLight
    assert got == ([C.sizeof(T)] + [getattr(T, k).offset for k in names]
                   + [_lib.LIGHTS_MAX, _lib.LIGHT_SAMPLES_MAX, _lib.LIGHT_DIRECTIONAL, _lib.LIGHT_POINT,
                      _lib.LIGHT_SPOT])
