"""Camera-path frames under analytic light rigs, on the CPU.

tir_ground_lights_sample and tir_path_lights_composite are built for the host (tests/host_path_lights.cpp: the same C
ABI, argument checks and per-slot / per-pixel math of csrc/tir_path_body.h, loops instead of kernels) and driven
through the real ctypes wrappers of tensoir_b200.camera_path.  They are compared with a float64 restatement of the
definitions in include/tensoir_b200.h.  The per-frame rotation of a rig and the --rig options of tools/render_path.py
are checked here too."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from test_camera_path_cpu import GROUND_Z, _tool, ground_rays, slab64
from test_lighting_cpu import _disc64, _frame64, random_chunk, run_chunk
from tensoir_b200 import _lib, lighting
from tensoir_b200 import camera_path as P
from tensoir_b200.light_fit import linear_to_srgb, srgb_to_linear
from tensoir_b200.lighting import Light, Setup

EPS = float(np.finfo(np.float32).eps)
BOX = ([-0.6, -0.5, -0.7], [0.5, 0.7, 0.6])


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_path_lights"), "host_relight.cpp", "host_lights.cpp",
                          "host_path.cpp", "host_path_lights.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


def _spot(power, position, target, inner, outer, **kw):
    axis = lighting._unit(tuple(t - p for t, p in zip(target, position)), "")
    return Light("spot", power, position=position, direction=axis, cos_inner=math.cos(math.radians(inner)),
                 cos_outer=math.cos(math.radians(outer)), **kw)


# Every kind of light, hard and soft.  The hard point light sits low beside the box, so that many ground points see it
# with the box behind it: their shadow rays pass the light before they enter the box (the distance cull).
GROUND_RIG = Setup((
    Light("directional", (3.0, 3.0, 2.8), direction=lighting._unit((0.3, -0.2, 1.0), "")),
    Light("directional", (0.5, 0.6, 0.7), direction=lighting._unit((-0.5, 0.4, 0.6), ""),
          extent=math.tan(math.radians(6.0)), samples=8),
    Light("point", (40.0, 36.0, 30.0), position=(1.2, 0.1, -0.3)),
    Light("point", (20.0, 20.0, 20.0), position=(-1.5, -1.2, 1.6), extent=0.15, samples=16),
    _spot((60.0, 60.0, 60.0), (2.0, 2.0, 1.5), (0.0, 0.0, GROUND_Z), 25, 45),
    _spot((30.0, 20.0, 10.0), (-2.0, 1.5, 1.0), (0.0, 0.0, GROUND_Z), 20, 40, extent=0.2, samples=5),
), background=(0.8, 0.5, 0.25))


def sample64(l, p, uu):
    """The light sample of include/tensoir_b200.h seen from the points p [m,3] in float64, uu [m,K,2] -> (L [m,K,3],
    falloff [m,K], bound on the fp32 falloff's spot-cone error [m,K], distance to the sample [m,K], inf for a
    directional light)."""
    m, K = uu.shape[:2]
    centre = K == 1 or not l.extent > 0
    x, y = (torch.zeros(m, K, dtype=torch.float64),) * 2 if centre else _disc64(uu)
    axis = torch.tensor(l.direction, dtype=torch.float64)
    if l.kind == "directional":
        t1, t2 = _frame64(axis)
        q = axis + l.extent * (x[..., None] * t1 + y[..., None] * t2)
        L = q / q.norm(dim=-1, keepdim=True)
        one = torch.ones(m, K, dtype=torch.float64)
        return L, one, torch.zeros_like(one), torch.full_like(one, math.inf)
    c = torch.tensor(l.position, dtype=torch.float64)
    w = (c - p) / (c - p).norm(dim=-1, keepdim=True)
    t1, t2 = _frame64(w)
    q = c + l.extent * (x[..., None] * t1[:, None] + y[..., None] * t2[:, None])
    to = q - p[:, None]
    d = to.norm(dim=-1)
    L = to / d[..., None]
    cone, dcone = torch.ones(m, K, dtype=torch.float64), torch.zeros(m, K, dtype=torch.float64)
    if l.kind == "spot":
        cs = -(L * axis).sum(-1)
        s = ((cs - l.cos_outer) / max(l.cos_inner - l.cos_outer, 1e-300)).clamp(0, 1)
        cone = torch.where(cs >= l.cos_inner, 1.0, torch.where(cs <= l.cos_outer, 0.0, s * s * (3 - 2 * s)))
        if l.cos_inner > l.cos_outer:                      # smoothstep slope <= 1.5 on a cosine off by <= 8 eps
            dcone = torch.full_like(cone, 12 * EPS / (l.cos_inner - l.cos_outer))
    return L, cone / d ** 2, dcone / d ** 2, d


def run_ground_lights(monkeypatch, setup, rays, box, seed=1):
    """ground_lights_visibility on the host build with a march that records its list and returns seeded
    visibilities."""
    n = rays.shape[0]
    u = torch.rand(n * lighting.slots_per_ray(setup), 2, dtype=torch.float64,
                   generator=torch.Generator().manual_seed(seed))
    seen = {}

    def march(model, o, d, **kw):
        seen.update(o=o.clone(), d=d.clone(), table=kw["table"])
        v = torch.rand(o.shape[0], generator=torch.Generator().manual_seed(seed + 1))
        return v, 1 - v, torch.zeros_like(v)

    from tensoir_b200 import ops
    monkeypatch.setattr(ops, "march_density", march)
    g, pos, vis = P.ground_lights_visibility(types.SimpleNamespace(), setup, rays, GROUND_Z, box, u, "nerv",
                                             torch.linspace(0.05, 1.0, 8))
    return u, g, pos, vis, seen


def test_ground_lights_sample_against_float64(host_lib, monkeypatch):
    rays = ground_rays(13, 900)
    n = rays.shape[0]
    u, g, pos, vis, seen = run_ground_lights(monkeypatch, GROUND_RIG, rays, BOX)
    # the ground point as the kernels compute it (checked against float64 in test_camera_path_cpu)
    o, d = rays[:, :3].double(), rays[:, 3:].double()
    ground = (d[:, 2] < 0) & ((GROUND_Z - o[:, 2]) / d[:, 2] > 0)
    t32 = (torch.tensor(GROUND_Z, dtype=torch.float32) - rays[:, 2]) / rays[:, 5]
    p32 = rays[:, :3] + t32[:, None] * rays[:, 3:]
    p32[:, 2] = GROUND_Z
    p = p32.double()
    lo_in, hi_in = [x + 1e-4 for x in BOX[0]], [x - 1e-4 for x in BOX[1]]
    lo_out, hi_out = [x - 1e-4 for x in BOX[0]], [x + 1e-4 for x in BOX[1]]
    k0, sure_all, rows_all, culled_by_distance = 0, [], [], 0
    want_L, want_te = [], []
    for l in GROUND_RIG.lights:
        K = l.samples
        sl = slice(n * k0, n * (k0 + K))
        k0 += K
        L, fall, dfall, dist = sample64(l, p, u[sl].reshape(n, K, 2))
        g64 = fall * L[..., 2]
        gk, qk = g[sl].reshape(n, K).double(), pos[sl].reshape(n, K)
        # g = falloff * L.z: the falloff's fp32 error (16 eps relative plus the cone's), L.z's (8 eps) and the product's
        gm = ground[:, None].expand(n, K)
        assert ((gk - g64)[gm].abs() <= (32 * EPS * fall + dfall)[gm] + 1e-12).all()
        assert not gk[~gm].any() and (qk[~gm] == -1).all()
        # the codes
        joins = (L[..., 2] > 1e-6) & (g64 > 0)
        pf, Lf = p[:, None].expand(n, K, 3).reshape(-1, 3), L.reshape(-1, 3)
        hit, te = (x.reshape(n, K) for x in slab64(pf, Lf, *BOX))
        h_in, h_out = (slab64(pf, Lf, a, b)[0].reshape(n, K) for a, b in ((lo_in, hi_in), (lo_out, hi_out)))
        beyond = hit & (te >= dist)
        free = joins & (~hit | beyond)
        # membership that no fp32 rounding can change: L.z away from 1e-6, the falloff away from the cone's edge, the
        # shadow ray away from the box's faces and its entry away from the light's distance
        sure = (gm & ((L[..., 2] - 1e-6).abs() > 1e-5) & ((fall > 1e-6) | (fall == 0)) & (h_in == h_out)
                & (~hit | ((te - dist).abs() > 1e-4 * (1 + te))))
        assert sure[gm].float().mean() > 0.95, l
        assert torch.equal(qk[sure] == -1, ~joins[sure])
        assert torch.equal(qk[sure] == -2, free[sure])
        assert torch.equal(qk[sure] >= 0, (joins & ~free)[sure])
        culled_by_distance += int((sure & joins & beyond).sum())
        sure_all.append(sure.reshape(-1))
        rows_all.append(qk.reshape(-1))
        want_L.append(Lf)
        want_te.append(te.reshape(-1))
    assert culled_by_distance > 30                        # the hard point light low beside the box
    rows, sure = torch.cat(rows_all), torch.cat(sure_all)
    assert (rows == -2).sum() > 500 and (rows >= 0).sum() > 500
    # the list, in slot order: each row the slot's direction, its origin on the shadow ray, SHADOW_NEAR before the
    # entry
    marched = rows >= 0
    assert torch.equal(rows[marched].long(), torch.arange(int(marched.sum())))
    Ld, te = torch.cat(want_L)[marched], torch.cat(want_te)[marched]
    assert (seen["d"].double() - Ld).abs().max() < 8 * EPS
    ray_of = torch.cat([torch.arange(n).repeat_interleave(l.samples) for l in GROUND_RIG.lights])[marched]
    off = seen["o"].double() - p[ray_of]
    s = (off * Ld).sum(-1)
    assert (off - s[:, None] * Ld).abs().max() < 1e-5
    ok = sure[marched]
    assert ((s - (te - 0.05).clamp(min=0))[ok].abs() <= 1e-3 * (1 + te[ok])).all()
    # repeated calls give the same bits
    again = run_ground_lights(monkeypatch, GROUND_RIG, rays, BOX)
    assert torch.equal(again[1], g) and torch.equal(again[2], pos) and torch.equal(again[4]["o"], seen["o"])


def test_ground_lights_sample_without_ground_or_box(host_lib, monkeypatch):
    rays = ground_rays(4, 300)
    n = rays.shape[0]
    u = torch.rand(n * lighting.slots_per_ray(GROUND_RIG), 2, dtype=torch.float64)
    g, pos, _ = P.ground_lights_visibility(types.SimpleNamespace(), GROUND_RIG, rays, float("nan"), BOX, u, "nerv",
                                           torch.linspace(0.05, 1.0, 8))
    assert not g.any() and (pos == -1).all()
    _, g, pos, _, seen = run_ground_lights(monkeypatch, GROUND_RIG, rays, ([1.0, 1.0, 1.0], [-1.0, -1.0, -1.0]))
    assert set(pos.unique().tolist()) == {-1, -2} and "o" not in seen and (g[pos == -2] > 0).all()


def composite_inputs(setup, n, seed, vis_one=False):
    """Seeded g, pos and vis of n ground rays as tir_ground_lights_sample leaves them: g > 0 where pos != -1."""
    gen = torch.Generator().manual_seed(seed)
    slots = n * lighting.slots_per_ray(setup)
    g = torch.rand(slots, generator=gen) * 0.3
    r = torch.rand(slots, generator=gen)
    pos = torch.full((slots,), -1, dtype=torch.int32)
    pos[r < 0.9] = -2
    marched = r < 0.6
    pos[marched] = torch.arange(int(marched.sum()), dtype=torch.int32)
    g[pos == -1] = torch.where(torch.rand(int((pos == -1).sum()), generator=gen) < 0.5, 0.0, 0.1)
    m = max(int(marched.sum()), 1)
    vis = torch.ones(m) if vis_one else torch.rand(m, generator=gen)
    return g, pos, vis


def run_composite(setup, rays, acc, ground_z, visibility, wo=None):
    n = rays.shape[0]
    without = torch.rand(n + 2, 3, generator=torch.Generator().manual_seed(9)) if wo is None else wo
    with_bg = torch.full((n + 2, 3), -7.0)
    shadow = torch.full((n + 2, 3), -7.0)
    P.path_lights_composite(setup, rays, acc, ground_z, visibility, "nerv", (with_bg, without), 1, shadow)
    return with_bg, without, shadow


def ratio64(setup, g, pos, vis, n):
    num, den, k0 = torch.zeros(n, 3, dtype=torch.float64), torch.zeros(n, 3, dtype=torch.float64), 0
    for l in setup.lights:
        K = l.samples
        sl = slice(n * k0, n * (k0 + K))
        k0 += K
        gg, q = g[sl].reshape(n, K).double(), pos[sl].reshape(n, K).long()
        keep = (q != -1).double()
        v = torch.where(q >= 0, vis.double()[q.clamp(min=0)], torch.ones_like(gg))
        power = torch.tensor(l.power, dtype=torch.float64)
        num += power * ((gg * v * keep).sum(1) / K)[:, None]
        den += power * ((gg * keep).sum(1) / K)[:, None]
    return torch.where(den > 0, (num / den).clamp(0, 1), torch.ones_like(den))


def test_composite_ratio_against_float64(host_lib):
    n = 500
    rays = ground_rays(5, n)
    acc = torch.rand(n, generator=torch.Generator().manual_seed(2))
    g, pos, vis = composite_inputs(GROUND_RIG, n, 11)
    with_bg, without, shadow = run_composite(GROUND_RIG, rays, acc, GROUND_Z, (g, pos, vis))
    assert (with_bg[0] == -7).all() and (with_bg[-1] == -7).all() and (shadow[0] == -7).all()
    r64 = ratio64(GROUND_RIG, g, pos, vis, n)
    d = rays[:, 5].double()
    ground = (d < 0) & ((GROUND_Z - rays[:, 2].double()) / d > 0)
    r64[~ground] = 1
    # per light: each term one rounding, the lane sums and the butterfly at most K - 1 additions, the mean and the
    # power two more; the lights' sums J - 1 more; num <= den, so the quotient is off by at most twice the relative
    # error of the sums
    K, J = max(l.samples for l in GROUND_RIG.lights), len(GROUND_RIG.lights)
    bound = (2 * (K + J + 4) + 2) * EPS * (r64 + 1)
    r = shadow[1:-1].double()
    assert ((r - r64).abs() <= bound).all()
    assert (r[~ground] == 1).all() and (r[ground] < 0.9).float().mean() > 0.5
    # the background: where r_c < 1 the linear background times r, tone-mapped; acc_t = 0 leaves it alone
    wb0, _, _ = run_composite(GROUND_RIG, rays, torch.zeros(n), GROUND_Z, (g, pos, vis))
    lin = srgb_to_linear(torch.tensor(GROUND_RIG.background)).float().double()    # the fp32 value the kernel reads
    want = linear_to_srgb(lin * r)
    dark = r < 1
    # fp32: the product (one rounding, under the curve's slope <= 12.92) and powf (a few ulps)
    assert ((wb0[1:-1].double() - want)[dark].abs() <= 13 * 2 * EPS * lin.expand_as(r)[dark] + 8 * EPS).all()
    assert torch.equal(wb0[1:-1][~dark], torch.tensor(GROUND_RIG.background).float().expand(n, 3)[~dark])
    # the composite under the object: lt_finish's expression
    acc_t = torch.where(acc > 0.9, acc, torch.zeros_like(acc))[:, None]
    want_wb = acc_t * without[1:-1] + (1 - acc_t) * wb0[1:-1]
    assert (with_bg[1:-1] - want_wb).abs().max() < 4 * EPS


def test_composite_unoccluded_is_exactly_one(host_lib):
    n = 300
    rays = ground_rays(6, n)
    g, pos, vis = composite_inputs(GROUND_RIG, n, 12, vis_one=True)
    wb, _, shadow = run_composite(GROUND_RIG, rays, torch.zeros(n), GROUND_Z, (g, pos, vis))
    assert (shadow[1:-1] == 1).all()
    assert torch.equal(wb[1:-1], torch.tensor(GROUND_RIG.background).expand(n, 3))


@pytest.mark.parametrize("vis_kind", [0, 1])
def test_composite_without_ground_is_lights_shade(host_lib, vis_kind):
    """No ground: with_bg has the bits of the host tir_lights_shade's."""
    n = 400
    ch = random_chunk(21, n, 3)
    u = torch.rand(n * lighting.slots_per_ray(GROUND_RIG), 2, dtype=torch.float64,
                   generator=torch.Generator().manual_seed(4))
    res = run_chunk(GROUND_RIG, ch, u, vis_kind, [1.1, 0.9, 1.0])
    with_bg = torch.full_like(res["with_bg"], -7.0)
    P.path_lights_composite(GROUND_RIG, ch["rays"], ch["acc"], None, None, "nerfactor" if vis_kind else "nerv",
                            (with_bg, res["without_bg"]), 2)
    assert torch.equal(with_bg, res["with_bg"])


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def test_argument_checks_write_nothing(host_so):
    lib = host_so
    setup = Setup((GROUND_RIG.lights[2], GROUND_RIG.lights[3]))
    tab = lighting.light_table(setup)
    n = 8
    slots = n * lighting.slots_per_ray(setup)
    rays, acc = ground_rays(1, n), torch.ones(n)
    u = torch.rand(slots, 2, dtype=torch.float64)
    g, pos = torch.full((slots,), 77.0), torch.full((slots,), 77, dtype=torch.int32)
    lo, ld = torch.full((slots, 3), 5.0), torch.full((slots, 3), 5.0)
    cnt = torch.zeros(1, dtype=torch.int64)
    blo, bhi = (C.c_float * 3)(*BOX[0]), (C.c_float * 3)(*BOX[1])
    bad_type = lighting.light_table(setup)
    bad_type[1].type = 7
    bad_k = lighting.light_table(setup)
    bad_k[0].n_samples = 0
    many = (_lib.TirLight * 17)(*([tab[0]] * 17))

    def sample(tab=tab, J=2, rays=rays, n=n, blo=blo, bhi=bhi, u=u, g=g, pos=pos, lo=lo, ld=ld, cap=slots, cnt=cnt):
        return lib.tir_ground_lights_sample(tab, J, _ptr(rays), n, GROUND_Z, blo, bhi, _ptr(u), _ptr(g), _ptr(pos),
                                            _ptr(lo), _ptr(ld), cap, _ptr(cnt), None)

    for rc, kw in ((-1, dict(rays=None)), (-1, dict(u=None)), (-1, dict(g=None)), (-1, dict(pos=None)),
                   (-1, dict(cnt=None)), (-1, dict(blo=None)), (-1, dict(bhi=None)), (-1, dict(lo=None)),
                   (-1, dict(tab=None)), (-2, dict(tab=many, J=17)), (-2, dict(n=-1)), (-2, dict(J=-1)),
                   (-2, dict(cap=-1)), (-2, dict(tab=bad_k)), (-3, dict(tab=bad_type))):
        assert sample(**kw) == rc, kw
        assert (g == 77).all() and (pos == 77).all() and (lo == 5).all() and int(cnt) == 0
    assert sample() == 0 and int(cnt) >= 0 and (pos != 77).all()

    vis = torch.rand(slots)
    wo, wb = torch.rand(n, 3), torch.full((n, 3), -7.0)
    bg = (C.c_float * 3)(*GROUND_RIG.background)

    def comp(tab=tab, J=2, rays=rays, acc=acc, n=n, gz=GROUND_Z, bg=bg, bgl=bg, g=g, pos=pos, vis=vis, kind=0, wo=wo,
             wb=wb, rows=n, row0=0):
        return lib.tir_path_lights_composite(tab, J, _ptr(rays), _ptr(acc), n, gz, bg, bgl, _ptr(g), _ptr(pos),
                                             _ptr(vis), kind, _ptr(wo), _ptr(wb), None, rows, row0, None)

    for rc, kw in ((-1, dict(rays=None)), (-1, dict(acc=None)), (-1, dict(bg=None)), (-1, dict(bgl=None)),
                   (-1, dict(wo=None)), (-1, dict(wb=None)), (-1, dict(g=None)), (-1, dict(pos=None)),
                   (-1, dict(vis=None)), (-1, dict(tab=None)), (-2, dict(tab=many, J=17)), (-2, dict(tab=bad_k)),
                   (-3, dict(tab=bad_type)), (-3, dict(kind=2)), (-2, dict(rows=n - 1)), (-2, dict(row0=1)),
                   (-2, dict(row0=-1)), (-2, dict(n=-1))):
        assert comp(**kw) == rc, kw
        assert (wb == -7).all()
    # without a ground, g / pos / vis are not read
    assert comp(gz=float("nan"), g=None, pos=None, vis=None) == 0 and (wb != -7).all()


# ---- turning a rig per frame ----------------------------------------------------------------------------------------

def test_rotated_setup_is_float64_rotation_rounded_once():
    for a in (37.0, 90.0, -123.5, 360.0):
        turned = P.rotated_setup(GROUND_RIG, a)
        R64 = P.rotation_matrix(a).double().numpy()
        got, src = lighting.light_table(turned), GROUND_RIG.lights
        for k, l in enumerate(src):
            for field, v in (("dir", l.direction), ("pos", l.position)):
                want = (R64 @ np.asarray(v, np.float64)).astype(np.float32)
                assert np.array_equal(np.asarray(getattr(got[k], field)[:], np.float32), want), (a, k, field)
            assert turned.lights[k].power == l.power and turned.lights[k].extent == l.extent
            assert (turned.lights[k].cos_inner, turned.lights[k].samples) == (l.cos_inner, l.samples)
        assert turned.background == GROUND_RIG.background
    # the convention: a map rotated by a lights from w where its lookup w @ R(a) is the texel, so a light authored at
    # d arrives from R(a) d, whose lookup is d again
    d = np.asarray(GROUND_RIG.lights[0].direction)
    back = np.asarray(P.rotated_setup(GROUND_RIG, 90.0).lights[0].direction) @ P.rotation_matrix(90.0).double().numpy()
    assert np.allclose(back, d, atol=1e-6)
    # the identity leaves the table bit for bit
    same, orig = lighting.light_table(P.rotated_setup(GROUND_RIG, 0.0)), lighting.light_table(GROUND_RIG)
    assert C.string_at(same, C.sizeof(same)) == C.string_at(orig, C.sizeof(orig))


def test_frame_rigs_reject_a_light_turned_into_the_aabb():
    aabb = torch.tensor([[-3.0, -0.5, -1.0], [3.0, 0.5, 1.0]])                  # long in x, thin in y
    rig = lighting.load_rig({"key": {"lights": [{"type": "directional", "direction": [0, 0, 1], "irradiance": 1}]},
                             "lamp": {"lights": [{"type": "directional", "direction": [1, 0, 1], "irradiance": 1},
                                                 {"type": "point", "position": [0, 2, 0], "intensity": 5}]}})
    rigs = P.frame_rigs(rig, [0.0, 10.0], aabb)
    assert len(rigs) == 2 and list(rigs[1]) == ["key", "lamp"]
    with pytest.raises(ValueError, match=r"frame 2 \(rotation 90 degrees\): setup 'lamp' light 1"):
        P.frame_rigs(rig, [0.0, 45.0, 90.0], aabb)


def test_render_path_rejects_a_rig_with_learned_lights(tmp_path):
    args = types.SimpleNamespace(out=str(tmp_path), batch_size=16, light="learned")
    rig = {"s": {"lights": [{"type": "directional", "direction": [0, 0, 1], "irradiance": 1}]}}
    with pytest.raises(ValueError, match="light must be unset"):
        P.render_path(None, args, torch.eye(4)[None], [0.0], tensoIR=object(), rig=rig)
    for extra in (dict(sampling="mis"), dict(indirect_samples=2)):
        with pytest.raises(ValueError):
            P.render_path(None, types.SimpleNamespace(out=str(tmp_path), batch_size=16, **extra), torch.eye(4)[None],
                          [0.0], tensoIR=object(), rig=rig)


# ---- the command line -----------------------------------------------------------------------------------------------

def test_rig_options(tmp_path):
    tool = _tool()
    rig = tmp_path / "rig.json"
    rig.write_text('{"s": {"lights": [{"type": "directional", "direction": [0, 0, 1], "irradiance": 1}]}}')
    argv = ["x", "--config", "c.txt", "--rig", str(rig), "--shadow_far", "2.5", "--path", "orbit", "--ground",
            "--out", "o"]
    assert tool.rig_options(argv) == dict(rig=str(rig), shadow_far=2.5)
    assert argv == ["x", "--config", "c.txt", "--path", "orbit", "--ground", "--out", "o"]
    # path_options sees what is left, and returns what it always has
    assert tool.path_options(argv) == dict(path=("orbit", "orbit"), frames=120, rotation=(0.0, 0.0), ground=True,
                                           light=None, out="o")
    argv = ["x", "--rig", str(rig), "--out", "o"]
    assert tool.rig_options(argv) == dict(rig=str(rig), shadow_far=None) and argv == ["x", "--out", "o"]
    argv = ["x", "--light", "learned", "--out", "o"]
    assert tool.rig_options(argv) == dict(rig=None, shadow_far=None) and len(argv) == 5
    for bad in (["--rig", str(rig), "--light", "learned"],
                ["--light", "learned", "--rig", str(rig)],
                ["--shadow_far", "2.0"],
                ["--rig", str(rig), "--shadow_far", "0.01"],
                ["--rig", str(rig), "--shadow_far", "nan"],
                ["--rig", str(rig), "--shadow_far", "far"],
                ["--rig", str(tmp_path / "missing.json")],
                ["--rig"]):
        with pytest.raises(SystemExit):
            tool.rig_options(["x"] + bad + ["--out", "o"])
    assert "--rig" in tool.USAGE and "--shadow_far" in tool.USAGE and "--rig" in tool.__doc__
