"""Relighting with one bounce of indirect light, on the CPU.

The indirect entry points are built for the host (tests/host_indirect.cpp: the same C ABI, argument checks and
per-slot math of csrc/tir_indirect_body.h, loops instead of kernels), together with the environment-map pass
(tests/host_relight.cpp), and driven through the real ctypes wrappers in tensoir_b200.indirect.  Each stage is
compared with a float64 restatement of the definitions in include/tensoir_b200.h, within a bound derived from the fp32
expressions.  The sampler is checked for unbiasedness in float64 against quadrature."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from tensoir_b200 import _lib, indirect, relighting
from tensoir_b200.relight import Environment_Light
from tensoir_b200.relight_utils import GGX_specular
from test_lighting_cpu import random_chunk

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
EPS = float(np.finfo(np.float32).eps)
AABB = torch.tensor([[-1.5] * 3, [1.5] * 3])


class Model:
    """What the indirect path reads of a model besides the march: the aabb and its normalisation."""
    aabb = AABB
    invaabbSize = 2.0 / (AABB[1] - AABB[0])

    def normalize_coord(self, x):
        return (x - self.aabb[0]) * self.invaabbSize - 1


def plane_march(z_plane=0.2, t_last=0.25):
    """A march through a horizontal slab at z = z_plane: a ray that crosses it within relight()'s [0.05, 1.5] ends with
    transmittance t_last, acc 1 - t_last and depth acc * t, so x = p + (depth / acc) d lies on the plane."""
    def march(model, rays_o, rays_d, *, table=None, counters=None, **kw):
        o, d = rays_o.double(), rays_d.double()
        t = (z_plane - o[:, 2]) / torch.where(d[:, 2] == 0, torch.full_like(d[:, 2], 1e-30), d[:, 2])
        crosses = (t >= 0.05) & (t <= 1.5)
        acc = torch.where(crosses, 1.0 - t_last, 0.0)
        return (torch.where(crosses, t_last, 1.0).float(), acc.float(), (acc * t).float())
    return march


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_indirect"), "host_relight.cpp", "host_indirect.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so, plane_march())
    return host_so


def env_light(names, H=8, W=16, seed=0):
    g = np.random.default_rng(seed)
    return Environment_Light({k: g.uniform(0.05, 2.0, (H, W, 3)).astype(np.float32) for k in names}, device="cpu")


def analytic_material(x):
    """A material that varies over space, in the heads' ranges."""
    m = x.shape[0]
    s = torch.sin(3 * x)
    normal = torch.stack([0.3 * s[:, 0], 0.2 * s[:, 1], torch.ones(m, device=x.device)], -1)
    normal = normal / normal.norm(dim=-1, keepdim=True)
    albedo = 0.5 + 0.4 * torch.cos(2 * x)
    rough = 0.3 + 0.5 * (0.5 + 0.5 * s[:, 2:3])
    return normal.contiguous(), albedo.contiguous(), rough.contiguous(), torch.full((m, 3), 0.04, device=x.device)


def chunk(seed, n, stride=1):
    ch = random_chunk(seed, n, stride)
    return ch, (ch["depth"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"])


# ---- float64 restatements ---------------------------------------------------------------------------------------------

def disc64(u):
    """lt_disc in float64 (Shirley & Chiu's concentric map)."""
    a, b = 2 * u[..., 0] - 1, 2 * u[..., 1] - 1
    big = a.abs() > b.abs()
    r = torch.where(big, a, b)
    phi = torch.where(big, math.pi / 4 * (b / torch.where(a == 0, 1.0, a)),
                      math.pi / 2 - math.pi / 4 * (a / torch.where(b == 0, 1.0, b)))
    x, y = r * torch.cos(phi), r * torch.sin(phi)
    zero = (a == 0) & (b == 0)
    return torch.where(zero, 0.0, x), torch.where(zero, 0.0, y)


def frame64(w):
    s = torch.where(w[..., 2] >= 0, 1.0, -1.0)
    a = -1 / (s + w[..., 2])
    b = w[..., 0] * w[..., 1] * a
    t1 = torch.stack([1 + s * w[..., 0] ** 2 * a, s * b, -s * w[..., 0]], -1)
    t2 = torch.stack([b, s + w[..., 1] ** 2 * a, -w[..., 1]], -1)
    return t1, t2


def directions64(normal, u):
    """omega [n,K,3] and z [n,K] of the header's sampler in float64."""
    nh = torch.nn.functional.normalize(normal.double(), dim=-1)[:, None].expand(-1, u.shape[1], -1)
    t1, t2 = frame64(nh)
    x, y = disc64(u.double())
    z = (1 - x * x - y * y).clamp(min=0).sqrt()
    return x[..., None] * t1 + y[..., None] * t2 + z[..., None] * nh, z


def brdf64(normal, view, L, albedo, rough, fresnel):
    """(albedo/pi + GGX) [n,K,3], the raw cosine L . normal [n,K] and nom0 of GGX (for the bound), in float64."""
    normal, view, L = normal.double(), view.double(), L.double()
    spec = GGX_specular(normal, view, L, rough.double(), fresnel.double())
    V = torch.nn.functional.normalize(view, dim=-1)
    N = torch.nn.functional.normalize(normal, dim=-1)
    N = N * (V * N).sum(-1, keepdim=True).sign()
    Hh = torch.nn.functional.normalize(torch.nn.functional.normalize(L, dim=-1) + V[:, None], dim=-1)
    NoH = (N[:, None] * Hh).sum(-1, keepdim=True).clamp(1e-6, 1)
    nom0 = NoH * NoH * ((rough.double() ** 4)[:, None] - 1) + 1
    return albedo.double()[:, None] / math.pi + spec, (L * normal[:, None]).sum(-1), spec, nom0


# ---- 1. sampler: directions, throughput, list ------------------------------------------------------------------------

def run_sample(ch, K, seed, rescale=(1.1, 0.9, 1.0)):
    n = ch["rays"].shape[0]
    u = torch.rand(n, K, 2, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    resc = torch.tensor(rescale, dtype=torch.float32)
    hits = indirect.secondary_hits(Model(), ch["rays"], ch["depth"], ch["normal"], ch["albedo"], ch["rough"],
                                   ch["fresnel"], ch["acc"], resc, u, 0.5, 'nerv')
    return u, resc, hits


@pytest.mark.parametrize("stride", [1, 3])
def test_sample_matches_float64(host_lib, stride):
    n, K = 300, 24
    ch = random_chunk(11 + stride, n, stride)
    u, resc, res = run_sample(ch, K, stride)
    hit = ch["acc"] > 0.5
    om = res["dirs"].double()
    om64, z64 = directions64(ch["normal"], u)
    # directions: unit, on n^'s hemisphere, and the float64 map within its fp32 error: n^ and the frame ~8 eps each,
    # the disc rounded once, z = sqrt(1 - x^2 - y^2) with an absolute error ~3 eps / (2 z)
    assert not om[~hit].any()
    dz = EPS * (24 + 3 / z64.clamp(min=1e-30))
    assert ((om - om64)[hit].abs() <= dz[hit][..., None]).all()
    nh = torch.nn.functional.normalize(ch["normal"].double(), dim=-1)
    assert ((om.norm(dim=-1) - 1)[hit].abs() <= 32 * EPS).all()
    assert ((om * nh[:, None]).sum(-1)[hit] >= -dz[hit]).all()
    # throughput: rl_contrib's term with vis * rgb = 1 and pdf = z / pi, on the kernel's own direction
    B, cos, spec, nom0 = brdf64(ch["normal"], -ch["rays"][:, 3:], res["dirs"], ch["albedo"] * resc, ch["rough"],
                                ch["fresnel"])
    cos32 = (res["dirs"] * ch["normal"][:, None]).sum(-1)        # the cut in the kernel's fp32 cosine, re-evaluated
    ok = hit[:, None] & (cos32 > 1e-6) & (z64 > 1e-6)
    w = cos / (z64 / math.pi)
    T64 = B * w[..., None]
    bound = EPS * (32 * T64.abs() + 16 * (spec * w[..., None]).abs() / nom0
                   + 8 * B * (ch["normal"].double().norm(dim=-1)[:, None] / (z64 / math.pi))[..., None]
                   + 4 * T64.abs() / z64.clamp(min=1e-30)[..., None] ** 2)
    T = res["T"].double()
    marched = res["pos"] >= 0
    assert torch.equal(marched, ok) and ok.any() and (~ok).any()
    err = (T - T64).abs()[ok]
    assert (err <= bound[ok]).all(), float((err / bound[ok]).max())
    assert float((err / bound[ok]).max()) > 1e-3
    assert not T[~ok].any()
    # pos -1 on non-hit rays and failed slots; list rows in slot order in the host build; origins have the bits of
    # tir_relight_sample's (rl_surface)
    assert (res["pos"][~hit] == -1).all()
    rows = res["pos"][marched].long()
    assert torch.equal(rows, torch.arange(rows.shape[0]))
    i, _ = marched.nonzero(as_tuple=True)
    names = ["a"]
    env = env_light(names)
    envs, keep = relighting.env_tables(env, names)
    u1 = torch.rand(1, n, 4, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    lo = torch.empty(n * 4, 3)
    cnt = torch.zeros(1, dtype=torch.int64)
    bins, pos = torch.empty(1, n, 4, dtype=torch.int32), torch.empty(1, n, 4, dtype=torch.int32)
    assert host_lib.tir_relight_sample(envs, 1, *(C.c_void_p(t.data_ptr()) for t in (ch["rays"], ch["depth"],
                                                                                       ch["normal"], ch["acc"])),
                                       n, 4, 0.5, C.c_void_p(u1.data_ptr()), C.c_void_p(bins.data_ptr()),
                                       C.c_void_p(pos.data_ptr()), C.c_void_p(lo.data_ptr()),
                                       C.c_void_p(torch.empty(n * 4, 3).data_ptr()), n * 4,
                                       C.c_void_p(cnt.data_ptr()), None) == 0
    origin = torch.full((n, 3), float("nan"))
    has = pos[0] >= 0
    ri, si = has.nonzero(as_tuple=True)
    origin[ri] = lo[pos[0][ri, si].long()]
    both = torch.isfinite(origin[i]).all(-1)
    assert both.sum() > 50
    assert torch.equal(res["list_o"][rows][both], origin[i][both])
    assert torch.equal(res["list_d"][rows], res["dirs"][marched])


@pytest.mark.parametrize("rough", [0.8, 0.2])
def test_sampler_is_unbiased(rough):
    """E[T] = the directional albedo: the integral of (albedo/pi + GGX) cos over the hemisphere, by quadrature."""
    g = torch.Generator().manual_seed(int(rough * 10))
    normal = torch.tensor([[0.3, -0.2, 0.9]], dtype=torch.float64)
    view = torch.tensor([[0.5, 0.1, 0.8]], dtype=torch.float64)
    albedo = torch.tensor([[0.6, 0.4, 0.2]], dtype=torch.float64)
    r = torch.full((1, 1), rough, dtype=torch.float64)
    fres = torch.full((1, 3), 0.04, dtype=torch.float64)
    N = 400000
    u = torch.rand(1, N, 2, generator=g, dtype=torch.float64)
    om, z = directions64(normal, u)
    B, cos, _, _ = brdf64(normal, view, om, albedo, r, fres)
    T = (B * (cos / (z / math.pi))[..., None])[0]
    mean, sigma = T.mean(0), T.std(0) / math.sqrt(N)
    # quadrature in the normal's frame: midpoint rule in (cos theta, phi)
    nq, mq = 2000, 512
    ct = (torch.arange(nq, dtype=torch.float64) + 0.5) / nq
    ph = (torch.arange(mq, dtype=torch.float64) + 0.5) / mq * 2 * math.pi
    ct, ph = torch.meshgrid(ct, ph, indexing="ij")
    st = (1 - ct * ct).sqrt()
    nh = torch.nn.functional.normalize(normal, dim=-1)
    t1, t2 = frame64(nh)
    d = (st * ph.cos()).reshape(-1, 1) * t1 + (st * ph.sin()).reshape(-1, 1) * t2 + ct.reshape(-1, 1) * nh
    Bq, cq, _, _ = brdf64(normal, view, d[None], albedo, r, fres)
    quad = (Bq[0] * cq[0, :, None]).sum(0) * (2 * math.pi / (nq * mq))
    assert ((mean - quad).abs() <= 4 * sigma + 1e-3 * quad).all(), (mean, quad, sigma)


# ---- 2. secondary hits ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("vis_kind", [0, 1])
def test_hits_compaction(host_so, vis_kind):
    g = torch.Generator().manual_seed(3 + vis_kind)
    n, K, m = 60, 7, 300
    pos = torch.randperm(n * K, generator=g)[:m]
    posm = torch.full((n * K,), -1, dtype=torch.int32)
    posm[pos] = torch.randperm(m, generator=g).int()
    list_o = torch.rand(m, 3, generator=g) * 2 - 1
    list_d = torch.nn.functional.normalize(torch.randn(m, 3, generator=g), dim=-1)
    t_last = torch.rand(m, generator=g)
    acc = 1 - torch.rand(m, generator=g)
    one_minus = np.float32(1) - np.float32(1e-3)
    near = torch.tensor(np.array([one_minus, np.nextafter(one_minus, 0, dtype=np.float32),
                                  np.nextafter(one_minus, 1, dtype=np.float32), 1.0], dtype=np.float32))
    if vis_kind == 0:
        t_last[:4] = near
    else:
        acc[:4] = torch.tensor(np.float32(1) - near.numpy())
    acc[10:20] = 0
    depth = acc * (0.05 + 1.4 * torch.rand(m, generator=g))
    hit = torch.empty(n * K, dtype=torch.int32)
    rays, xn, w = torch.empty(m, 6), torch.empty(m, 3), torch.empty(m)
    count = torch.zeros(1, dtype=torch.int64)
    aabb = (C.c_float * 6)(*AABB[0].tolist(), *Model.invaabbSize.tolist())
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert host_so.tir_indirect_hits(n, K, p(posm), p(list_o), p(list_d), p(t_last), p(acc), p(depth), vis_kind,
                                     aabb, p(rays), p(xn), p(w), p(hit), m, p(count), None, 0, None) == 0
    vis = (np.float32(1) - acc.numpy()) if vis_kind else t_last.numpy()
    w32 = np.float32(1) - vis
    flag = (w32 > np.float32(1e-3)) & (acc.numpy() > 0)
    want = posm >= 0
    want[want.clone()] = torch.from_numpy(flag)[posm[posm >= 0].long()]
    m_h = int(want.sum())
    assert int(count) == m_h and 0 < m_h < m
    assert torch.equal(hit >= 0, want)
    assert torch.equal(hit[want], torch.arange(m_h, dtype=torch.int32))          # slot order
    q = posm[want].long()
    assert torch.equal(w[:m_h], torch.from_numpy(w32)[q])
    if vis_kind == 0:                                                           # the 1e-3 cut, at its fp32 neighbours
        assert [bool(flag[k]) for k in range(4)] == [False, True, False, False]
    x64 = list_o.double()[q] + (depth.double()[q] / acc.double()[q])[:, None] * list_d.double()[q]
    t = (depth / acc).double()[q]
    bound = EPS * (list_o.double()[q].abs() + 3 * t[:, None] * list_d.double()[q].abs())
    assert ((rays[:m_h, :3].double() - x64).abs() <= bound).all()
    assert torch.equal(rays[:m_h, 3:], list_d[q])
    assert torch.equal(xn[:m_h], (rays[:m_h, :3] - AABB[0]) * Model.invaabbSize - 1)


# ---- 3. radiance and shade --------------------------------------------------------------------------------------------

def test_radiance_and_shade_match_float64(host_lib):
    names = ["a", "b"]
    env = env_light(names, seed=1)
    n, K, S, S2 = 200, 8, 64, 16
    ch, maps = chunk(21, n)
    u = torch.rand(2, n, S, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    gen = torch.Generator().manual_seed(2)
    seen = {}

    def material(x):
        seen["x"] = x.clone()
        seen["mats"] = analytic_material(x)
        return seen["mats"]
    ind = torch.zeros(2, n, 3)
    wb, wo = indirect.relight_chunk_indirect(Model(), env, names, ch["rays"], maps, [1.0, 1.0, 1.0], u, gen,
                                             indirect_samples=K, indirect_light_samples=S2, material=material,
                                             indirect_out=ind)
    # replay the draws to get every stage's inputs
    gen = torch.Generator().manual_seed(2)
    u_ind = torch.rand(n, K, 2, generator=gen, dtype=torch.float64)
    resc = torch.ones(3)
    hits = indirect.secondary_hits(Model(), ch["rays"], ch["depth"], ch["normal"], ch["albedo"], ch["rough"],
                                   ch["fresnel"], ch["acc"], resc, u_ind, 0.5, 'nerv')
    m_h = hits["rays"].shape[0]
    assert m_h > 20 and torch.equal(seen["x"], hits["rays"][:, :3])
    assert torch.allclose(hits["rays"][:, 2], torch.full((m_h,), 0.2), atol=1e-5)    # on the slab
    u2 = torch.rand(2, m_h, S2, generator=gen, dtype=torch.float64)
    envs, keep = relighting.env_tables(env, names)
    normal, albedo, rough, fresnel = seen["mats"]
    Lo = torch.zeros(2, m_h, 3)
    indirect.secondary_radiance(Model(), envs, 2, hits, seen["mats"], resc, Lo, 0, u2, 'nerv')
    # Lo in float64 from the sampled bins and the march's visibility
    bins, pos, vis = relighting.relight_visibility(Model(), envs, 2, hits["rays"], torch.zeros(m_h), normal,
                                                   torch.ones(m_h), u2, S2, 0.5, 'nerv')
    for l, name in enumerate(names):
        b = bins[l].long()
        Ld = env.hdr_dir[name].reshape(-1, 3)[b].float()
        rgb = env.hdr_rgbs[name].reshape(-1, 3)[b].double()
        pdf = env.hdr_pdf_return[name].reshape(-1)[b].double()
        v = torch.where(pos[l] >= 0, vis.double()[pos[l].long().clamp(min=0)], 0.0)
        B, cos, spec, nom0 = brdf64(normal, -hits["rays"][:, 3:], Ld, albedo, rough, fresnel)
        wgt = (v * cos)[..., None] * rgb / pdf[..., None]
        term = B * wgt
        bnd = EPS * (32 * term.abs() + 16 * (spec * wgt).abs() / nom0
                     + 8 * B * (v[..., None] * rgb / pdf[..., None]) * normal.double().norm(dim=-1)[:, None, None])
        lo64 = term.mean(1)
        bound = bnd.mean(1) + S2 * EPS * term.abs().mean(1)
        assert ((Lo[l].double() - lo64).abs() <= bound + 1e-30).all()
    # the indirect term from the fp32 T, w and Lo
    hit = hits["hit"]
    h = hit.long().clamp(min=0)
    terms = (hits["T"].double()[None] * hits["w"].double()[h][None, ..., None] * Lo.double()[:, h]
             * (hit >= 0)[None, ..., None])
    ind64 = terms.sum(2) / K
    bound = EPS * (3 * terms.abs().sum(2) + K * terms.abs().sum(2)) / K
    assert ((ind.double() - ind64).abs() <= bound + 1e-30).all()
    some = (hit >= 0).any(1)
    assert some.any() and not ind[:, ~some].any()
    # the outputs: tone(direct + indirect) with the direct term of relight_chunk_fused
    fwb, fwo = relighting.relight_chunk_fused(Model(), env, names, ch["rays"], maps, [1.0, 1.0, 1.0], u, S)
    assert torch.equal(wo[:, ~some], fwo[:, ~some]) and torch.equal(wb[:, ~some], fwb[:, ~some])
    hitrow = some & (ch["acc"] > 0.5)
    assert (wo[:, hitrow] >= fwo[:, hitrow]).all() and (wb[:, hitrow] >= fwb[:, hitrow]).all()
    assert (wo[:, hitrow] > fwo[:, hitrow]).any()


def test_direct_term_unchanged_where_every_slot_misses(host_so, monkeypatch):
    use_host(monkeypatch, host_so, plane_march(z_plane=50.0))
    names = ["a"]
    env = env_light(names, seed=4)
    ch, maps = chunk(8, 150, 3)
    u = torch.rand(1, 150, 64, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    for vis in ("nerv", "nerfactor"):
        ind = torch.full((1, 150, 3), 7.0)
        a = indirect.relight_chunk_indirect(Model(), env, names, ch["rays"], maps, 1.0, u, torch.Generator(),
                                            indirect_samples=4, material=analytic_material, vis_equation=vis,
                                            indirect_out=ind)
        b = relighting.relight_chunk_fused(Model(), env, names, ch["rays"], maps, 1.0, u, 64, vis_equation=vis)
        assert all(torch.equal(x, y) for x, y in zip(a, b)) and not ind.any()


def test_more_maps_than_one_call_takes_and_determinism(host_lib):
    G = _lib.RELIGHT_MAX_LIGHTS
    names = [f"m{k}" for k in range(G + 2)]
    env = env_light(names, H=4, W=8, seed=6)
    ch, maps = chunk(30, 40)
    u = torch.rand(len(names), 40, 32, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    run = lambda: indirect.relight_chunk_indirect(Model(), env, names, ch["rays"], maps, 1.0, u,  # noqa: E731
                                                  torch.Generator().manual_seed(4), indirect_samples=6,
                                                  indirect_light_samples=8, material=analytic_material)
    a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert a[0].shape == (G + 2, 40, 3) and torch.isfinite(a[0]).all()
    # the direct term of every group is relight_chunk_fused's
    wb, wo = relighting.relight_chunk_fused(Model(), env, names, ch["rays"], maps, 1.0, u, 32)
    assert (a[1] >= wo).all() and (a[1] > wo).any()


# ---- 4. arguments -----------------------------------------------------------------------------------------------------

def test_indirect_arguments(host_so):
    lib = host_so
    v = C.c_void_p(8)
    envs = (_lib.TirEnvMap * 1)()
    envs[0].H, envs[0].W = 2, 2
    envs[0].rgb = envs[0].dir = envs[0].pdf_return = envs[0].cdf = 8
    cnt = C.c_int64(0)
    aabb = (C.c_float * 6)()
    S = lambda K=4, n=1, rs=1, cap=4: lib.tir_indirect_sample(v, v, v, v, v, rs, v, v, n, K, 0.5, v, v, v, v, v, v,  # noqa: E731
                                                             v, cap, v, None)
    assert S(n=0) == 0
    assert S(K=0) == -2 and S(K=1025) == -2 and S(rs=2) == -2 and S(cap=-1) == -2
    assert S(n=(1 << 31) // 4 + 1) == -2
    assert lib.tir_indirect_sample(v, None, v, v, v, 1, v, v, 1, 4, 0.5, v, v, v, v, v, v, v, 4, v, None) == -1
    assert lib.tir_indirect_hits_work_size(1, 4, None) == -1
    assert lib.tir_indirect_hits_work_size(1, 0, C.byref(cnt)) == -2
    Hh = lambda vk=0, K=4, pos=v, ab=aabb: lib.tir_indirect_hits(0, K, pos, v, v, v, v, v, vk, ab, v, v, v, v, 4,  # noqa: E731
                                                                 C.byref(cnt), None, 0, None)
    assert Hh() == 0 and Hh(vk=2) == -3 and Hh(K=2000) == -2 and Hh(pos=None) == -1 and Hh(ab=None) == -1
    R = lambda L=1, S2=4, vk=0, row0=0, Lo=v: lib.tir_indirect_radiance(envs, L, v, v, v, v, 1, v, 1, S2, v, v, v, v,  # noqa: E731
                                                                        vk, Lo, 1, row0, None)
    assert R(S2=0) == -2 and R(S2=1025) == -2 and R(vk=5) == -3 and R(row0=1) == -2 and R(Lo=None) == -1
    assert R(L=_lib.RELIGHT_MAX_LIGHTS + 1) == -2
    Sh = lambda L=1, K=4, vk=0, row0=0, T=v: lib.tir_indirect_shade(envs, L, v, v, v, v, 1, v, v, 1, 4, 0.5, v, v,  # noqa: E731
                                                                    v, v, vk, K, T, v, v, v, 1, v, v, None, 1, row0,
                                                                    None)
    assert Sh(K=0) == -2 and Sh(K=1025) == -2 and Sh(vk=2) == -3 and Sh(row0=1) == -2 and Sh(T=None) == -1
    assert Sh(L=_lib.RELIGHT_MAX_LIGHTS + 1) == -2


def test_header_documents_the_estimator():
    hdr = open(os.path.join(REPO, "include", "tensoir_b200.h")).read()
    body = open(os.path.join(REPO, "tensoir_b200", "csrc", "tir_indirect_body.h")).read()
    line = "linear[l,i] = (1/S)  * sum_s direct_s"
    assert line in hdr and line in body and "(1/K)  * sum_k T[i,k] * w[i,k] * Lo[l, h(i,k)]" in hdr


# ---- 5. plumbing ------------------------------------------------------------------------------------------------------

class FakeModel:
    device = torch.device("cpu")

    def __call__(self, rays, light_idx, **kw):
        n = rays.shape[0]
        g = torch.Generator().manual_seed(n)
        acc = (torch.arange(n) % 3 != 0).float()
        return (torch.rand(n, 3, generator=g), torch.full((n,), 3.0), torch.tensor([[0.0, 0.0, 1.0]]).expand(n, 3),
                torch.full((n, 3), 0.5), torch.full((n, 1), 0.4), torch.full((n, 3), 0.04), acc)


@pytest.mark.parametrize("K", [0, 3])
def test_relight_takes_the_indirect_path_only_when_asked(tmp_path, monkeypatch, K):
    from types import SimpleNamespace

    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    names = ["a", "b"]
    H = W = 12
    ds = SyntheticViews(hemisphere_poses(1), H, W, light_names=names)
    calls = {"fused": 0, "indirect": 0}

    def fused(tensoIR, envir_light, light_names, rays, maps, rescale_value, u, num_samples, thr, vis, out, row0,
              tables):
        calls["fused"] += 1
        out[0][:, row0:row0 + rays.shape[0]] = 0.5
        out[1][:, row0:row0 + rays.shape[0]] = 0.25

    def ind(tensoIR, envir_light, light_names, rays, maps, rescale_value, u, gen, *, indirect_samples,
            indirect_light_samples, acc_mask_threshold, vis_equation, out, row0, tables, indirect_out):
        calls["indirect"] += 1
        assert indirect_samples == K and indirect_light_samples == 8
        assert gen.initial_seed() == 77
        out[0][:, row0:row0 + rays.shape[0]] = 0.5
        out[1][:, row0:row0 + rays.shape[0]] = 0.25
        indirect_out[:, row0:row0 + rays.shape[0]] = 0.125

    monkeypatch.setattr(relighting, "relight_chunk_fused", fused)
    monkeypatch.setattr(indirect, "relight_chunk_indirect", ind)
    monkeypatch.setattr(relighting, "env_tables", lambda env, n: (None, []))
    monkeypatch.setattr(relighting, "pair_metrics",
                        lambda a, b, H, W: torch.tensor([[1.0, 0.5]] * a.shape[0], dtype=torch.float64))
    monkeypatch.setattr(torch, "Generator", _cpu_generator(torch.Generator))
    hdr = {k: np.ones((4, 8, 3), np.float32) for k in names}
    args = SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(tmp_path), batch_size=50, indirect_samples=K,
                           indirect_light_samples=8, indirect_seed=77, save_indirect=1, render_video=False,
                           if_render_normal=False, if_save_albedo=False)
    relighting.relight(ds, args, FakeModel(), rescale_value=[1.0, 1.0, 1.0])
    chunks = -(-H * W // 50)
    assert calls == ({"fused": chunks, "indirect": 0} if K == 0 else {"fused": 0, "indirect": chunks})
    view = tmp_path / "test_000"
    assert (view / "relighting_with_bg" / "a.png").exists()
    assert ((view / "relighting_indirect").exists()) == (K > 0)
    if K:
        from tensoir_b200.relight import read_hdr
        img = read_hdr(str(view / "relighting_indirect" / "b.hdr"))
        assert img.shape == (H, W, 3) and np.allclose(img, 0.125)
    txt = (view / "relighting_without_bg" / "relight_psnr.txt").read_text().splitlines()
    assert [t.split(":")[0] for t in txt] == names and all("PNSR" in t and "SSIM" in t for t in txt)


def _cpu_generator(cls):
    """torch.Generator pinned to the CPU: relight() asks for one on its model's device."""
    return lambda device=None: cls()


def test_relight_importance_parses_indirect_flags():
    sys.path.insert(0, os.path.join(REPO, "tools"))
    import relight_importance as tool
    import relight_lights
    assert tool.pop_option is relight_lights.pop_option
    argv = ["x", "--config", "c", "--indirect_samples", "16", "--save_indirect", "1", "--ckpt", "k"]
    assert tool.indirect_options(argv) == dict(indirect_samples=16, indirect_light_samples=32, save_indirect=True)
    assert argv == ["x", "--config", "c", "--ckpt", "k"]
    argv = ["x", "--indirect_light_samples", "8"]
    assert tool.indirect_options(argv) == dict(indirect_samples=0, indirect_light_samples=8, save_indirect=False)
    with pytest.raises(SystemExit):
        tool.indirect_options(["x", "--indirect_samples", "many"])
