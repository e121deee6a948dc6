"""Relighting with multiple importance sampling, on the CPU.

The MIS entry points are built for the host (tests/host_mis.cpp: the same C ABI, argument checks and per-sample math of
csrc/tir_mis_body.h, loops instead of kernels), together with the environment-map pass (tests/host_relight.cpp), and
driven through the real ctypes wrappers in tensoir_b200.mis, with the march replaced by a fake.  Each stage is compared
with a float64 restatement of the header's definitions; the densities are checked for normalisation by quadrature, and
the estimator for unbiasedness against a float64 quadrature of the piecewise-constant integral."""
import ctypes as C
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import test_indirect_cpu as H
from helpers import build_host_lib, use_host
from tensoir_b200 import _lib, mis, relighting
from tensoir_b200.relight import Environment_Light

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
EPS = H.EPS
f32 = np.float32


def empty_march(model, rays_o, rays_d, *, table=None, counters=None, **kw):
    """An empty scene: every shadow ray is unoccluded (t_last 1, acc 0), so V = 1."""
    m = rays_o.shape[0]
    return torch.ones(m), torch.zeros(m), torch.zeros(m)


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    lib = build_host_lib(tmp_path_factory.mktemp("host_mis"), "host_relight.cpp", "host_mis.cpp")
    lib.host_mis_texel.argtypes = [C.POINTER(_lib.TirEnvMap), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.host_mis_pdf_brdf.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                      C.c_void_p]
    return lib


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so, H.plane_march())
    return host_so


def p(t):
    return C.c_void_p(t.data_ptr())


# ---- float64 restatements ---------------------------------------------------------------------------------------------

def texel64(d, Hh, W):
    """rl_texel in float64 -> (bin, fractional row, fractional column) before the floor."""
    d = d.double()
    z = (d[:, 2] / d.norm(dim=-1)).clamp(-1, 1)
    fr = torch.acos(z) * Hh / math.pi
    fc = (math.pi - torch.atan2(d[:, 1], d[:, 0])) * W / (2 * math.pi)
    r = fr.floor().clamp(0, Hh - 1).long()
    c = fc.floor().clamp(0, W - 1).long()
    return r * W + c, fr, fc


def solid_angle64(Hh, W, r):
    return 2 * math.pi / W * (torch.cos(r * math.pi / Hh) - torch.cos((r + 1) * math.pi / Hh))


def pdf_light64(env, name, b):
    cdf = env._cdf[name].double()
    P = cdf[b] - torch.where(b > 0, cdf[(b - 1).clamp(min=0)], torch.zeros_like(cdf[b]))
    Hh, W = env.hdr_rgbs[name].shape[:2]
    return P / solid_angle64(Hh, W, (b // W).double())


def point32(rays, normal):
    """Np and V of tir::ggx_point, in float32 with ggx_point's order of operations (the host build's bits)."""
    n = normal.numpy().astype(f32)
    V = (-rays[:, 3:]).numpy().astype(f32)
    nn = np.zeros(n.shape[0], f32)
    vn = np.zeros(n.shape[0], f32)
    for d in range(3):
        nn = nn + n[:, d] * n[:, d]
        vn = vn + V[:, d] * V[:, d]
    inv_nn = f32(1) / np.maximum(np.sqrt(nn), f32(1e-12))
    inv_vn = f32(1) / np.maximum(np.sqrt(vn), f32(1e-12))
    nov = np.zeros(n.shape[0], f32)
    for d in range(3):
        V[:, d] = V[:, d] * inv_vn
        nov = nov + V[:, d] * n[:, d] * inv_nn
    sgn = np.sign(nov).astype(f32)
    Np = (n * inv_nn[:, None]) * sgn[:, None]
    return torch.from_numpy(Np), torch.from_numpy(V)


def frame32(w):
    """lt_frame in float32, operation by operation."""
    w = w.numpy().astype(f32)
    s = np.where(w[:, 2] >= 0, f32(1), f32(-1)).astype(f32)
    s = np.copysign(f32(1), w[:, 2]).astype(f32)
    a = f32(-1) / (s + w[:, 2])
    b = (w[:, 0] * w[:, 1]) * a
    t1 = np.stack([f32(1) + (s * (w[:, 0] * w[:, 0])) * a, s * b, -s * w[:, 0]], -1)
    t2 = np.stack([b, s + (w[:, 1] * w[:, 1]) * a, -w[:, 1]], -1)
    return torch.from_numpy(t1.astype(f32)), torch.from_numpy(t2.astype(f32))


def alpha64(rough):
    r = rough.double().mean(-1) if rough.shape[1] == 3 else rough.double()[:, 0]
    return r * r


def brdf_dirs64(rays, normal, rough, u):
    """The BRDF strategy's directions [n,K,3] in float64 from the host build's float32 Np, V and frame."""
    Np, V = point32(rays, normal)
    t1, t2 = frame32(Np)
    Np, V, t1, t2 = (t.double()[:, None] for t in (Np, V, t1, t2))
    a = alpha64(rough)[:, None, None]
    dot = lambda x, y: (x * y).sum(-1, keepdim=True)  # noqa: E731
    vl = torch.cat([dot(V, t1), dot(V, t2), dot(V, Np)], -1).expand(-1, u.shape[1], -1)
    vh = torch.cat([a * vl[..., :2], vl[..., 2:]], -1)
    vh = vh / vh.norm(dim=-1, keepdim=True)
    lensq = (vh[..., :2] ** 2).sum(-1, keepdim=True)
    il = torch.where(lensq > 0, lensq.rsqrt(), 0.0)
    T1 = torch.where(lensq > 0, torch.cat([-vh[..., 1:2] * il, vh[..., 0:1] * il, torch.zeros_like(il)], -1),
                     torch.tensor([1.0, 0.0, 0.0], dtype=torch.float64))
    T2 = torch.linalg.cross(vh, T1)
    rr = u[..., 1:2].sqrt()
    p1 = rr * torch.cos(2 * math.pi * u[..., 2:3])
    s = 0.5 * (1 + vh[..., 2:3])
    p2 = (1 - s) * (1 - p1 * p1).clamp(min=0).sqrt() + s * rr * torch.sin(2 * math.pi * u[..., 2:3])
    p3 = (1 - p1 * p1 - p2 * p2).clamp(min=0).sqrt()
    nh = p1 * T1 + p2 * T2 + p3 * vh
    ne = torch.cat([a * nh[..., :2], nh[..., 2:].clamp(min=0)], -1)
    ne = ne / ne.norm(dim=-1, keepdim=True)
    h = ne[..., 0:1] * t1 + ne[..., 1:2] * t2 + ne[..., 2:3] * Np
    vndf = 2 * dot(V, h) * h - V
    x, y = H.disc64(u[..., 1:])
    x, y = x.float().double()[..., None], y.float().double()[..., None]        # lt_disc rounds once to fp32
    cosd = x * t1 + y * t2 + (1 - x * x - y * y).clamp(min=0).sqrt() * Np
    return torch.where(u[..., :1] < 0.5, vndf, cosd)


def pdf_brdf64(rays, normal, rough, w):
    """p_brdf [n,K] of directions w [n,K,3] in float64 from the host build's float32 Np and V."""
    Np, V = point32(rays, normal)
    Np, V = Np.double()[:, None], V.double()[:, None]
    a2 = (alpha64(rough) ** 2)[:, None]
    L = w.double() / w.double().norm(dim=-1, keepdim=True)
    h = L + V
    hn = h.norm(dim=-1)
    noh = (Np * h).sum(-1) / hn
    nov = (Np * V).sum(-1).clamp(min=0)
    D = torch.where(noh > 0, a2 / (math.pi * (1 - noh * noh * (1 - a2)) ** 2), 0.0)
    vndf = D / (2 * (nov + (a2 + (1 - a2) * nov * nov).sqrt()))
    return 0.5 * vndf + 0.5 * (Np * L).sum(-1).clamp(min=0) / math.pi


def cos32(w, normal):
    """rl_cosine in float32: ((L0 n0 + L1 n1) + L2 n2), each rounded."""
    w, n = w.numpy().astype(f32), normal.numpy().astype(f32)[:, None]
    return torch.from_numpy((w[..., 0] * n[..., 0] + w[..., 1] * n[..., 1]) + w[..., 2] * n[..., 2])


def env_maps(names, Hh=8, W=16, seed=0):
    g = np.random.default_rng(seed)
    return Environment_Light({k: g.uniform(0.05, 2.0, (Hh, W, 3)).astype(np.float32) for k in names}, device="cpu")


def run_sample(env, names, ch, S_l, S_b, seed):
    L, n = len(names), ch["rays"].shape[0]
    g = torch.Generator().manual_seed(seed)
    u_l = torch.rand(L, n, S_l, 3, generator=g, dtype=torch.float64)
    u_b = torch.rand(n, S_b, 3, generator=g, dtype=torch.float64)
    envs, keep = relighting.env_tables(env, names)
    rays, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(
        ch["rays"], (ch["depth"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"]))
    dirs, pos, vis = mis.mis_visibility(H.Model(), envs, L, rays, depth, normal, albedo, rough, fresnel, acc, u_l,
                                        u_b, 0.5, 'nerv')
    return u_l, u_b, dirs, pos, vis


# ---- 1. texel lookup and texel density --------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(8, 16), (17, 31), (256, 512)])
def test_texel_lookup_matches_float64(host_lib, shape):
    host_so = host_lib
    Hh, W = shape
    names = ["a"]
    env = env_maps(names, Hh, W, seed=Hh)
    envs, keep = relighting.env_tables(env, names)
    g = torch.Generator().manual_seed(W)
    rnd = torch.nn.functional.normalize(torch.randn(20000, 3, generator=g, dtype=torch.float64), dim=-1)
    # directions on texel edges (fp64 edge, rounded to fp32), texel centres, both poles and the atan2 seam
    th = torch.arange(Hh + 1, dtype=torch.float64) * math.pi / Hh
    ph = math.pi - torch.arange(W + 1, dtype=torch.float64) * 2 * math.pi / W
    th, ph = torch.meshgrid(torch.cat([th, th[:-1] + math.pi / (2 * Hh)]), torch.cat([ph, ph[:-1] - math.pi / W]),
                            indexing="ij")
    edge = torch.stack([th.sin() * ph.cos(), th.sin() * ph.sin(), th.cos()], -1).reshape(-1, 3)
    special = torch.tensor([[0, 0, 1], [0, 0, -1], [1e-8, 0, 1], [0, 1e-8, -1], [-1, 0, 0], [-1, -0.0, 0],
                            [-1, 1e-8, 0], [-1, -1e-8, 0], [1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 2.5]],
                           dtype=torch.float64)
    d = torch.cat([rnd, edge, special]).float().contiguous()
    n = d.shape[0]
    bins = torch.empty(n, dtype=torch.int32)
    pl = torch.empty(n, dtype=torch.float64)
    assert host_so.host_mis_texel(envs, p(d), n, p(bins), p(pl)) == 0
    b64, fr, fc = texel64(d, Hh, W)
    # fp32 acos / atan2 of the rounded direction: a few ulp of the angle, divided by sin(theta) near the poles for acos
    sin_t = (1 - (d.double()[:, 2] / d.double().norm(dim=-1)) ** 2).clamp(min=0).sqrt()
    tol_r = 16 * EPS * Hh / math.pi * (math.pi + 1 / sin_t.clamp(min=1e-30))
    tol_c = 16 * EPS * W
    near = ((fr - fr.round()).abs() <= tol_r) | ((fc - fc.round()).abs() <= tol_c) | ((fc - W).abs() <= tol_c)
    same = bins.long() == b64
    assert same[~near].all()
    assert same[near].any() and near.sum() > 100
    r32, c32, r64, c64 = bins.long() // W, bins.long() % W, b64 // W, b64 % W
    dc = (c32 - c64).abs()
    assert ((r32 - r64).abs() <= 1).all() and ((dc <= 1) | (dc == W - 1)).all()
    # poles and the seam
    assert bins[-12].item() // W == 0 and bins[-11].item() // W == Hh - 1
    assert bins[-8].item() % W == 0 and bins[-7].item() % W == W - 1
    # p_light = P_b / dOmega_b of the returned texel, fp64 throughout
    want = pdf_light64(env, "a", bins.long())
    assert torch.allclose(pl, want, rtol=1e-9, atol=0)


def test_pdf_light_integrates_to_one(host_lib):
    host_so = host_lib
    for (Hh, W), seed in (((8, 16), 1), ((32, 64), 2)):
        env = env_maps(["a"], Hh, W, seed)
        img = env.hdr_rgbs["a"].numpy().copy()
        img[Hh // 2] = 0.0                       # a row without light: p_light = 0 there
        env = Environment_Light({"a": img}, device="cpu")
        envs, keep = relighting.env_tables(env, ["a"])
        nz, nph = 1024, 2048                     # equal-area quadrature: midpoints in (z, azimuth)
        z = 1 - (torch.arange(nz, dtype=torch.float64) + 0.5) * 2 / nz
        ph = (torch.arange(nph, dtype=torch.float64) + 0.5) * 2 * math.pi / nph - math.pi
        z, ph = torch.meshgrid(z, ph, indexing="ij")
        s = (1 - z * z).sqrt()
        d = torch.stack([s * ph.cos(), s * ph.sin(), z], -1).reshape(-1, 3).float().contiguous()
        pl = torch.empty(d.shape[0], dtype=torch.float64)
        bins = torch.empty(d.shape[0], dtype=torch.int32)
        assert host_so.host_mis_texel(envs, p(d), d.shape[0], p(bins), p(pl)) == 0
        total = float(pl.sum()) * 4 * math.pi / d.shape[0]
        assert abs(total - 1) < 1e-3, total
        assert not pl[(bins.long() // W) == Hh // 2].any()


# ---- 2. sampling ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("stride", [1, 3])
def test_sample_matches_float64(host_lib, stride):
    names = ["a", "b"]
    env = env_maps(names, 17, 31, seed=3)
    n, S_l, S_b = 400, 24, 16
    ch = H.random_chunk(5 + stride, n, stride)
    u_l, u_b, dirs, pos, vis = run_sample(env, names, ch, S_l, S_b, seed=stride)
    hit = ch["acc"] > 0.5
    nl = 2 * n * S_l
    dl, db = dirs[:nl].reshape(2, n, S_l, 3), dirs[nl:].reshape(n, S_b, 3)
    pl, pb = pos[:nl].reshape(2, n, S_l), pos[nl:].reshape(n, S_b)
    # light strategy: texel by searchsorted, a point uniform in its solid angle, in fp64 rounded once
    for k, name in enumerate(names):
        Hh, W = env.hdr_rgbs[name].shape[:2]
        cdf = env._cdf[name].double()
        b = torch.searchsorted(cdf, u_l[k, ..., 0].contiguous(), right=True).clamp(max=Hh * W - 1)
        r, c = (b // W).double(), (b % W).double()
        zt, zb = torch.cos(r * math.pi / Hh), torch.cos((r + 1) * math.pi / Hh)
        z = zt + u_l[k, ..., 1] * (zb - zt)
        ph = math.pi - (c + u_l[k, ..., 2]) * 2 * math.pi / W
        s = (1 - z * z).clamp(min=0).sqrt()
        w64 = torch.stack([s * ph.cos(), s * ph.sin(), z], -1)
        err = (dl[k].double() - w64).abs()[hit]
        assert (err <= EPS * w64.abs()[hit] + 1e-12).all(), float(err.max())
        assert not dl[k][~hit].any()
        # the drawn point lies in its texel (up to the lookup's edge tolerance)
        got, fr, fc = texel64(dl[k][hit].reshape(-1, 3), Hh, W)
        inside = got == b[hit].reshape(-1)
        assert inside.float().mean() > 0.999
    # BRDF strategy: VNDF or cosine from the float32 frame, in fp64 rounded once
    w64 = brdf_dirs64(ch["rays"], ch["normal"], ch["rough"], u_b)
    err = (db.double() - w64).abs()[hit]
    assert (err <= 4 * EPS * w64.abs()[hit].clamp(min=1e-3)).all(), float(err.max())
    assert not db[~hit].any()
    # the cosine test in fp32 decides which slots were marched; rows in slot order in the host build
    cl = torch.stack([cos32(dl[k], ch["normal"]) for k in range(2)])
    assert torch.equal(pl >= 0, (cl > 1e-6) & hit[None, :, None])
    assert torch.equal(pb >= 0, (cos32(db, ch["normal"]) > 1e-6) & hit[:, None])
    m = pos >= 0
    assert torch.equal(pos[m], torch.arange(int(m.sum()), dtype=torch.int32))
    # about half the BRDF slots of a hit ray took the GGX lobe, and more of those than cosine slots face the normal
    assert 0.4 < float((u_b[hit][..., 0] < 0.5).double().mean()) < 0.6


def test_pdf_brdf_matches_float64(host_so):
    n, K = 300, 64
    ch = H.random_chunk(9, n, 3)
    g = torch.Generator().manual_seed(4)
    w = torch.nn.functional.normalize(torch.randn(n, K, 3, generator=g), dim=-1).contiguous()
    # half the directions near the mirror direction, where D peaks
    V = torch.nn.functional.normalize(-ch["rays"][:, 3:], dim=-1)
    nh = torch.nn.functional.normalize(ch["normal"], dim=-1)
    R = 2 * (V * nh).sum(-1, keepdim=True) * nh - V
    w[:, ::2] = torch.nn.functional.normalize(R[:, None] + 0.02 * w[:, ::2], dim=-1)
    out = torch.empty(n, K, dtype=torch.float64)
    assert host_so.host_mis_pdf_brdf(p(ch["rays"]), p(ch["normal"]), p(ch["rough"]), 3, n, p(w), K, p(out)) == 0
    want = pdf_brdf64(ch["rays"], ch["normal"], ch["rough"], w)
    assert torch.allclose(out, want, rtol=1e-9, atol=1e-300)
    assert (out >= 0).all() and (out > 0).float().mean() > 0.5 and float(out.max()) > 10


@pytest.mark.parametrize("rough", [0.09, 0.3, 0.99])
def test_pdf_brdf_integrates_to_one(host_so, rough):
    """p_brdf is a density on the whole sphere: quadrature in polar coordinates about the mirror direction, with
    log-spaced polar cells so that the narrowest lobe (alpha = 0.0081) spans hundreds of them, and azimuth cells fine
    enough for the lobe's compression across the plane of incidence at grazing views."""
    nb, nph = 1500, 2048
    edges = torch.cat([torch.zeros(1, dtype=torch.float64),
                       torch.logspace(math.log10(1e-7), math.log10(math.pi), nb, dtype=torch.float64)])
    beta = 0.5 * (edges[1:] + edges[:-1])
    dbeta = edges[1:] - edges[:-1]
    ph = (torch.arange(nph, dtype=torch.float64) + 0.5) * 2 * math.pi / nph
    for view_deg in (0.0, 40.0, 75.0, 88.0):
        t = math.radians(view_deg)
        rays = torch.tensor([[0.0, 0.0, 0.0, -math.sin(t), 0.0, -math.cos(t)]], dtype=torch.float32)
        normal = torch.tensor([[0.0, 0.0, 1.0]])
        V = -rays[0, 3:].double()
        R = 2 * V[2] * torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64) - V
        t1 = torch.linalg.cross(R, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64))
        t1 = t1 / t1.norm()
        t2 = torch.linalg.cross(R, t1)
        bb, pp = torch.meshgrid(beta, ph, indexing="ij")
        d = (bb.sin() * pp.cos())[..., None] * t1 + (bb.sin() * pp.sin())[..., None] * t2 + bb.cos()[..., None] * R
        dw = (dbeta[:, None] * bb.sin() * (2 * math.pi / nph)).reshape(-1)
        d = d.reshape(1, -1, 3).float().contiguous()
        out = torch.empty(1, d.shape[1], dtype=torch.float64)
        assert host_so.host_mis_pdf_brdf(p(rays), p(normal), p(torch.tensor([[rough]])), 1, 1, p(d), d.shape[1],
                                         p(out)) == 0
        total = float((out[0] * dw).sum())
        assert abs(total - 1) < 1e-3, (rough, view_deg, total)


# ---- 3. shading: per-sample contribution ------------------------------------------------------------------------------

def shade_ref(lib, env, names, k, ch, dirs, pos, vis, S_l, S_b, resc):
    """The linear estimate of map k in float64 from the sampler's own fp32 directions, slot map and visibility, and its
    bound: each term carries rl_contrib's fp32 error (the test_indirect_cpu derivation, with the denominator rounded
    once to fp32) and the sum a chain of S_l + S_b additions.  Texels and p_light come from the host lookup, which
    test_texel_lookup_matches_float64 checks.  -> (want, bound) [n, 3]."""
    name = names[k]
    n, L = ch["rays"].shape[0], len(names)
    nl = L * n * S_l
    envs, keep = relighting.env_tables(env, names)
    w = torch.cat([dirs[k * n * S_l:(k + 1) * n * S_l].reshape(n, S_l, 3), dirs[nl:].reshape(n, S_b, 3)], 1)
    q = torch.cat([pos[k * n * S_l:(k + 1) * n * S_l].reshape(n, S_l), pos[nl:].reshape(n, S_b)], 1)
    flat = w.reshape(-1, 3).contiguous()
    bins = torch.empty(flat.shape[0], dtype=torch.int32)
    pl = torch.empty(flat.shape[0], dtype=torch.float64)
    assert lib.host_mis_texel(relighting.env_group(envs, k), p(flat), C.c_int64(flat.shape[0]), p(bins), p(pl)) == 0
    pl = pl.reshape(n, -1)
    assert torch.allclose(pl, pdf_light64(env, name, bins.long()).reshape(n, -1), rtol=1e-9, atol=0)
    den = S_l * pl + (S_b * pdf_brdf64(ch["rays"], ch["normal"], ch["rough"], w) if S_b else 0)
    rgb = env.hdr_rgbs[name].reshape(-1, 3)[bins.long()].double().reshape(n, -1, 3)
    v = torch.where(q >= 0, vis.double()[q.long().clamp(min=0)], 0.0)
    B, cos, spec, nom0 = H.brdf64(ch["normal"], -ch["rays"][:, 3:], w, ch["albedo"] * resc, ch["rough"],
                                  ch["fresnel"])
    wgt = torch.where((q >= 0) & (den > 0), v * cos / den.clamp(min=1e-300), 0.0)[..., None] * rgb
    term = B * wgt
    bnd = EPS * (32 * term.abs() + 16 * (spec * wgt).abs() / nom0
                 + 8 * B * (v[..., None] * rgb / den.clamp(min=1e-300)[..., None])
                 * ch["normal"].double().norm(dim=-1)[:, None, None] * (q >= 0)[..., None])
    return term.sum(1), bnd.sum(1) + (S_l + S_b) * EPS * term.abs().sum(1)


@pytest.mark.parametrize("S_b", [0, 16])
def test_shade_matches_float64(host_lib, S_b):
    names = ["a", "b"]
    env = env_maps(names, 17, 31, seed=6)
    n, S_l = 300, 24
    ch = H.random_chunk(31 + S_b, n, 3)
    u_l, u_b, dirs, pos, vis = run_sample(env, names, ch, S_l, S_b, seed=7)
    resc = torch.tensor([1.1, 0.9, 1.0])
    lin = torch.zeros(2, n, 3)
    mis.relight_chunk_mis(H.Model(), env, names, ch["rays"],
                          (ch["depth"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"]), resc,
                          u_l, u_b, linear_out=lin)
    hit = ch["acc"] > 0.5
    for k, name in enumerate(names):
        want, bound = shade_ref(host_lib, env, names, k, ch, dirs, pos, vis, S_l, S_b, resc)
        got = lin[k].double()
        assert ((got - want).abs() <= bound + 1e-30)[hit].all(), float(((got - want).abs() / bound)[hit].max())
        assert not got[~hit].any() and (got[hit] > 0).all()


# ---- 4. unbiasedness --------------------------------------------------------------------------------------------------

def one_hit(n, view, normal, rough, albedo=(0.6, 0.5, 0.4)):
    """n copies of one surface hit at the origin seen along -view."""
    d = -torch.nn.functional.normalize(torch.tensor(view, dtype=torch.float64), dim=0)
    rays = torch.cat([-3 * d, d]).float()[None].expand(n, 6).contiguous()
    ch = dict(rays=rays, depth=torch.full((n,), 3.0), normal=torch.tensor([normal], dtype=torch.float32).expand(n, 3),
              albedo=torch.tensor([albedo]).expand(n, 3), rough=torch.full((n, 1), float(rough)),
              fresnel=torch.full((n, 3), 0.04), acc=torch.ones(n))
    return ch, tuple(ch[k].contiguous() for k in ("depth", "normal", "albedo", "rough", "fresnel", "acc"))


def texel_grid(Hh, W, sub, r, c):
    """Midpoints of a sub x sub equal-area grid of texel (r, c) -> directions [sub*sub, 3] and their solid angle."""
    zt, zb = math.cos(r * math.pi / Hh), math.cos((r + 1) * math.pi / Hh)
    z = zt + (torch.arange(sub, dtype=torch.float64) + 0.5) / sub * (zb - zt)
    ph = math.pi - (c + (torch.arange(sub, dtype=torch.float64) + 0.5) / sub) * 2 * math.pi / W
    z, ph = torch.meshgrid(z, ph, indexing="ij")
    s = (1 - z * z).sqrt()
    d = torch.stack([s * ph.cos(), s * ph.sin(), z], -1).reshape(-1, 3)
    return d, 2 * math.pi / W * (zt - zb) / (sub * sub)


def integrand64(ch, d):
    """f cos over directions d [K,3] for the hit of ``ch`` (V = 1), with the cosine cut -> [K, 3]."""
    B, cos, _, _ = H.brdf64(ch["normal"][:1], -ch["rays"][:1, 3:], d[None], ch["albedo"][:1], ch["rough"][:1],
                            ch["fresnel"][:1])
    return (B * torch.where(cos > 1e-6, cos, 0.0)[..., None])[0]


def quadrature(ch, rgb, sub):
    """float64 quadrature of the piecewise-constant integral: sum over texels of E_b * integral of f cos over the
    texel, each by the midpoint rule on a sub x sub equal-area grid."""
    Hh, W = rgb.shape[:2]
    total = torch.zeros(3, dtype=torch.float64)
    for r in range(Hh):
        for c in range(W):
            d, dw = texel_grid(Hh, W, sub, r, c)
            total += torch.from_numpy(rgb[r, c]).double() * integrand64(ch, d).sum(0) * dw
    return total


@pytest.mark.parametrize("rough", [0.2, 0.5, 0.99])
def test_estimator_is_unbiased(host_so, monkeypatch, rough):
    use_host(monkeypatch, host_so, empty_march)
    Hh, W = 8, 16
    view, normal = (0.5, -0.2, 0.8), (0.1, 0.05, 0.99)
    ch, maps = one_hit(1 << 16, view, normal, rough)
    # the bright texel holds the mirror direction of the view
    V = np.array(view) / np.linalg.norm(view)
    nn = np.array(normal) / np.linalg.norm(normal)
    Rm = 2 * V.dot(nn) * nn - V
    b, _, _ = texel64(torch.tensor([Rm]), Hh, W)
    bright = np.full((Hh, W, 3), 0.05, np.float32)
    bright.reshape(-1, 3)[int(b)] = (40.0, 30.0, 20.0)
    hdr = {"bright": bright, "furnace": np.ones((Hh, W, 3), np.float32)}
    names = list(hdr)
    env = Environment_Light(hdr, device="cpu")
    n, S_l, S_b = ch["rays"].shape[0], 12, 4
    g = torch.Generator().manual_seed(int(rough * 100))
    u_l = torch.rand(2, n, S_l, 3, generator=g, dtype=torch.float64)
    u_b = torch.rand(n, S_b, 3, generator=g, dtype=torch.float64)
    lin = torch.zeros(2, n, 3)
    mis.relight_chunk_mis(H.Model(), env, names, ch["rays"], maps, 1.0, u_l, u_b, linear_out=lin)
    sub = 192 if rough < 0.5 else 32
    for k, name in enumerate(names):
        q = quadrature(ch, hdr[name], sub)
        q2 = quadrature(ch, hdr[name], sub // 2)
        assert ((q - q2).abs() <= 1e-4 * q).all(), (name, q, q2)     # the sub-grid resolves the lobe
        est = lin[k].double()
        mean, se = est.mean(0), est.std(0) / math.sqrt(n)
        assert ((mean - q).abs() <= 5 * se + 1e-4 * q).all(), (name, rough, mean, q, se)
        if name == "furnace":
            assert (se < 0.02 * q).all()


def test_mis_agrees_with_the_default_within_the_texel_bound(host_so, monkeypatch):
    """A diffuse surface under a smooth 32x64 map: the MIS mean (continuous integral) and the default estimator's
    mean (texel centres, sin of the row centre) differ by at most the discretisation bound of DESIGN.md §3.7:
    sum_b E_b (dOmega_b osc_b(g) + |g(c_b)| |dOmega_b - dOmega'_b|), plus 5 standard errors."""
    use_host(monkeypatch, host_so, empty_march)
    Hh, W = 32, 64
    th = (torch.arange(Hh, dtype=torch.float64) + 0.5) / Hh * math.pi
    ph = (torch.arange(W, dtype=torch.float64) + 0.5) / W * 2 * math.pi
    th, ph = torch.meshgrid(th, ph, indexing="ij")
    smooth = (0.3 + 0.2 * th.cos() + 0.1 * (ph.sin() * th.sin()))
    rgb = torch.stack([smooth, 0.8 * smooth, 0.6 * smooth + 0.05], -1).float().numpy()
    env = Environment_Light({"s": rgb}, device="cpu")
    view, normal = (0.3, 0.2, 0.9), (0.0, 0.1, 0.99)
    n = 1 << 15
    ch, maps = one_hit(n, view, normal, 0.99, albedo=(0.5, 0.5, 0.5))
    g = torch.Generator().manual_seed(11)
    u_l = torch.rand(1, n, 96, 3, generator=g, dtype=torch.float64)
    u_b = torch.rand(n, 32, 3, generator=g, dtype=torch.float64)
    lin = torch.zeros(1, n, 3)
    mis.relight_chunk_mis(H.Model(), env, ["s"], ch["rays"], maps, 1.0, u_l, u_b, linear_out=lin)
    u = torch.rand(1, n, 128, generator=g, dtype=torch.float64)
    _, wo = relighting.relight_chunk_fused(H.Model(), env, ["s"], ch["rays"], maps, 1.0, u, 128)
    wo = wo[0].double()
    assert (wo > 0.05).all() and (wo < 0.95).all()        # inside the sRGB curve's power branch, below the clamp
    d_lin = ((wo + 0.055) / 1.055) ** 2.4 - 1e-6           # the tone map, inverted
    m_mis, se_mis = lin[0].double().mean(0), lin[0].double().std(0) / math.sqrt(n)
    m_def, se_def = d_lin.mean(0), d_lin.std(0) / math.sqrt(n)
    # the bound, with g = f cos evaluated at each texel's centre and on a 9 x 9 grid of its points (edges included)
    bound = torch.zeros(3, dtype=torch.float64)
    dirs = env.hdr_dir["s"].reshape(-1, 3).double()
    gc = integrand64(ch, dirs)
    k = 9
    for r in range(Hh):
        zt, zb = math.cos(r * math.pi / Hh), math.cos((r + 1) * math.pi / Hh)
        dom = 2 * math.pi / W * (zt - zb)
        dom_ref = 2 * math.pi ** 2 * math.sin((r + 0.5) * math.pi / Hh) / (Hh * W)
        for c in range(W):
            z = zt + torch.linspace(0, 1, k, dtype=torch.float64) * (zb - zt)
            a = math.pi - (c + torch.linspace(0, 1, k, dtype=torch.float64)) * 2 * math.pi / W
            z, a = torch.meshgrid(z, a, indexing="ij")
            s = (1 - z * z).sqrt()
            gv = integrand64(ch, torch.stack([s * a.cos(), s * a.sin(), z], -1).reshape(-1, 3))
            osc = gv.max(0).values - gv.min(0).values
            E = torch.from_numpy(rgb[r, c]).double()
            bound += E * (dom * osc + gc[r * W + c].abs() * abs(dom - dom_ref))
    diff = (m_mis - m_def).abs()
    assert (diff <= bound + 5 * (se_mis ** 2 + se_def ** 2).sqrt()).all(), (diff, bound)
    assert (bound < 0.2 * m_mis).all()                     # the bound says something


# ---- 5. more maps than one call takes, determinism ----------------------------------------------------------------------

def test_groups_of_maps_and_determinism(host_lib):
    G = _lib.RELIGHT_MAX_LIGHTS
    names = [f"m{k}" for k in range(G + 2)]
    env = env_maps(names, 4, 8, seed=8)
    ch, maps = H.chunk(30, 40)
    g = torch.Generator().manual_seed(3)
    u_l = torch.rand(len(names), 40, 16, 3, generator=g, dtype=torch.float64)
    u_b = torch.rand(40, 8, 3, generator=g, dtype=torch.float64)
    lin = torch.zeros(len(names), 40, 3)
    a = mis.relight_chunk_mis(H.Model(), env, names, ch["rays"], maps, 1.0, u_l, u_b, linear_out=lin)
    b = mis.relight_chunk_mis(H.Model(), env, names, ch["rays"], maps, 1.0, u_l, u_b)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and a[0].shape == (G + 2, 40, 3)
    # each map's rows are those of a call with that map alone
    one = torch.zeros(1, 40, 3)
    k = G + 1
    c = mis.relight_chunk_mis(H.Model(), env, [names[k]], ch["rays"], maps, 1.0, u_l[k:k + 1], u_b, linear_out=one)
    assert torch.equal(c[1][0], a[1][k]) and torch.equal(one[0], lin[k])
    hit = ch["acc"] > 0.5
    assert torch.equal(a[1][:, ~hit], torch.ones_like(a[1][:, ~hit])) and not lin[:, ~hit].any()


# ---- 6. arguments -----------------------------------------------------------------------------------------------------

def test_mis_arguments(host_so):
    lib = host_so
    v = C.c_void_p(8)
    envs = (_lib.TirEnvMap * 1)()
    envs[0].H, envs[0].W = 2, 2
    envs[0].rgb = envs[0].dir = envs[0].pdf_return = envs[0].cdf = 8
    cnt = C.c_int64(0)

    def S(L=1, n=1, S_l=4, S_b=2, rs=1, cap=4, u_b=v, e=envs, rays=v, dr=v, lo=v):
        return lib.tir_relight_mis_sample(e, L, rays, v, v, v, v, rs, v, v, n, S_l, S_b, 0.5, v, u_b, dr, v, lo, v,
                                          cap, C.byref(cnt), None)
    assert S(S_l=0) == -2 and S(S_b=-1) == -2 and S(rs=2) == -2 and S(cap=-1) == -2 and S(cap=1 << 31) == -2
    assert S(L=_lib.RELIGHT_MAX_LIGHTS + 1) == -2 and S(n=-1) == -2
    assert S(e=None) == -1 and S(rays=None) == -1 and S(dr=None) == -1 and S(u_b=None) == -1 and S(lo=None) == -1
    assert S(n=0) == 0 and S(L=0) == 0

    def Sh(L=1, n=1, S_l=4, S_b=2, rs=1, vk=0, rows=1, row0=0, dr=v, vis=v, wb=v):
        return lib.tir_relight_mis_shade(envs, L, v, v, v, v, rs, v, v, n, S_l, S_b, 0.5, v, dr, v, vis, vk, wb, v,
                                         None, rows, row0, None)
    assert Sh(S_l=0) == -2 and Sh(S_b=-1) == -2 and Sh(rs=0) == -2 and Sh(vk=2) == -3 and Sh(row0=1) == -2
    assert Sh(rows=0) == -2 and Sh(row0=-1) == -2 and Sh(L=_lib.RELIGHT_MAX_LIGHTS + 1) == -2
    assert Sh(dr=None) == -1 and Sh(vis=None) == -1 and Sh(wb=None) == -1
    assert Sh(n=0, rows=0) == 0


def test_header_documents_the_estimator():
    hdr = open(os.path.join(REPO, "include", "tensoir_b200.h")).read()
    body = open(os.path.join(REPO, "tensoir_b200", "csrc", "tir_mis_body.h")).read()
    line = "f(w) * V(w) * E_l(w) * cos(w) / (S_l * p_light_l(w) + S_b * p_brdf(w))"
    assert line in hdr and line in body


# ---- 7. plumbing ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bad", [dict(sampling="brdf"), dict(sampling="mis", brdf_samples=512),
                                 dict(sampling="mis", brdf_samples=-1), dict(brdf_samples=1.5),
                                 dict(sampling="mis", indirect_samples=4)])
def test_relight_rejects_bad_options_before_any_work(bad):
    args = SimpleNamespace(**bad)                # no ckpt, dataset or hdrdir: the check comes first
    with pytest.raises(ValueError):
        relighting.relight(None, args)


@pytest.mark.parametrize("sampling", ["light", "mis"])
def test_relight_takes_the_mis_path_only_when_asked(tmp_path, monkeypatch, sampling):
    from tensoir_b200 import indirect
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    names = ["a", "b"]
    Hh = W = 12
    ds = SyntheticViews(hemisphere_poses(1), Hh, W, light_names=names)
    calls = {"fused": 0, "mis": 0}

    def fused(tensoIR, envir_light, light_names, rays, maps, rescale_value, u, num_samples, thr, vis, out, row0,
              tables):
        calls["fused"] += 1
        out[1][:, row0:row0 + rays.shape[0]] = 0.25

    def with_mis(tensoIR, envir_light, light_names, rays, maps, rescale_value, u_light, u_brdf, *, acc_mask_threshold,
                 vis_equation, out, row0, tables):
        calls["mis"] += 1
        n = rays.shape[0]
        assert u_light.shape == (2, n, relighting.NUM_SAMPLES - 100, 3) and u_brdf.shape == (n, 100, 3)
        assert u_light.dtype == u_brdf.dtype == torch.float64
        out[0][:, row0:row0 + n] = 0.5
        out[1][:, row0:row0 + n] = 0.25

    monkeypatch.setattr(relighting, "relight_chunk_fused", fused)
    monkeypatch.setattr(mis, "relight_chunk_mis", with_mis)
    monkeypatch.setattr(indirect, "relight_chunk_indirect", None)
    monkeypatch.setattr(relighting, "env_tables", lambda env, n: (None, []))
    monkeypatch.setattr(relighting, "pair_metrics",
                        lambda a, b, H, W: torch.tensor([[1.0, 0.5]] * a.shape[0], dtype=torch.float64))
    hdr = {k: np.ones((4, 8, 3), np.float32) for k in names}
    args = SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(tmp_path), batch_size=50, sampling=sampling,
                           brdf_samples=100, render_video=False, if_render_normal=False, if_save_albedo=False)
    relighting.relight(ds, args, H.FakeModel(), rescale_value=[1.0, 1.0, 1.0])
    chunks = -(-Hh * W // 50)
    assert calls == ({"fused": chunks, "mis": 0} if sampling == "light" else {"fused": 0, "mis": chunks})
    view = tmp_path / "test_000"
    assert (view / "relighting_with_bg" / "a.png").exists()
    txt = (view / "relighting_without_bg" / "relight_psnr.txt").read_text().splitlines()
    assert [t.split(":")[0] for t in txt] == names


def test_relight_importance_parses_sampling_flags():
    sys.path.insert(0, os.path.join(REPO, "tools"))
    import relight_importance as tool
    argv = ["x", "--config", "c", "--sampling", "mis", "--brdf_samples", "64", "--ckpt", "k"]
    assert tool.sampling_options(argv) == dict(sampling="mis", brdf_samples=64)
    assert argv == ["x", "--config", "c", "--ckpt", "k"]
    assert tool.sampling_options(["x"]) == dict(sampling="light", brdf_samples=128)
    with pytest.raises(SystemExit):
        tool.sampling_options(["x", "--brdf_samples", "many"])
