"""Fitting environment maps to photographs, on the CPU.

tir_transport_sample and tir_transport_build are built for the host (tests/host_transport.cpp: the same C ABI,
argument checks and per-(hit, texel) math of csrc/tir_transport_body.h, loops instead of kernels) and driven through
the real ctypes wrapper tensoir_b200.light_fit.  They are compared with a restatement of the definitions in
include/tensoir_b200.h: the cosine test in fp32 with the kernels' operation order (so membership is exact), the
transport in float64 with relight_utils.GGX_specular and a derived fp32 bound.  The solver is compared with
scipy.optimize.lsq_linear on the same regularised problem."""
import ctypes as C
import importlib.util
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from tensoir_b200 import _lib, light_fit as LF
from tensoir_b200.relight_utils import GGX_specular
from test_lighting_cpu import random_chunk

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
EPS = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_transport"), "host_transport.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


# ---- 1. the host build against the definitions ------------------------------------------------------------------------

def run_transport(ch, grid, vis_kind, rescale, seed=0):
    """transport_sample + a seeded random visibility list + transport_build through whatever _lib.load() gives."""
    pos, list_o, list_d = LF.transport_sample(grid, ch["rays"], ch["depth"], ch["normal"], ch["acc"], 0.5)
    vis = torch.rand(max(list_o.shape[0], 1), generator=torch.Generator().manual_seed(seed)).to(ch["rays"].device)
    T = LF.transport_build(grid, ch["rays"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"], 0.5,
                           rescale, pos, vis, 'nerfactor' if vis_kind else 'nerv')
    return dict(pos=pos, list_o=list_o, list_d=list_d, vis=vis, T=T)


def expected_joins(ch, dirs, thr=0.5):
    """The cosine test of the header in fp32 with rl_cosine's order ((x + y) + z, no fused multiply-add)."""
    d, nrm = dirs.numpy(), ch["normal"].numpy()
    cos = (d[None, :, 0] * nrm[:, None, 0] + d[None, :, 1] * nrm[:, None, 1]).astype(np.float32) \
        + (d[None, :, 2] * nrm[:, None, 2])
    assert cos.dtype == np.float32
    return torch.from_numpy((cos > np.float32(1e-6)) & (ch["acc"].numpy() > thr)[:, None])


def transport64(ch, grid, res, vis_kind, rescale, thr=0.5):
    """T [3, n, K] in float64 from the header's definition with the visibility the build's pos selects, and the bound
    on |T32 - T64|.

    Bound.  T = (a/pi + S) v c w with S = frac/nom the GGX term, v the visibility, c = L.n the raw cosine and w the
    solid angle, as in test_lighting_cpu.reference64 with the falloff replaced by w: every factor is a chain of at most
    ~30 rounded fp32 operations, each adding a relative error <= eps, except nom0 = NoH^2 (alpha^2 - 1) + 1, which
    cancels near a highlight (absolute error ~4 eps in NoH^2, so relative 4 eps / nom0, squared in nom), and c, which
    carries the absolute error <= 4 eps |n| of the fp32 products.  So |dT| <= eps (32 |T| + 16 |S v c w| / nom0 +
    8 B v w |n|)."""
    dirs, domega = (t.double() for t in grid)
    t = lambda x: x.double()  # noqa: E731
    rays, normal, acc = t(ch["rays"]), t(ch["normal"]), t(ch["acc"])
    albedo = t(ch["albedo"]) * torch.as_tensor(rescale, dtype=torch.float64).reshape(-1).expand(3)
    rough, fresnel = t(ch["rough"]), t(ch["fresnel"])
    n, K = rays.shape[0], dirs.shape[0]
    hit = acc > thr
    Ld = dirs[None].expand(n, K, 3)
    cos = (Ld * normal[:, None]).sum(-1)
    pos = res["pos"].long()
    v = res["vis"].double()[pos.clamp(min=0)]
    v = torch.where(pos >= 0, 1 - v if vis_kind else v, 0.0)
    spec = GGX_specular(normal, -rays[:, 3:], Ld, rough, fresnel)
    B = albedo[:, None] / math.pi + spec
    w = (v * cos * domega)[..., None]
    T = torch.where(hit[:, None, None], B * w, 0.0)
    V = torch.nn.functional.normalize(-rays[:, 3:], dim=-1)
    N = torch.nn.functional.normalize(normal, dim=-1)
    N = N * (V * N).sum(-1, keepdim=True).sign()
    H = torch.nn.functional.normalize(Ld + V[:, None], dim=-1)
    NoH = (N[:, None] * H).sum(-1, keepdim=True).clamp(1e-6, 1)
    nom0 = NoH * NoH * ((rough ** 4)[:, None] - 1) + 1
    dT = EPS * (32 * T.abs() + 16 * (spec * w).abs() / nom0
                + 8 * B * (v * domega)[..., None] * normal.norm(dim=-1)[:, None, None])
    return T.permute(2, 0, 1), dT.permute(2, 0, 1), hit


def check_against_definition(ch, grid, res, vis_kind, rescale, list_order=True, factor=1):
    """``factor`` widens the fp32 bound: 1 for the host build, 2 for the device's, whose compiler contracts the GGX
    terms into fused multiply-adds."""
    n, K = ch["rays"].shape[0], grid[0].shape[0]
    joins = expected_joins(ch, grid[0])
    got = res["pos"] >= 0
    assert torch.equal(got, joins) and joins.any() and (~joins).any()
    rows = res["pos"][got].long()
    assert torch.equal(rows if list_order else rows.sort().values, torch.arange(int(got.sum())))
    assert res["list_o"].shape[0] == int(got.sum())
    i, k = got.nonzero(as_tuple=True)
    p32 = torch.from_numpy(ch["rays"][:, :3].numpy() + ch["depth"][:, None].numpy() * ch["rays"][:, 3:].numpy())
    assert torch.equal(res["list_o"][rows], p32[i]) and torch.equal(res["list_d"][rows], grid[0][k])
    T64, bound, hit = transport64(ch, grid, res, vis_kind, rescale)
    T = res["T"].double()
    assert T.shape == (3, n, K)
    err = (T - T64).abs()
    assert (err <= factor * bound + 1e-30).all(), float((err / (bound + 1e-30)).max())
    assert float((err / (bound + 1e-30)).max()) > 1e-3                       # the bound is not vacuous
    assert not T[:, ~hit].any()                                              # non-hit rows are zero
    assert not T.permute(1, 2, 0)[~joins].any()                              # cosine <= 1e-6: zero
    assert (T.permute(1, 2, 0)[joins] > 0).float().mean() > 0.9


@pytest.mark.parametrize("stride,vis_kind", [(1, 0), (3, 1)])
def test_host_build_matches_definition(host_lib, stride, vis_kind):
    n = 400
    ch = random_chunk(70 + stride, n, stride)
    grid = LF.texel_tables(8, 16)
    rescale = [1.2, 0.9, 1.05]
    res = run_transport(ch, grid, vis_kind, rescale, seed=stride)
    check_against_definition(ch, grid, res, vis_kind, rescale)
    again = run_transport(ch, grid, vis_kind, rescale, seed=stride)
    assert all(torch.equal(res[k], again[k]) for k in res)


def test_empty_chunk(host_lib):
    ch = random_chunk(3, 0, 1)
    grid = LF.texel_tables(4, 8)
    pos, list_o, _ = LF.transport_sample(grid, ch["rays"], ch["depth"], ch["normal"], ch["acc"], 0.5)
    assert pos.shape == (0, 32) and list_o.shape == (0, 3)
    T = LF.transport_build(grid, ch["rays"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"], 0.5,
                           1.0, pos, torch.zeros(1), 'nerv')
    assert T.shape == (3, 0, 32)
    assert LF.transport_chunk(None, ch["rays"], tuple(ch[k] for k in ("depth", "normal", "albedo", "rough",
                                                                       "fresnel", "acc")), 1.0, grid).shape == (3, 0, 32)


def test_transport_arguments(host_so):
    lib = host_so
    buf = (C.c_float * 4096)()
    ibuf = (C.c_int32 * 1024)()
    cnt = (C.c_int64 * 1)()

    def sample(K=8, n=4, dirs=buf, rays=buf, cap=32, lo=buf, cnt_=cnt, pos=ibuf):
        cnt[0] = 0
        return lib.tir_transport_sample(dirs, K, rays, buf, buf, buf, n, 0.5, pos, lo, buf, cap, cnt_, None)

    def build(K=8, n=4, dirs=buf, dom=buf, stride=1, vis_kind=0, alb=buf, T=buf, vis=buf, pos=ibuf):
        return lib.tir_transport_build(dirs, dom, K, buf, buf, alb, buf, stride, buf, buf, n, 0.5, buf, pos, vis,
                                       vis_kind, T, None)
    assert sample() == 0 and build() == 0 and build(stride=3) == 0 and build(vis_kind=1) == 0
    for call in (sample, build):
        assert call(n=0) == 0 and call(n=0, dirs=None) == 0               # nothing to do
        assert call(n=-1) == -2 and call(K=0) == -2 and call(K=-1) == -2
        assert call(K=_lib.TRANSPORT_MAX_TEXELS + 1) == -2 and call(K=_lib.TRANSPORT_MAX_TEXELS + 1, n=0) == -2
        assert call(K=2048, n=(1 << 31) // 2048) == -2                      # more than INT32_MAX (ray, texel) pairs
        assert call(dirs=None) == -1 and call(pos=None) == -1
    assert sample(rays=None) == -1 and sample(cnt_=None) == -1 and sample(lo=None) == -1
    assert sample(cap=0, lo=None) == 0 and sample(cap=-1) == -2 and sample(cap=1 << 31) == -2
    assert build(stride=2) == -2 and build(vis_kind=2) == -3 and build(vis_kind=-1) == -3
    assert build(dom=None) == -1 and build(alb=None) == -1 and build(T=None) == -1 and build(vis=None) == -1


def test_max_texels_constant(tmp_path):
    src = tmp_path / "k.c"
    src.write_text('#include <stdio.h>\n#include "tensoir_b200.h"\n'
                   'int main(void){printf("%d %d\\n", TIR_TRANSPORT_MAX_TEXELS, TIR_ABI_VERSION);return 0;}\n')
    exe = tmp_path / "k"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert [int(v) for v in out] == [_lib.TRANSPORT_MAX_TEXELS, 4] == [2048, _lib.ABI_VERSION]


# ---- 2. the texel tables ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("H", [4, 16, 32])
def test_texel_tables_are_environment_lights(H):
    from tensoir_b200.relight import Environment_Light
    W = 2 * H
    rgb = np.random.default_rng(H).uniform(0.1, 2.0, (H, W, 3)).astype(np.float32)
    env = Environment_Light({"m": rgb}, device="cpu")
    dirs, domega = LF.texel_tables(H, W)
    assert dirs.dtype == domega.dtype == torch.float32 and dirs.shape == (H * W, 3) and domega.shape == (H * W,)
    assert torch.equal(dirs, env.hdr_dir["m"].reshape(-1, 3))
    ratio = (env.hdr_pdf_sample["m"] / env.hdr_pdf_return["m"]).reshape(-1)
    assert torch.allclose(domega, ratio, rtol=8 * EPS, atol=0)


@pytest.mark.parametrize("res", [(3, 6), (33, 66), (16, 16), (16, 33), (8.0, 16)])
def test_texel_tables_reject(res):
    with pytest.raises(ValueError):
        LF.texel_tables(*res)


# ---- 3. the solver ----------------------------------------------------------------------------------------------------

def augmented(T, y, H_e, W_e, smooth, ridge):
    """[T; sqrt(smooth s) D; sqrt(ridge s) I] and [y; 0; 0] with s = trace(T^T T) / K."""
    K = T.shape[1]
    s = float((T * T).sum()) / K
    D = LF.difference_operator(H_e, W_e).numpy()
    A = np.concatenate([T, math.sqrt(smooth * s) * D, math.sqrt(ridge * s) * np.eye(K)])
    return A, np.concatenate([y, np.zeros(A.shape[0] - T.shape[0])])


def lsq_objective(A, b, x):
    return 0.5 * float(((A @ x - b) ** 2).sum())


@pytest.mark.parametrize("case", ["well_posed", "rank_deficient"])
def test_solve_matches_lsq_linear(case):
    from scipy.optimize import lsq_linear
    H_e, W_e = 4, 8
    K = H_e * W_e
    g = np.random.default_rng(1 if case == "well_posed" else 2)
    if case == "well_posed":
        Ts = [g.uniform(0, 1, (300, K)) * (g.uniform(size=(300, K)) < 0.6) for _ in range(3)]
        smooth, ridge = 1e-3, 1e-6
    else:                                   # rank 5, and half the texels never seen
        Ts = [np.concatenate([g.uniform(0, 1, (300, 5)) @ g.uniform(0, 1, (5, K // 2)), np.zeros((300, K // 2))], 1)
              for _ in range(3)]
        smooth, ridge = 1e-2, 1e-3
    L_true = g.uniform(0, 2, (K, 3)) * (g.uniform(size=(K, 3)) < 0.7)
    ys = [[Tc @ L_true[:, c] + g.normal(0, 0.05, 300) for c, Tc in enumerate(Ts)],
          [Tc @ (0.5 * L_true[:, c]) - 0.3 for c, Tc in enumerate(Ts)]]           # two lights
    G = torch.tensor(np.stack([Tc.T @ Tc for Tc in Ts]))
    B = torch.tensor(np.stack([np.stack([Tc.T @ ys[l][c] for l in range(2)], 1) for c, Tc in enumerate(Ts)]))
    X, info = LF.solve(G, B, H_e, W_e, smooth, ridge, max_iters=50000, tol=1e-12)
    assert X.shape == (2, K, 3) and (X >= 0).all() and len(info) == 2
    for l in range(2):
        assert info[l]["iterations"] < 50000 and info[l]["change"] < 1e-12
        for c in range(3):
            A, b = augmented(Ts[c], ys[l][c], H_e, W_e, smooth, ridge)
            ref = lsq_linear(A, b, bounds=(0, np.inf), tol=1e-14, max_iter=10000).x
            want, got = lsq_objective(A, b, ref), lsq_objective(A, b, X[l, :, c].numpy())
            assert got <= want * (1 + 1e-6) + 1e-12, (l, c, got, want)
    X2, _ = LF.solve(G, B, H_e, W_e, smooth, ridge, max_iters=50000, tol=1e-12)
    assert torch.equal(X, X2)                                                    # deterministic
    one, _ = LF.solve(G, B[:, :, 1:2].clone(), H_e, W_e, smooth, ridge, max_iters=50000, tol=1e-12)
    assert torch.equal(one[0], X[1])                                             # a light does not see its company


def test_solve_zero_data():
    K = 32
    X, info = LF.solve(torch.zeros(3, K, K, dtype=torch.float64), torch.zeros(3, K, 2, dtype=torch.float64), 4, 8)
    assert not X.any() and X.shape == (2, K, 3) and info[0]["iterations"] == 1
    # data that asks for negative light gives the zero map too
    G = torch.eye(K, dtype=torch.float64).expand(3, K, K).clone()
    X, _ = LF.solve(G, -torch.ones(3, K, 1, dtype=torch.float64), 4, 8)
    assert not X.any()


def test_difference_operator_wraps_in_longitude():
    D = LF.difference_operator(4, 8)
    assert D.shape == (4 * 8 + 3 * 8, 32)
    x = torch.arange(32, dtype=torch.float64).view(4, 8)
    d = D @ x.reshape(-1)
    assert torch.equal(d[:32].view(4, 8)[:, :7], torch.ones(4, 7, dtype=torch.float64))
    assert torch.equal(d[:32].view(4, 8)[:, 7], torch.full((4,), -7.0, dtype=torch.float64))   # column 7 -> column 0
    assert torch.equal(d[32:], torch.full((24,), 8.0, dtype=torch.float64))
    assert torch.equal(D @ torch.ones(32, dtype=torch.float64), torch.zeros(56, dtype=torch.float64))


def test_normal_equations_and_residual():
    g = torch.Generator().manual_seed(4)
    K, L, n = 32, 3, 200
    ne = LF.Normals(K, L, "cpu")
    chunks = []
    for _ in range(2):
        T = torch.rand(3, n, K, generator=g)
        y = torch.rand(L, n, 3, generator=g, dtype=torch.float64)
        use = torch.rand(n, 3, generator=g) < 0.8
        ne.add(T, y, use)
        chunks.append((T, y, use))
    X = torch.rand(L, K, 3, generator=g, dtype=torch.float64)
    ss, cnt = torch.zeros(L, dtype=torch.float64), 0
    for T, y, use in chunks:
        pred = torch.einsum('cnk,lkc->lnc', T.double(), X)
        ss += (((pred - y) ** 2) * use[None]).sum(dim=(1, 2))
        cnt += int(use.sum())
    assert sum(ne.used) == cnt
    assert np.allclose(ne.residual_rms(X), torch.sqrt(ss / cnt).numpy(), rtol=1e-9)
    # the columns of a three-light accumulator are single-light accumulators, to the bit
    for l in range(L):
        one = LF.Normals(K, 1, "cpu")
        for T, y, use in chunks:
            one.add(T, y[l:l + 1], use)
        assert torch.equal(one.G, ne.G) and torch.equal(one.B[:, :, 0], ne.B[:, :, l])


# ---- 4. colour and arguments -----------------------------------------------------------------------------------------

def tone32(x):
    """tir::tone in fp32."""
    t = torch.as_tensor(x, dtype=torch.float32).clamp(0, 1)
    return torch.where(t <= 0.0031308, t * 12.92, 1.055 * torch.pow(t + 1e-6, 1 / 2.4) - 0.055)


def test_srgb_inverse_reproduces_every_code():
    codes = torch.arange(256, dtype=torch.float64) / 255
    lin = LF.srgb_to_linear(codes)
    assert lin.dtype == torch.float64 and (lin >= 0).all() and (lin[1:] > lin[:-1]).all()
    assert (tone32(lin.float()).double() - codes).abs().max() < 0.5 / 255
    assert (LF.linear_to_srgb(lin) - codes).abs().max() < 1e-6
    assert (tone32(lin.float()) * 255 + 0.5).floor().to(torch.int64).tolist() == list(range(256))


def test_saturated_channels_are_excluded_for_every_light():
    y = torch.full((3, 4, 3), 0.5, dtype=torch.float64)
    y[1, 0, 2] = 255 / 255                   # pixel 0, blue, clipped under light 1 only
    y[2, 1, 0] = 254.6 / 255                 # pixel 1, red, above 254.5/255 under light 2
    y[0, 2, 1] = 254.4 / 255                 # pixel 2, green, still usable
    hit = torch.tensor([True, True, True, False])
    use = LF.usable(y, hit)
    want = torch.ones(4, 3, dtype=torch.bool)
    want[0, 2] = want[1, 0] = False
    want[3] = False
    assert torch.equal(use, want)


@pytest.mark.parametrize("spec,n,want", [("0::10", 25, [0, 10, 20]), ("5::10", 25, [5, 15]), ("1,3", 4, [1, 3]),
                                         ("none", 4, []), ("2:5", 9, [2, 3, 4]), (":3", 9, [0, 1, 2]),
                                         ("0:100:40", 50, [0, 40])])
def test_parse_views(spec, n, want):
    assert LF.parse_views(spec, n) == want


@pytest.mark.parametrize("spec", ["4", "-1", "a:b", "0:4:0", "0:4:-1", "1,1", "1:2:3:4", "1;2", "x"])
def test_parse_views_rejects(spec):
    with pytest.raises(ValueError):
        LF.parse_views(spec, 4)


def _tool():
    spec = importlib.util.spec_from_file_location("fit_lights_tool", os.path.join(REPO, "tools", "fit_lights.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_fit_tool_arguments():
    tool = _tool()
    argv = ["fit_lights.py", "--config", "c.txt", "--fit_views", "0:40:4", "--fit_res", "8x16", "--out", "o",
            "--pixels_per_view", "1000", "--smooth", "0.01", "--ridge", "0", "--eval_views", "none", "--ckpt", "k"]
    got = tool.parse_fit_args(argv)
    assert argv == ["fit_lights.py", "--config", "c.txt", "--ckpt", "k"]            # left for opt.config_parser
    assert got == {"fit_views": "0:40:4", "eval_views": "none", "fit_res": (8, 16), "pixels_per_view": 1000,
                   "smooth": 0.01, "ridge": 0.0, "out": "o"}
    assert tool.parse_fit_args(["x", "--out", "o"]) == {"out": "o"}


@pytest.mark.parametrize("argv,msg", [
    (["x"], "--out"),
    (["x", "--out"], "needs a value"),
    (["x", "--out", "o", "--fit_res", "16x16"], "H x 2H"),
    (["x", "--out", "o", "--fit_res", "big"], "16x32"),
    (["x", "--out", "o", "--fit_res", "2x4"], "H x 2H"),
    (["x", "--out", "o", "--fit_views", "a:b"], "views"),
    (["x", "--out", "o", "--eval_views", "0:9:0"], "views"),
    (["x", "--out", "o", "--pixels_per_view", "many"], "bad value"),
    (["x", "--out", "o", "--pixels_per_view", "0"], "at least 1"),
    (["x", "--out", "o", "--smooth", "-1"], ">= 0"),
])
def test_fit_tool_rejects(argv, msg):
    with pytest.raises(SystemExit, match=msg):
        _tool().parse_fit_args(list(argv))
