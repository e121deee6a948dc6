"""Fitting environment maps to photographs on the H100: the tir_transport kernels against their host build, the
transport against the expectation of relight()'s own estimator, round trips on the lego scene (exact transport
photographs, and relight() photographs), one pass for many lights, and fit_lights end to end.

The lego scene's appearance is untrained and its predicted normals mean nothing, so the scene tests shade with the
boxes' face normals, as tests/test_lighting_gpu.py does.  The GGX terms (csrc/tir_ggx.h) are contracted into FMAs by the
device compiler, so the transport agrees with the host build to rounding, not to the bit; what the sample kernel writes
does to the bit, up to the order of the list."""
import math
import os
import types

import numpy as np
import pytest
import torch

from gpu_helpers import load_fixture, model_from_fixture
from helpers import build_host_lib, use_host
from test_lighting_cpu import random_chunk
from test_light_fit_cpu import check_against_definition, transport64
from test_material_edit_gpu import Replay

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H_E, W_E = 16, 32


@pytest.fixture(scope="module")
def fx():
    import __graft_entry__ as g
    g.build()
    return load_fixture("rotated_g24.pt")


# ---- 5. kernels against the host build ----------------------------------------------------------------------------------

@pytest.mark.parametrize("stride,vis_kind", [(1, 0), (3, 1)])
def test_kernels_match_host_build(fx, tmp_path, monkeypatch, stride, vis_kind):
    from tensoir_b200 import light_fit as LF
    n = 3000
    ch = random_chunk(90 + stride, n, stride)
    grid = LF.texel_tables(H_E, W_E)
    dgrid = tuple(t.to(DEV) for t in grid)
    dch = {k: v.to(DEV) for k, v in ch.items()}
    rescale = [1.2, 0.9, 1.05]
    pos, list_o, list_d = (t.cpu() for t in LF.transport_sample(dgrid, dch["rays"], dch["depth"], dch["normal"],
                                                                 dch["acc"], 0.5))
    host = build_host_lib(tmp_path, "host_transport.cpp")
    use_host(monkeypatch, host)
    hpos, hlist_o, hlist_d = LF.transport_sample(grid, ch["rays"], ch["depth"], ch["normal"], ch["acc"], 0.5)
    monkeypatch.undo()
    joined = hpos >= 0
    assert torch.equal(pos >= 0, joined) and list_o.shape == hlist_o.shape
    rows, hrows = pos[joined].long(), hpos[joined].long()
    assert torch.equal(rows.sort().values, torch.arange(rows.numel()))     # the append order differs, the set does not
    assert torch.equal(list_o[rows], hlist_o[hrows]) and torch.equal(list_d[rows], hlist_d[hrows])
    # the same visibility per (ray, texel) for both builds: the kernel's list is the host's, permuted
    hvis = torch.rand(max(hrows.numel(), 1), generator=torch.Generator().manual_seed(5))
    vis = torch.empty_like(hvis)
    vis[rows] = hvis[hrows]
    eq = 'nerfactor' if vis_kind else 'nerv'
    T = LF.transport_build(dgrid, dch["rays"], dch["normal"], dch["albedo"], dch["rough"], dch["fresnel"], dch["acc"],
                           0.5, rescale, pos.to(DEV), vis.to(DEV), eq)
    T2 = LF.transport_build(dgrid, dch["rays"], dch["normal"], dch["albedo"], dch["rough"], dch["fresnel"],
                            dch["acc"], 0.5, rescale, pos.to(DEV), vis.to(DEV), eq)
    assert torch.equal(T, T2)
    res = dict(pos=pos, list_o=list_o, list_d=list_d, vis=vis, T=T.cpu())
    check_against_definition(ch, grid, res, vis_kind, rescale, list_order=False, factor=2)
    use_host(monkeypatch, host)
    hT = LF.transport_build(grid, ch["rays"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"], 0.5,
                            rescale, hpos, hvis, eq)
    monkeypatch.undo()
    # the host build lies within the bound of the float64 result and the device's within twice it
    _, bound, _ = transport64(ch, grid, res, vis_kind, rescale)
    assert ((res["T"].double() - hT.double()).abs() <= 3 * bound + 1e-30).all()


# ---- 6. consistency with relight() -----------------------------------------------------------------------------------------

def test_transport_is_the_expectation_of_relight(fx):
    """For a random positive 16x32 map L: sum_k T L equals, within the fp32 bound, the float64 expectation of
    relight_chunk_fused's estimator over Environment_Light's sampling distribution with the same visibility; and
    relight_chunk_fused with 8192 samples lands within 6 estimated standard errors of it on every hit row."""
    from tensoir_b200 import light_fit as LF, relighting as R
    from tensoir_b200.relight import Environment_Light
    m = model_from_fixture(fx, DEV)
    rays, maps = R.chunk_inputs(fx["rays"].to(DEV), tuple(t.to(DEV) for t in fx["relight_maps"]))
    depth, normal, albedo, rough, fresnel, acc = maps
    n = rays.shape[0]
    g = np.random.default_rng(6)
    rgb = g.uniform(0.05, 1.0, (H_E, W_E, 3)).astype(np.float32)
    rescale = 1.1
    grid = LF.texel_tables(H_E, W_E, DEV)
    pos, lo, ld = LF.transport_sample(grid, rays, depth, normal, acc, 0.5)
    vis = R.march_list(m, lo, ld, 'nerv')
    T = LF.transport_build(grid, rays, normal, albedo, rough, fresnel, acc, 0.5, rescale, pos, vis, 'nerv')
    hit = (acc > 0.5).cpu()
    assert hit.sum() > 10
    ch = {k: v.cpu() for k, v in dict(rays=rays, depth=depth, normal=normal, albedo=albedo, rough=rough,
                                      fresnel=fresnel, acc=acc).items()}
    res = dict(pos=pos.cpu(), vis=vis.cpu())
    T64, bound, _ = transport64(ch, tuple(t.cpu() for t in grid), res, 0, rescale)
    # scale the map so that the brightest hit stays below the tone map's clip
    lin = torch.einsum('cnk,kc->nc', T64, torch.tensor(rgb, dtype=torch.float64).reshape(-1, 3))
    rgb = rgb * np.float32(0.5 / float(lin[hit].max()))
    Lmap = torch.tensor(rgb, dtype=torch.float64).reshape(-1, 3)
    env = Environment_Light({"r": rgb}, device=DEV)
    pdf = env.hdr_pdf_sample["r"].reshape(-1).double().cpu()
    pdf_ret = env.hdr_pdf_return["r"].reshape(-1).double().cpu()
    # X_b = brdf vis rgb_b cos / pdf_return_b for a draw of bin b with probability pdf_b: T64 / dOmega is brdf vis cos
    X = (T64 / grid[1].cpu().double()).permute(1, 2, 0) * Lmap[None] / pdf_ret[None, :, None]         # [n, K, 3]
    mean = (pdf[None, :, None] * X).sum(1)
    second = (pdf[None, :, None] * X * X).sum(1)
    got = torch.einsum('cnk,kc->nc', T.cpu().double(), Lmap)
    tol = 2 * torch.einsum('cnk,kc->nc', bound, Lmap) + 8 * 1.2e-7 * torch.einsum('cnk,kc->nc', T64.abs(), Lmap)
    assert ((got - mean).abs() <= tol + 1e-30).all(), float(((got - mean).abs() / (tol + 1e-30)).max())
    S = 8192
    u = torch.rand(1, n, S, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(8))
    _, wo = R.relight_chunk_fused(m, env, ["r"], rays, maps, rescale, u, S)
    est = LF.srgb_to_linear(wo[0].cpu())
    se = ((second - mean * mean).clamp(min=0) / S).sqrt()
    z = ((est - mean).abs() - 1e-5) / se.clamp(min=1e-30)
    assert (z[hit] <= 6).all(), float(z[hit].max())
    assert not (wo[0].cpu()[~hit] != 1).any()


# ---- the lego scene ---------------------------------------------------------------------------------------------------------

def sky_and_sun(dirs):
    """L* [K, 3]: a sky gradient over a dim ground and a sun lobe."""
    z = dirs[:, 2:3]
    sky = torch.tensor([0.25, 0.3, 0.45], device=dirs.device) * (0.3 + 0.7 * z.clamp(min=0))
    ground = torch.tensor([0.12, 0.1, 0.08], device=dirs.device) * (z < 0)
    s = torch.tensor([0.4, -0.3, 0.87], device=dirs.device)
    s = s / s.norm()
    sun = 6.0 * torch.exp(((dirs * s).sum(-1, keepdim=True) - 1) / 0.03) * torch.tensor([1.0, 0.9, 0.7],
                                                                                           device=dirs.device)
    return (sky + ground + sun).double()


@pytest.fixture(scope="module")
def lego():
    return lego_views()


def lego_views():
    """12 hemisphere views of the lego scene at 200x200: per view the hit rows' rays, maps with the boxes' face normals
    and transport chunks (batch 4096) to the 16x32 texels."""
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import light_fit as LF, relighting as R
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    m = make_lego_model(96, DEV)
    ds = SyntheticViews(hemisphere_poses(12), 200, 200, light_names=["a"])
    grid = LF.texel_tables(H_E, W_E, DEV)
    views = []
    for i in range(len(ds)):
        item = ds[i]
        rays_v = item["rays"].to(DEV)
        li = torch.zeros(rays_v.shape[0], 1, dtype=torch.int32, device=DEV)
        with torch.no_grad():
            _, depth, _, albedo, rough, fresnel, acc, *_ = m(rays_v, li, is_train=False, white_bg=True, ndc_ray=False,
                                                              N_samples=-1)
        fg = (acc.reshape(-1) > 0.5).nonzero().reshape(-1)
        rays, maps = R.chunk_inputs(rays_v[fg], tuple(t.detach()[fg] for t in (depth, item["normals"].to(DEV), albedo,
                                                                               rough, fresnel, acc)))
        chunks = []
        for s in range(0, fg.numel(), 4096):
            sl = slice(s, s + 4096)
            chunks.append(LF.transport_chunk(m, rays[sl], tuple(t[sl] for t in maps), 1.0, grid))
        views.append(dict(rays=rays, maps=maps, T=chunks))
        assert fg.numel() > 4000
    return m, grid, views


def exact_photos(T, X):
    """tone(T X) rounded to 8 bits, [L, n, 3] fp64: X [L, K, 3]."""
    from tensoir_b200 import light_fit as LF
    return (LF.linear_to_srgb(torch.einsum('cnk,lkc->lnc', T.double(), X)) * 255).round() / 255


def psnr(a, b):
    return -10 * math.log10(float(((a - b) ** 2).mean()))


def test_exact_round_trip(lego):
    """Photos tone(T L*) on 8 bits: fit on 8 views, the 4 held-out views' foreground within 40 dB."""
    from tensoir_b200 import light_fit as LF
    m, grid, views = lego
    K = H_E * W_E
    X_true = sky_and_sun(grid[0])[None]
    ne = LF.Normals(K, 1, DEV)
    for v in views[:8]:
        for T in v["T"]:
            y = exact_photos(T, X_true)
            ne.add(T, LF.srgb_to_linear(y), LF.usable(y, torch.ones(T.shape[1], dtype=torch.bool, device=DEV)))
    X, info = LF.solve(ne.G, ne.B, H_E, W_E)
    assert ne.saturated < 0.01 * sum(ne.used)
    pred, want = [], []
    for v in views[8:]:
        for T in v["T"]:
            pred.append(LF.linear_to_srgb(torch.einsum('cnk,lkc->lnc', T.double(), X)))
            want.append(exact_photos(T, X_true))
    p = psnr(torch.cat(pred, 1), torch.cat(want, 1))
    err = (X[0] - X_true[0]).abs()
    print(f"exact round trip: held-out PSNR {p:.2f} dB; per-texel |L - L*| mean {float(err.mean()):.4f}, "
          f"max {float(err.max()):.4f}, mean |L*| {float(X_true.abs().mean()):.4f}; {info[0]}")
    assert p >= 40.0


def test_round_trip_through_relight(lego):
    """Photos are relight()'s images under L* (512 importance samples, 8 bits): the held-out views relit under the
    fitted map score no more than 0.5 dB below relight() under L* itself with another random stream."""
    from tensoir_b200 import light_fit as LF, relighting as R
    from tensoir_b200.relight import Environment_Light
    m, grid, views = lego
    K = H_E * W_E
    L_true = sky_and_sun(grid[0]).float()
    env = Environment_Light({"true": L_true.reshape(H_E, W_E, 3).cpu().numpy()}, device=DEV)
    gen = torch.Generator(DEV).manual_seed(21)

    def render(e, name, v, sl):
        rays = v["rays"][sl]
        u = torch.rand(1, rays.shape[0], 512, dtype=torch.float64, device=DEV, generator=gen)
        return R.relight_chunk_fused(m, e, [name], rays, tuple(t[sl] for t in v["maps"]), 1.0, u, 512)[1]

    photos = []
    for v in views:
        photos.append([(render(env, "true", v, slice(s, s + 4096)) * 255).to(torch.uint8).double() / 255
                       for s in range(0, v["rays"].shape[0], 4096)])
    ne = LF.Normals(K, 1, DEV)
    for v, ph in zip(views[:8], photos[:8]):
        for T, y in zip(v["T"], ph):
            ne.add(T, LF.srgb_to_linear(y), LF.usable(y, torch.ones(T.shape[1], dtype=torch.bool, device=DEV)))
    X, info = LF.solve(ne.G, ne.B, H_E, W_E)
    fitted = Environment_Light({"fit": X[0].float().reshape(H_E, W_E, 3).cpu().numpy()}, device=DEV)
    fit, floor, want = [], [], []
    for v, ph in zip(views[8:], photos[8:]):
        for k, s in enumerate(range(0, v["rays"].shape[0], 4096)):
            fit.append(render(fitted, "fit", v, slice(s, s + 4096)).double())
            floor.append(render(env, "true", v, slice(s, s + 4096)).double())
            want.append(ph[k])
    want = torch.cat(want, 1)
    p_fit, p_floor = psnr(torch.cat(fit, 1), want), psnr(torch.cat(floor, 1), want)
    print(f"relight round trip: fitted {p_fit:.2f} dB, noise floor {p_floor:.2f} dB; {info[0]}")
    assert p_fit >= p_floor - 0.5


def test_one_pass_serves_all_lights(lego):
    """Three lights fitted in one pass give, on the same (replayed) transport, the maps of three single-light fits to
    the bit."""
    from tensoir_b200 import light_fit as LF
    m, grid, views = lego
    K = H_E * W_E
    base = sky_and_sun(grid[0])
    X_true = torch.stack([0.5 * base, base.roll(5, 0) * 0.4, 0.2 + 0.1 * base.flip(1)])
    chunks = [T for v in views[:4] for T in v["T"]]
    photos = [exact_photos(T, X_true) for T in chunks]
    assert all(bool((y < LF.SATURATED).all()) for y in photos)       # one Gram matrix: no clipped channel anywhere
    ones = lambda T: torch.ones(T.shape[1], dtype=torch.bool, device=DEV)  # noqa: E731
    ne = LF.Normals(K, 3, DEV)
    for T, y in zip(chunks, photos):
        ne.add(T, LF.srgb_to_linear(y), LF.usable(y, ones(T)))
    X3, info3 = LF.solve(ne.G, ne.B, H_E, W_E)
    for l in range(3):
        one = LF.Normals(K, 1, DEV)
        for T, y in zip(chunks, photos):
            one.add(T, LF.srgb_to_linear(y[l:l + 1]), LF.usable(y[l:l + 1], ones(T)))
        X1, info1 = LF.solve(one.G, one.B, H_E, W_E)
        assert torch.equal(one.G, ne.G) and torch.equal(X1[0], X3[l]) and info1[0] == info3[l]


# ---- 10. fit_lights end to end ------------------------------------------------------------------------------------------------

def test_fit_lights_end_to_end(tmp_path, monkeypatch):
    import cv2
    from tensoir_b200 import light_fit as LF
    from tensoir_b200.relight import read_hdr
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model
    m = make_lego_model(64, DEV)
    ds = SyntheticViews(hemisphere_poses(6), 40, 40, light_names=["sun_a", "sun_b"])
    rep = Replay(m)
    outs = []
    for run in ("a", "b"):
        args = types.SimpleNamespace(out=str(tmp_path / run / "fit"), geo_buffer_path=str(tmp_path / run / "eval"),
                                     batch_size=700, fit_views="0:4", eval_views="4,5", fit_res="8x16",
                                     pixels_per_view=900)
        outs.append(LF.fit_lights(ds, args, tensoIR=m))
        rep.i = 0
    (report, maps), (_, maps_b) = outs
    a = tmp_path / "a"
    assert sorted(os.listdir(a / "fit")) == ["fit_report.json", "sun_a.hdr", "sun_b.hdr"]
    with open(a / "fit" / "fit_report.json") as f:
        assert __import__("json").load(f) == __import__("json").loads(__import__("json").dumps(report))
    assert report["fit_res"] == [8, 16] and report["fit_views"] == [0, 1, 2, 3] and report["eval_views"] == [4, 5]
    for name in ("sun_a", "sun_b"):
        e = report["lights"][name]
        assert set(e) == {"views", "pixels_used", "pixels_excluded", "pixels_missed", "residual_rms_linear",
                          "psnr_srgb", "unobserved_texels", "iterations", "final_change", "written"}
        assert e["views"] == 4 and e["pixels_used"] > 0 and e["written"] and 0 <= e["unobserved_texels"] <= 128
        assert e["psnr_srgb"] > 10 and e["residual_rms_linear"] >= 0 and e["iterations"] >= 1
        hdr = read_hdr(str(a / "fit" / f"{name}.hdr"))
        assert hdr.shape == (8, 16, 3) and (np.abs(hdr - maps[name]) <= maps[name].max(-1, keepdims=True) / 128 + 1e-30).all()
        scale = float(np.abs(maps[name]).max())
        assert np.abs(maps[name] - maps_b[name]).max() <= 1e-5 * scale
    for i in range(2):
        for sub in ("with_bg", "without_bg"):
            for name in ("sun_a", "sun_b"):
                assert cv2.imread(str(a / "eval" / f"test_{i:03d}" / f"relighting_{sub}" / f"{name}.png")) is not None
    txt = (a / "eval" / "relight_psnr.txt").read_text().splitlines()
    assert [t.split(":")[0] for t in txt] == ["sun_a", "sun_b"]
