"""Relighting with multiple importance sampling on the H100: the tir_relight_mis kernels against their host build and
float64, determinism on the lego box field (synthetic.make_lego_model), the noise of the estimator against the default
one and against light sampling alone, and relight() end to end.

The sampler computes its directions in fp64 and rounds them once, so they match the host build to an ulp; the shade goes
through GGX terms that the device compiler contracts into fused multiply-adds, so it is checked against float64 within
twice the host build's fp32 bound (test_mis_cpu.shade_ref), on the kernels' own directions, slot map and visibility."""
import math
import types

import numpy as np
import pytest
import torch

import test_indirect_cpu as H
import test_mis_cpu as M
from helpers import build_host_lib, use_host
from tensoir_b200 import mis, relighting
from tensoir_b200.relight import Environment_Light
from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = H.EPS


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_mis_gpu"), "host_relight.cpp", "host_mis.cpp")


@pytest.fixture(scope="module")
def lego():
    import __graft_entry__ as g
    g.build()
    return make_lego_model(128, DEV)


def env_maps(names, lo=0.05, hi=3.0, seed=7):
    g = np.random.default_rng(seed)
    maps = {k: g.uniform(lo, hi, (16, 32, 3)).astype(np.float32) for k in names}
    return maps, Environment_Light(maps, device=DEV)


def lego_chunks(model, views=2, size=64):
    ds = SyntheticViews(hemisphere_poses(views, seed=3), size, size)
    out = []
    for v in range(views):
        rays = ds[v]["rays"].to(DEV)
        li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=DEV)
        with torch.no_grad():
            _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays, li, is_train=False, white_bg=True,
                                                                      ndc_ray=False, N_samples=-1)
        out.append((rays, [depth, normal, albedo, rough, fresnel, acc]))
    return out


def test_kernels_match_host_build(lego, host_so, monkeypatch):
    names = ["a", "b", "c"]
    hdr, env = env_maps(names)
    n, S_l, S_b = 2000, 48, 16
    ch = H.random_chunk(61, n, 3)
    g = torch.Generator().manual_seed(5)
    u_l = torch.rand(3, n, S_l, 3, generator=g, dtype=torch.float64)
    u_b = torch.rand(n, S_b, 3, generator=g, dtype=torch.float64)
    monkeypatch.setattr(relighting.ops, "march_density", H.plane_march())
    d = {k: t.to(DEV) for k, t in ch.items()}
    maps = (d["depth"], d["normal"], d["albedo"], d["rough"], d["fresnel"], d["acc"])
    envs, keep = relighting.env_tables(env, names)
    rays, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(d["rays"], maps)
    dirs, pos, vis = mis.mis_visibility(lego, envs, 3, rays, depth, normal, albedo, rough, fresnel, acc, u_l.to(DEV),
                                        u_b.to(DEV), 0.5, 'nerv')
    resc = torch.tensor([1.1, 0.9, 1.0])
    lin = torch.zeros(3, n, 3, device=DEV)
    mis.relight_chunk_mis(lego, env, names, d["rays"], maps, resc, u_l.to(DEV), u_b.to(DEV), linear_out=lin)
    lin2 = torch.zeros(3, n, 3, device=DEV)
    mis.relight_chunk_mis(lego, env, names, d["rays"], maps, resc, u_l.to(DEV), u_b.to(DEV), linear_out=lin2)
    assert torch.equal(lin, lin2)
    env_cpu = Environment_Light(hdr, device="cpu")
    with monkeypatch.context() as mp:
        use_host(mp, host_so, H.plane_march())
        _, _, hdirs, hpos, hvis = M.run_sample(env_cpu, names, ch, S_l, S_b, seed=5)
    dirs, pos, vis = dirs.cpu(), pos.cpu(), vis.cpu()
    # light directions: fp64 rounded once in both builds, to an ulp.  BRDF directions start from ggx_point's Np and V,
    # which the device compiler contracts into FMAs: a few ulp of the frame, carried through the reflection
    nl = 3 * n * S_l
    assert ((dirs[:nl] - hdirs[:nl]).abs() <= EPS * hdirs[:nl].abs().clamp(min=1e-3)).all()
    assert ((dirs[nl:] - hdirs[nl:]).abs() <= 32 * EPS).all(), float((dirs[nl:] - hdirs[nl:]).abs().max())
    # the cosine test can only disagree on slots whose cosine sits at the 1e-6 cut
    t = torch.arange(dirs.shape[0])
    ray = torch.where(t < nl, (t // S_l) % n, (t - nl) // S_b)
    cos = (dirs.double() * ch["normal"].double()[ray]).sum(-1)
    differ = (pos >= 0) != (hpos >= 0)
    assert ((cos[differ] - 1e-6).abs() <= 64 * EPS).all()
    # shade against float64 on the kernel's own directions, slot map and visibility
    lin = lin.cpu().double()
    hit = ch["acc"] > 0.5
    with monkeypatch.context() as mp:
        use_host(mp, host_so, H.plane_march())
        for k in range(3):
            want, bound = M.shade_ref(host_so, env_cpu, names, k, ch, dirs, pos, vis, S_l, S_b, resc)
            err = (lin[k] - want).abs()
            assert (err <= 2 * bound + 1e-30)[hit].all(), float((err / bound)[hit].max())
            assert not lin[k][~hit].any()


def test_lego_chunk_is_deterministic(lego):
    names = ["a", "b"]
    _, env = env_maps(names)
    rays, maps = lego_chunks(lego, views=1)[0]
    u_l, u_b = mis.mis_uniforms(2, rays.shape[0], 384, 128, DEV)
    a = mis.relight_chunk_mis(lego, env, names, rays, maps, 1.0, u_l, u_b)
    b = mis.relight_chunk_mis(lego, env, names, rays, maps, 1.0, u_l, u_b)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert torch.isfinite(a[0]).all() and (maps[5] > 0.5).sum() > 500


def _linear_default(env, names, lego, rays, maps, n_samples=512):
    """The default estimator's linear value, from its toned output (tone inverted below the clamp)."""
    u = relighting._uniforms(len(names), rays.shape[0], n_samples, DEV)
    _, wo = relighting.relight_chunk_fused(lego, env, names, rays, maps, 1.0, u, n_samples)
    lin = torch.where(wo <= 0.0031308 * 12.92, wo / 12.92, ((wo + 0.055) / 1.055) ** 2.4 - 1e-6)
    return lin, wo < 0.999


def test_mis_lowers_the_noise_of_glossy_highlights(lego, record_property):
    """Linear RMSE over the hit pixels of two views' chunks and three maps, against the mean of 16 MIS passes, with
    the same 512 samples per (map, hit): MIS (S_b = 128), continuous light sampling alone (S_b = 0) and the default
    estimator.  Maps dim enough that the default's sRGB output stays below its clamp."""
    names = ["a", "b", "c"]
    _, env = env_maps(names, lo=0.02, hi=0.6, seed=11)
    torch.manual_seed(0)
    chunks = lego_chunks(lego)
    ratios = {}
    for r in (0.1, 0.3, 0.99):
        sq = {"mis": 0.0, "light": 0.0, "default": 0.0}
        count = 0
        for rays, maps in chunks:
            maps = list(maps)
            maps[3] = torch.full_like(maps[3], r)
            n = rays.shape[0]
            hit = maps[5].reshape(-1) > 0.5

            def run(S_b):
                lin = torch.zeros(3, n, 3, device=DEV)
                u_l, u_b = mis.mis_uniforms(3, n, 512 - S_b, S_b, DEV)
                mis.relight_chunk_mis(lego, env, names, rays, maps, 1.0, u_l, u_b, linear_out=lin)
                return lin
            ref = sum(run(128) for _ in range(16)) / 16
            d_lin, ok = _linear_default(env, names, lego, rays, maps)
            mask = hit[None, :, None] & ok & (ref < 0.9)
            assert mask.float().mean() > 0.2
            for key, est in (("mis", run(128)), ("light", run(0)), ("default", d_lin)):
                sq[key] += float(((est - ref) ** 2)[mask].sum())
            count += int(mask.sum())
        rmse = {k: math.sqrt(v / count) for k, v in sq.items()}
        ratios[r] = dict(rmse, mis_over_light=rmse["mis"] / rmse["light"], mis_over_default=rmse["mis"] / rmse["default"])
        record_property(f"rmse_rough_{r}", ratios[r])
        print(f"roughness {r}: {ratios[r]}")
    for r in (0.1, 0.3):
        assert ratios[r]["mis"] < ratios[r]["light"] and ratios[r]["mis"] < ratios[r]["default"], ratios[r]
    assert ratios[0.99]["mis"] <= 1.1 * ratios[0.99]["light"], ratios[0.99]


def test_relight_end_to_end(lego, tmp_path):
    names = ["a", "b"]
    hdr, _ = env_maps(names)
    ds = SyntheticViews(hemisphere_poses(1, seed=2), 24, 24, light_names=names)
    files = {}
    for sampling in ("light", "mis"):
        out = tmp_path / sampling
        args = types.SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(out), batch_size=300, sampling=sampling,
                                     brdf_samples=64, render_video=False)
        relighting.relight(ds, args, lego, rescale_value=[1.0, 1.0, 1.0])
        files[sampling] = sorted(str(p.relative_to(out)) for p in out.rglob("*") if p.is_file())
        import cv2
        for name in names:
            img = cv2.imread(str(out / "test_000" / "relighting_without_bg" / f"{name}.png"))
            assert img is not None and img.shape == (24, 24, 3)
        txt = (out / "relight_psnr.txt").read_text()
        assert all(np.isfinite(float(t.split("PSNR")[1].split(";")[0])) for t in txt.splitlines())
    assert files["light"] == files["mis"]
