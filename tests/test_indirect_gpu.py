"""Relighting with one bounce of indirect light on the H100: the tir_indirect kernels against their host build and
float64, on random chunks and on the lego box field (synthetic.make_lego_model).

What the sampler and the hit compaction write (directions, slot map, list rows, hit list, x, xn, w) matches the host
build to the bit; the list itself is compared through the slot map, since its order follows warp scheduling.  T, Lo and
the maps go through GGX terms that the device compiler contracts into fused multiply-adds, so they are checked against
float64 within twice the host build's fp32 bound, as test_light_fit_gpu does for the transport."""
import contextlib
import math

import numpy as np
import pytest
import torch

import test_indirect_cpu as H
from helpers import build_host_lib, use_host
from oracle import tensoir_oracle as O
from tensoir_b200 import _lib, indirect, ops, relighting
from tensoir_b200.relight import Environment_Light, read_hdr
from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses, make_lego_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = H.EPS


def to(ch, dev):
    return {k: v.to(dev) for k, v in ch.items()}


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_indirect_gpu"), "host_relight.cpp", "host_indirect.cpp")


@pytest.fixture(scope="module")
def lego():
    _lib.load()
    return make_lego_model(128, DEV)


@pytest.fixture(scope="module")
def env():
    names = ["bridge", "city", "night"]
    g = np.random.default_rng(7)
    maps = {k: g.uniform(0.05, 3.0, (16, 32, 3)).astype(np.float32) for k in names}
    return names, Environment_Light(maps, device=DEV), maps


def lego_chunk(model, n=4096, seed=0):
    ds = SyntheticViews(hemisphere_poses(1, seed=seed), 96, 96)
    rays = ds[0]["rays"].to(DEV)[:n]
    li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays, li, is_train=False, white_bg=True,
                                                                  ndc_ray=False, N_samples=-1)
    return rays, (depth, normal, albedo, rough, fresnel, acc)


# ---- 1. kernels against the host build --------------------------------------------------------------------------------

def test_kernels_match_host_build(host_so, monkeypatch):
    ch = H.random_chunk(41, 3000, 3)
    K = 24
    u = torch.rand(3000, K, 2, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    resc = torch.tensor([1.1, 0.9, 1.0])
    march = H.plane_march()
    monkeypatch.setattr(indirect.ops, "march_density", march)
    dev_ch = to(ch, DEV)
    got = indirect.secondary_hits(H.Model(), dev_ch["rays"], dev_ch["depth"], dev_ch["normal"], dev_ch["albedo"],
                                  dev_ch["rough"], dev_ch["fresnel"], dev_ch["acc"], resc.to(DEV), u.to(DEV), 0.5,
                                  'nerv')
    again = indirect.secondary_hits(H.Model(), dev_ch["rays"], dev_ch["depth"], dev_ch["normal"], dev_ch["albedo"],
                                    dev_ch["rough"], dev_ch["fresnel"], dev_ch["acc"], resc.to(DEV), u.to(DEV), 0.5,
                                    'nerv')
    with monkeypatch.context() as mp:
        use_host(mp, host_so, march)
        want = indirect.secondary_hits(H.Model(), ch["rays"], ch["depth"], ch["normal"], ch["albedo"], ch["rough"],
                                       ch["fresnel"], ch["acc"], resc, u, 0.5, 'nerv')
    got = {k: v.cpu() for k, v in got.items()}
    assert torch.equal(got["dirs"], want["dirs"])
    assert torch.equal(got["pos"] >= 0, want["pos"] >= 0)
    m = got["pos"] >= 0
    for key in ("list_o", "list_d"):
        assert torch.equal(got[key][got["pos"][m].long()], want[key][want["pos"][m].long()])
    for key in ("hit", "rays", "xn", "w"):                               # the hit list is in slot order: to the bit
        assert torch.equal(got[key], want[key]), key
    assert all(torch.equal(got[k], again[k].cpu()) for k in ("T", "hit", "rays", "xn", "w"))
    # T within twice the host's fp32 bound of float64 (the CPU test's derivation)
    om64, z64 = H.directions64(ch["normal"], u)
    B, cos, spec, nom0 = H.brdf64(ch["normal"], -ch["rays"][:, 3:], got["dirs"], ch["albedo"] * resc, ch["rough"],
                                  ch["fresnel"])
    w = cos / (z64 / math.pi)
    T64 = B * w[..., None]
    bound = EPS * (32 * T64.abs() + 16 * (spec * w[..., None]).abs() / nom0
                   + 8 * B * (ch["normal"].double().norm(dim=-1)[:, None] / (z64 / math.pi))[..., None]
                   + 4 * T64.abs() / z64.clamp(min=1e-30)[..., None] ** 2)
    err = (got["T"].double() - T64).abs()[m]
    assert (err <= 2 * bound[m]).all(), float((err / bound[m]).max())
    assert not got["T"][~m].any()


def test_chunk_matches_host_build(host_so, monkeypatch, env):
    """The whole chunk through the kernels and through the host build on the same draws and the same march."""
    names, light, hdr = env
    ch, maps = H.chunk(52, 2000)
    u = torch.rand(3, 2000, 64, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    monkeypatch.setattr(indirect.ops, "march_density", H.plane_march())
    monkeypatch.setattr(relighting.ops, "march_density", H.plane_march())
    ind = torch.zeros(3, 2000, 3, device=DEV)
    got = indirect.relight_chunk_indirect(H.Model(), light, names, ch["rays"].to(DEV), tuple(t.to(DEV) for t in maps),
                                          1.0, u.to(DEV), torch.Generator(DEV).manual_seed(3), indirect_samples=8,
                                          indirect_light_samples=16, material=H.analytic_material, indirect_out=ind)
    # the same draws on the host: the device generator's stream, replayed
    g = torch.Generator(DEV).manual_seed(3)
    u_ind = torch.rand(2000, 8, 2, generator=g, device=DEV, dtype=torch.float64).cpu()
    light_cpu = Environment_Light(hdr, device="cpu")
    with monkeypatch.context() as mp:
        use_host(mp, host_so, H.plane_march())
        hits = indirect.secondary_hits(H.Model(), ch["rays"], ch["depth"], ch["normal"], ch["albedo"], ch["rough"],
                                       ch["fresnel"], ch["acc"], torch.ones(3), u_ind, 0.5, 'nerv')
        m_h = hits["rays"].shape[0]
        u2 = torch.rand(3, m_h, 16, generator=g, device=DEV, dtype=torch.float64).cpu()
        draws = [u_ind, u2]
        real_rand = torch.rand
        mp.setattr(torch, "rand", lambda *a, **k: draws.pop(0) if "generator" in k else real_rand(*a, **k))
        ind_h = torch.zeros(3, 2000, 3)
        want = indirect.relight_chunk_indirect(H.Model(), light_cpu, names, ch["rays"], maps, 1.0, u,
                                               torch.Generator(), indirect_samples=8, indirect_light_samples=16,
                                               material=H.analytic_material, indirect_out=ind_h)
    assert m_h > 100
    # to rounding: the device contracts the GGX terms into fused multiply-adds, which near a highlight of a low
    # roughness the cancellation in nom0 amplifies (the 16 |S w| / nom0 term of the CPU test's bound)
    for a, b in zip(got, want):
        assert ((a.cpu() - b).abs() <= 1e-3).all(), float((a.cpu() - b).abs().max())
    assert torch.equal(ind.cpu() == 0, ind_h == 0)
    assert ((ind.cpu() - ind_h).abs() <= 1e-3).all(), float((ind.cpu() - ind_h).abs().max())


# ---- 2. the lego box field ------------------------------------------------------------------------------------------

@contextlib.contextmanager
def f64():
    """The oracle evaluates its intermediates in the default dtype."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


@f64()
def materials64(model, x):
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    f = O.field_from_state_dict(sd, model.aabb.cpu(), model.gridSize.tolist(), kind="rotated")
    f.light_num = int(sd["light_line.weight"].shape[0])
    xn = model.normalize_coord(x).double().cpu()
    feats = O.intrin_feature(f, xn)
    brdf = O.mlp_pe_and_feature(f, f.mlp_brdf, xn, feats, torch.sigmoid)
    nrm = O.mlp_pe_and_feature(f, f.mlp_normal, xn, feats, torch.tanh)
    return (torch.nn.functional.normalize(nrm, dim=-1), brdf[:, :3].clamp(0, 1),
            (brdf[:, 3:4] * 0.9 + 0.09).clamp(0, 1))


@f64()
def march64(model, o, d):
    """relight()'s visibility march in float64 on the oracle field: (t_last, acc, depth)."""
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    f = O.field_from_state_dict(sd, model.aabb.cpu(), model.gridSize.tolist(), kind="rotated",
                                density_shift=float(model.density_shift), distance_scale=float(model.distance_scale))
    o, d = o.double().cpu(), d.double().cpu()
    z = torch.linspace(0.05, 1.5, 96, dtype=torch.float64)
    pts = o[:, None] + d[:, None] * z[None, :, None]
    sigma = torch.zeros(pts.shape[:2], dtype=torch.float64)
    inside = ((pts >= model.aabb[0].cpu()) & (pts <= model.aabb[1].cpu())).all(-1)
    if inside.any():
        sigma[inside] = O.feature2density(f, O.density_feature(f, O.normalize_coord(f, pts[inside])))
    dist = torch.cat([z[1:] - z[:-1], torch.zeros(1, dtype=torch.float64)])
    alpha = 1 - torch.exp(-sigma * dist * float(model.distance_scale))
    T = torch.cumprod(torch.cat([torch.ones(o.shape[0], 1, dtype=torch.float64), 1 - alpha + 1e-10], 1), 1)
    w = alpha * T[:, :-1]
    return T[:, -1], w.sum(1), (w * z).sum(1)


def test_chunk_without_secondary_rays(lego):
    """A chunk where no ray counts as a surface hit: the secondary list is empty, and no slot becomes a hit."""
    rays, maps = lego_chunk(lego)
    rays_c, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(rays, maps)
    u = torch.rand(rays.shape[0], 4, 2, generator=torch.Generator(DEV).manual_seed(5), device=DEV, dtype=torch.float64)
    hits = indirect.secondary_hits(lego, rays_c, depth, normal, albedo, rough, fresnel, acc, torch.ones(3, device=DEV),
                                   u, 2.0, 'nerv')
    assert hits["list_o"].shape[0] == 0 and hits["rays"].shape[0] == 0 and bool((hits["hit"] == -1).all())


def test_lego_stages(lego, env):
    names, light, hdr = env
    rays, maps = lego_chunk(lego)
    rays_c, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(rays, maps)
    K = 16
    u = torch.rand(rays.shape[0], K, 2, generator=torch.Generator(DEV).manual_seed(5), device=DEV,
                   dtype=torch.float64)
    resc = torch.ones(3, device=DEV)
    hits = indirect.secondary_hits(lego, rays_c, depth, normal, albedo, rough, fresnel, acc, resc, u, 0.5, 'nerv')
    m_h = hits["rays"].shape[0]
    assert m_h > 500, m_h                                   # the lego's concave regions
    # the march outputs give the hits and x, as the header defines them
    q = hits["pos"][hits["hit"] >= 0].long()
    t_last, acc_s, dep = hits["t_last"][q], hits["acc"][q], hits["depth"][q]
    assert torch.equal(hits["w"], 1 - t_last) and ((1 - t_last) > 1e-3).all() and (acc_s > 0).all()
    x64 = hits["list_o"][q].double() + (dep.double() / acc_s.double())[:, None] * hits["list_d"][q].double()
    t = (dep / acc_s).double()
    assert ((hits["rays"][:, :3].double() - x64).abs()
            <= EPS * (hits["list_o"][q].double().abs() + 3 * t[:, None])).all()
    missed = (hits["pos"] >= 0) & (hits["hit"] < 0)
    qm = hits["pos"][missed].long()
    assert (((1 - hits["t_last"][qm]) <= 1e-3) | (hits["acc"][qm] <= 0)).all()
    # the fp32 march against float64 (without the alpha mask, which skips cells of alpha < 1e-3) on a sample of the
    # secondary rays
    sel = torch.randperm(hits["list_o"].shape[0], generator=torch.Generator().manual_seed(0))[:512].to(DEV)
    T64, a64, _ = march64(lego, hits["list_o"][sel], hits["list_d"][sel])
    assert (hits["t_last"][sel].double().cpu() - T64).abs().max() < 2e-3
    # materials against float64 evaluation of the heads (split-BF16 tensor-core products: tolerance, not a bound)
    normal_h, albedo_h, rough_h, fresnel_h = indirect.point_materials(lego, hits["rays"][:, :3], hits["xn"])
    n64, a64m, r64 = materials64(lego, hits["rays"][:, :3])
    assert (albedo_h.double().cpu() - a64m).abs().max() < 2e-3
    assert (rough_h.double().cpu() - r64).abs().max() < 2e-3
    assert (normal_h.double().cpu() - n64).abs().max() < 5e-3
    assert torch.equal(fresnel_h, torch.full_like(fresnel_h, float(lego.fixed_fresnel)))


def test_same_draws_with_and_without_indirect_and_determinism(lego, env, monkeypatch):
    names, light, hdr = env
    rays, maps = lego_chunk(lego, seed=3)
    L, n = len(names), rays.shape[0]
    u = torch.rand(L, n, relighting.NUM_SAMPLES, device=DEV, dtype=torch.float64,
                   generator=torch.Generator(DEV).manual_seed(11))
    run = lambda: indirect.relight_chunk_indirect(  # noqa: E731
        lego, light, names, rays, maps, 1.0, u, torch.Generator(DEV).manual_seed(12), indirect_samples=16,
        indirect_light_samples=32, indirect_out=torch.zeros(L, n, 3, device=DEV))
    a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))                  # determinism
    # the same path with Lo = 0: the direct term alone, on the same draws and the same marches
    monkeypatch.setattr(indirect, "secondary_radiance", lambda *x, **k: None)
    fwb, fwo = run()
    wb, wo = a
    hits = indirect.secondary_hits(lego, *relighting.chunk_inputs(rays, maps)[:1],
                                   *relighting.chunk_inputs(rays, maps)[1], torch.ones(3, device=DEV),
                                   torch.rand(n, 16, 2, generator=torch.Generator(DEV).manual_seed(12), device=DEV,
                                              dtype=torch.float64), 0.5, 'nerv')
    some = (hits["hit"] >= 0).any(1)
    assert torch.equal(wo[:, ~some], fwo[:, ~some]) and torch.equal(wb[:, ~some], fwb[:, ~some])
    assert (wo >= fwo).all() and (wb >= fwb).all()
    assert (wo[:, some] > fwo[:, some]).any()
    # and that direct term is relight_chunk_fused's up to the march's last bits
    rwb, rwo = relighting.relight_chunk_fused(lego, light, names, rays, maps, 1.0, u)
    assert (rwo - fwo).abs().max() < 1e-4 and (rwb - fwb).abs().max() < 1e-4


def test_convex_object_gets_little_indirect_light(env):
    """One box: every secondary ray leaves the object, so the indirect term is bounded by what the float64 march
    lets through the box's own surface (its density tail), far below the direct term."""
    from tensoir_b200 import synthetic
    names, light, hdr = env
    model = make_lego_model(128, DEV)
    model.normals_kind = "purely_derived"        # outward normals: the secondary rays leave a convex object
    box = [((-0.6, -0.6, -0.6), (0.6, 0.6, 0.6), 0)]
    planes, lines = synthetic.box_density_factors(model.gridSize.tolist(), model.aabb.cpu(), boxes=box)
    with torch.no_grad():
        for k in range(3):
            model.density_plane[k].copy_(planes[k].to(DEV))
            model.density_line[k].copy_(lines[k].to(DEV))
    model.updateAlphaMask((128, 128, 128))
    ops.device_field(model).refresh(model, force=True)
    rays, maps = lego_chunk(model, seed=5)
    L, n = len(names), rays.shape[0]
    u = torch.rand(L, n, 512, device=DEV, dtype=torch.float64, generator=torch.Generator(DEV).manual_seed(1))
    ind = torch.zeros(L, n, 3, device=DEV)
    fwb, fwo = relighting.relight_chunk_fused(model, light, names, rays, maps, 1.0, u)
    indirect.relight_chunk_indirect(model, light, names, rays, maps, 1.0, u, torch.Generator(DEV).manual_seed(2),
                                    indirect_samples=16, indirect_out=ind)
    hit = maps[5].reshape(-1) > 0.5
    assert hit.sum() > 200
    # float64: the largest occlusion a secondary ray of this box sees
    rays_c, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(rays, maps)
    hits = indirect.secondary_hits(model, rays_c, depth, normal, albedo, rough, fresnel, acc, torch.ones(3, device=DEV),
                                   torch.rand(n, 16, 2, device=DEV, dtype=torch.float64,
                                              generator=torch.Generator(DEV).manual_seed(2)), 0.5, 'nerv')
    sel = torch.randperm(hits["list_o"].shape[0], generator=torch.Generator().manual_seed(1))[:1024].to(DEV)
    T64, _, _ = march64(model, hits["list_o"][sel], hits["list_d"][sel])
    w_mean = float((1 - T64).mean())
    assert w_mean < 0.1, w_mean                              # a convex object: most secondary rays leave it
    # the indirect term is E[T w Lo] <= E[T] E[w] max Lo, with E[T] (the directional albedo) <= 1 and Lo of the order
    # of the primary point's direct light: bounded by a few times E[w] of the direct term (linear, through the sRGB
    # inverse of the written maps)
    x = fwo[:, hit].double()
    direct = torch.where(x <= 0.04045, x / 12.92, ((x + 0.055) / 1.055) ** 2.4)
    ratio = float(ind[:, hit].double().mean() / direct.mean())
    assert ratio <= 4 * w_mean + 1e-6, (ratio, w_mean)


def test_relight_end_to_end_with_indirect(lego, tmp_path):
    from types import SimpleNamespace
    names = [f"m{k}" for k in range(_lib.RELIGHT_MAX_LIGHTS + 1)]
    g = np.random.default_rng(3)
    hdr = {k: g.uniform(0.1, 2.0, (8, 16, 3)).astype(np.float32) for k in names}
    ds = SyntheticViews(hemisphere_poses(1), 48, 48, light_names=names)
    base = dict(hdrdir=hdr, batch_size=1024, render_video=False)
    torch.manual_seed(0)
    relighting.relight(ds, SimpleNamespace(geo_buffer_path=str(tmp_path / "a"), **base), lego,
                       rescale_value=[1.0, 1.0, 1.0])
    torch.manual_seed(0)
    relighting.relight(ds, SimpleNamespace(geo_buffer_path=str(tmp_path / "b"), indirect_samples=8,
                                           indirect_light_samples=16, save_indirect=1, **base), lego,
                       rescale_value=[1.0, 1.0, 1.0])
    va, vb = tmp_path / "a" / "test_000", tmp_path / "b" / "test_000"
    assert sorted(p.name for p in (vb / "relighting_indirect").iterdir()) == sorted(f"{k}.hdr" for k in names)
    img = read_hdr(str(vb / "relighting_indirect" / "m3.hdr"))
    assert img.shape == (48, 48, 3) and np.isfinite(img).all() and img.max() > 0
    assert not (va / "relighting_indirect").exists()
    with torch.no_grad():
        acc = lego(ds[0]["rays"].to(DEV), torch.zeros(48 * 48, 1, dtype=torch.int32, device=DEV), is_train=False,
                   white_bg=True, ndc_ray=False, N_samples=-1)[6].reshape(48, 48).cpu().numpy()
    miss = acc < 0.4
    assert miss.any() and (~miss).any()
    for sub in ("relighting_with_bg", "relighting_without_bg"):
        for k in names:
            a, b = relighting._imread(str(va / sub / f"{k}.png")), relighting._imread(str(vb / sub / f"{k}.png"))
            assert np.array_equal(a[miss], b[miss])
            assert (b[acc > 0.6].astype(int) >= a[acc > 0.6].astype(int) - 1).all()
    lines = (vb / "relighting_without_bg" / "relight_psnr.txt").read_text().splitlines()
    assert len(lines) == len(names) and all(ln.startswith(f"{k}: PNSR ") for ln, k in zip(lines, names))
    assert (tmp_path / "b" / "relight_psnr.txt").read_text().count("PSNR") == len(names)
