"""Relighting evaluation on the H100: the fused chunk (csrc/tir_relight.cu around the density march) against the eager
relight_chunk and the fixture recorded from the reference (tests/golden/rotated_g24.pt), its edge cases, the pair-metric
kernel against utils.rgb_ssim, and relight() end to end against the eager chunk body on the same draws."""
import os
import re

import cv2
import numpy as np
import pytest
import torch

from gpu_helpers import load_fixture, model_from_fixture
from oracle import eval_oracle as EO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4


@pytest.fixture(scope="module")
def fx():
    import __graft_entry__ as g
    g.build()
    return load_fixture("rotated_g24.pt")


def _midpoints(cdf, idx):
    lo = torch.cat([torch.zeros(1, dtype=torch.float64, device=cdf.device), cdf])[idx]
    return (lo + cdf[idx]) / 2


def _setup(fx, names=("sunny",)):
    from tensoir_b200.relight import Environment_Light
    rgb = fx["env_rgb"].numpy()
    maps = {"sunny": rgb, "dim": rgb[:, ::-1].copy() * 0.4}
    env = Environment_Light({n: maps[n] for n in names}, device=DEV)
    m = model_from_fixture(fx, DEV)
    return m, env, tuple(t.to(DEV) for t in fx["relight_maps"]), fx["rays"].to(DEV)


@pytest.mark.parametrize("vis_equation", ["nerv", "nerfactor"])
def test_fused_chunk_matches_eager_and_reference(fx, vis_equation):
    from tensoir_b200.relight import relight_chunk
    from tensoir_b200.relighting import relight_chunk_fused
    m, env, maps, rays = _setup(fx)
    idx = fx["relight_idx"].to(DEV)
    acc = maps[5]
    u = torch.full((1, rays.shape[0], idx.shape[1]), 0.5, dtype=torch.float64, device=DEV)
    u[0, acc > 0.5] = _midpoints(env._cdf["sunny"], idx)
    w, wo = relight_chunk_fused(m, env, ["sunny"], rays, maps, 1.7, u, 64, vis_equation=vis_equation)
    ew, ewo = relight_chunk(m, env, "sunny", rays, maps, 1.7, idx, 64, vis_equation=vis_equation)
    assert (wo[0] - ewo).abs().max() < TOL and (w[0] - ew).abs().max() < TOL
    if vis_equation == "nerv":
        assert (wo[0].cpu() - fx["relight_without_bg"]).abs().max() < TOL
        assert (w[0].cpu() - fx["relight_with_bg"]).abs().max() < TOL
    w2, wo2 = relight_chunk_fused(m, env, ["sunny"], rays, maps, 1.7, u, 64, vis_equation=vis_equation)
    assert torch.equal(w, w2) and torch.equal(wo, wo2)                  # fixed-order sums: bit-identical reruns


def _eager_all(m, env, names, rays, maps, rescale, u, S, **kw):
    from tensoir_b200.relight import relight_chunk
    acc = maps[5]
    out = []
    for k, name in enumerate(names):
        cdf = env._cdf[name]
        idx = torch.searchsorted(cdf, u[k][acc > kw.get("acc_mask_threshold", 0.5)], right=True)
        idx = idx.clamp_(max=cdf.numel() - 1)
        out.append(relight_chunk(m, env, name, rays, maps, rescale, idx, S, **kw))
    return torch.stack([o[0] for o in out]), torch.stack([o[1] for o in out])


@pytest.mark.parametrize("case", ["no_hits", "all_cosines_masked", "odd_rows"])
def test_fused_chunk_edge_cases(fx, case):
    from tensoir_b200.relighting import relight_chunk_fused
    names = ["sunny", "dim"]
    m, env, maps, rays = _setup(fx, names)
    depth, normal, albedo, rough, fresnel, acc = maps
    if case == "no_hits":
        acc = torch.zeros_like(acc)
    elif case == "all_cosines_masked":
        normal = torch.zeros_like(normal)
    else:
        n = 37                                               # not a multiple of any block size
        rays, depth, normal, albedo, rough, fresnel, acc = (t[:n] for t in (rays, depth, normal, albedo, rough,
                                                                            fresnel, acc))
    maps = (depth, normal, albedo, rough, fresnel, acc)
    S = 96
    u = torch.rand(2, rays.shape[0], S, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(5))
    rescale = torch.tensor([1.2, 0.9, 1.1], device=DEV)
    w, wo = relight_chunk_fused(m, env, names, rays, maps, rescale, u, S)
    ew, ewo = _eager_all(m, env, names, rays, maps, rescale, u, S)
    assert (wo - ewo).abs().max() < TOL and (w - ew).abs().max() < TOL
    if case == "no_hits":
        assert torch.equal(wo, torch.ones_like(wo))
    if case == "all_cosines_masked":
        hit = acc > 0.5
        assert bool(hit.any()) and torch.equal(wo[:, hit], torch.zeros_like(wo[:, hit]))


@pytest.mark.parametrize("H,W", [(800, 800), (801, 797), (11, 300)])
def test_eval_pairs_matches_rgb_ssim_and_eval_view(H, W):
    from tensoir_b200.evaluation import view_metrics
    from tensoir_b200.relighting import pair_metrics
    g = torch.Generator().manual_seed(H + W)
    a = torch.rand(3, H, W, 3, generator=g)
    b = torch.rand(3, H, W, 3, generator=g)
    b[1] = (a[1] + 0.05 * torch.rand(H, W, 3, generator=g)).clamp(0, 1)
    a[2, : H // 2] = 0.5
    out = pair_metrics(a.to(DEV), b.to(DEV), H, W)
    out2 = pair_metrics(a.to(DEV), b.to(DEV), H, W)
    assert torch.equal(out, out2)
    o = out.cpu()
    for p in range(3):
        assert float(o[p, 0]) == pytest.approx(float((a[p] - b[p]).pow(2).double().sum()), rel=1e-9)
        if H * W < 300_000 or p == 0:
            assert abs(float(o[p, 1]) - EO.rgb_ssim(a[p].numpy(), b[p].numpy(), 1)) < 1e-12
        v, _, _ = view_metrics(H, W, a[p].to(DEV), a[p].to(DEV), b[p].to(DEV))
        assert float(v[5]) == float(o[p, 1])                                  # the same bits as tir_eval_view


def _read(path):
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img.ndim == 3:
        img = img[..., [2, 1, 0, 3]] if img.shape[2] == 4 else img[..., ::-1]
    return img


def test_relight_end_to_end(fx, tmp_path, monkeypatch):
    """relight() on two 32x24 synthetic views with two maps, batch_size 300 (three chunks per view): the written files,
    text formats and metrics against the eager chunk body on the same draws and the oracle's rgb_ssim."""
    import types
    import tensoir_b200.relighting as R
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    names = ["sunny", "dim"]
    m, env, _, _ = _setup(fx, names)
    rgb = fx["env_rgb"].numpy()
    hdr = {"sunny": rgb, "dim": rgb[:, ::-1].copy() * 0.4}
    H, W = 24, 32
    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=names)
    draws = []
    gen = torch.Generator(DEV).manual_seed(9)

    def uniforms(L, n, S, device):
        u = torch.rand(L, n, S, dtype=torch.float64, device=device, generator=gen)
        draws.append(u.clone())
        return u
    monkeypatch.setattr(R, "_uniforms", uniforms)
    out = tmp_path / "relight"
    args = types.SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(out), batch_size=300)
    R.relight(ds, args, tensoIR=m)
    n_chunks = -(-H * W // 300)
    assert len(draws) == len(ds) * n_chunks
    files = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)
    want = ["relight_psnr.txt"]
    for v in range(len(ds)):
        want += [f"test_{v:03d}/{f}" for f in ("acc.png", "albedo.png", "albedo_gamma_corrected.png",
                                               "gt_albedo_gamma_corrected.png", "normal.png", "roughness.png",
                                               "relighting_without_bg/relight_psnr.txt")]
        want += [f"test_{v:03d}/relighting_{s}/{n}.png" for s in ("with_bg", "without_bg") for n in names]
    assert [f for f in files if not f.endswith(".mp4")] == sorted(want)
    rescale = R.compute_rescale_ratio(m, ds)[1].to(DEV)
    psnrs = {n: [] for n in names}
    for v in range(len(ds)):
        item = ds[v]
        rays = item["rays"].to(DEV)
        li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=DEV)
        ew, ewo, accs = [], [], []
        for c, s in enumerate(range(0, rays.shape[0], 300)):
            r = rays[s:s + 300]
            _, depth, normal, albedo, rough, fresnel, acc, *_ = m(r, li[s:s + 300], is_train=False, white_bg=True,
                                                                  ndc_ray=False, N_samples=-1)
            w, wo = _eager_all(m, env, names, r, (depth, normal, albedo, rough, fresnel, acc), rescale,
                               draws[v * n_chunks + c], 512)
            ew.append(w), ewo.append(wo), accs.append(acc)
        ew, ewo, acc = torch.cat(ew, 1), torch.cat(ewo, 1), torch.cat(accs).detach()
        d = out / f"test_{v:03d}"
        hit = (acc > 0.5).reshape(-1)
        for k, n in enumerate(names):
            for sub, ref in (("without_bg", ewo[k]), ("with_bg", ew[k])):
                img = _read(str(d / f"relighting_{sub}" / f"{n}.png")).reshape(-1, 3).astype(np.int32)
                want_u8 = (ref.cpu().numpy() * 255).astype(np.uint8).astype(np.int32)
                diff = np.abs(img - want_u8)
                assert diff.max() <= 1 and (diff > 0).mean() <= 0.01, (sub, n, (diff > 0).mean())
            gt = item["rgbs"][k].reshape(H, W, 3).numpy()
            pred = ewo[k].reshape(H, W, 3).cpu().numpy()
            psnrs[n].append((-10.0 * np.log(np.mean((pred - gt) ** 2)) / np.log(10.0),
                             EO.rgb_ssim(pred, gt, 1)))
        acc_img = _read(str(d / "acc.png"))
        acc_t = acc.clone()
        acc_t[acc_t <= 0.9] = 0.0
        assert np.array_equal(acc_img, (acc_t.reshape(H, W).cpu().numpy() * 255).astype(np.uint8))
        alb = _read(str(d / "albedo.png"))
        assert alb.shape == (H, W, 4) and np.array_equal(alb[..., 3], acc_img)
        lines = open(d / "relighting_without_bg" / "relight_psnr.txt").read().splitlines()
        assert len(lines) == len(names)
        for k, (n, line) in enumerate(zip(names, lines)):
            mt = re.fullmatch(rf"{n}: PNSR (\S+); SSIM (\S+); L_Alex \S+; L_VGG \S+", line)
            assert mt, line
            assert abs(float(mt.group(1)) - psnrs[n][v][0]) < 1e-3 and abs(float(mt.group(2)) - psnrs[n][v][1]) < 1e-4
    lines = open(out / "relight_psnr.txt").read().splitlines()
    for n, line in zip(names, lines):
        mt = re.fullmatch(rf"{n}:  PSNR (\S+); SSIM (\S+); L_Alex \S+; L_VGG \S+", line)
        assert mt, line
        assert abs(float(mt.group(1)) - np.mean([p[0] for p in psnrs[n]])) < 1e-3
        assert abs(float(mt.group(2)) - np.mean([p[1] for p in psnrs[n]])) < 1e-4


def test_relight_matches_reference_recording(fx, tmp_path, monkeypatch):
    """relight() against the reference's own relight() (tests/golden/relight_reference.pt, written by
    tests/golden/make_relight_golden.py): the recorded multinomial draws are replayed through _uniforms at bin midpoints,
    the hit masks must be exact, every written PNG equal to the reference's array up to 1 LSB on a small fraction of
    values, the per-view and overall relight_psnr.txt the same lines with PSNR / SSIM within 1e-3 dB / 1e-4."""
    import lzma
    import sys
    import types
    import tensoir_b200.relighting as R
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    ref = torch.load(os.path.join(os.path.dirname(__file__), "golden", "relight_reference.pt"), weights_only=False)
    names, H, W, B = ref["light_names"], ref["H"], ref["W"], ref["batch_size"]
    L = len(names)
    idx = torch.from_numpy(np.frombuffer(lzma.decompress(ref["draws_int16_xz"]), np.int16).astype(np.int64))
    draws, o = [], 0
    for shp in ref["draw_shapes"]:
        n = int(np.prod(shp))
        draws.append(idx[o:o + n].reshape(shp))
        o += n
    hdrdir = tmp_path / "hdr"
    hdrdir.mkdir()
    for name, arr in ref["hdr"].items():
        cv2.imwrite(str(hdrdir / f"{name}.hdr"), np.ascontiguousarray(arr[..., ::-1]))
    model = model_from_fixture(fx, DEV)
    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=names)
    n_chunks = -(-H * W // B)
    hits = [(a > 0.5).to(DEV) for a in ref["acc"]]
    calls = []
    from tensoir_b200.relight import read_hdr
    cdfs = {}
    for name in names:
        from tensoir_b200.relight import Environment_Light
        cdfs[name] = Environment_Light({name: read_hdr(str(hdrdir / f"{name}.hdr"))}, device=DEV)._cdf[name]

    def uniforms(L_, n, S, device):
        c = len(calls)
        v, k = divmod(c, n_chunks)
        h = hits[v][k * B:k * B + n]
        u = torch.full((L_, n, S), 0.5, dtype=torch.float64, device=device)
        for li, name in enumerate(names):
            u[li, h] = _midpoints(cdfs[name], draws[c * L + li].to(device))
        calls.append(h)
        return u
    fused = R.relight_chunk_fused

    def checked(tensoIR, envir_light, light_names, rays, maps, *a, **k):
        assert torch.equal(maps[5].reshape(-1) > 0.5, calls[-1]), "hit mask differs from the reference's"
        return fused(tensoIR, envir_light, light_names, rays, maps, *a, **k)
    ratios = []
    crr = R.compute_rescale_ratio
    monkeypatch.setattr(R, "compute_rescale_ratio", lambda *a, **k: ratios.append(crr(*a, **k)) or ratios[-1])
    monkeypatch.setattr(R, "_uniforms", uniforms)
    monkeypatch.setattr(R, "relight_chunk_fused", checked)
    from test_eval_gpu import _ConstLpips
    monkeypatch.setitem(sys.modules, "lpips", types.SimpleNamespace(LPIPS=_ConstLpips(0.0)))
    import tensoir_b200.evaluation as E
    monkeypatch.setattr(E, "_LPIPS", {})
    out = tmp_path / "out"
    args = types.SimpleNamespace(hdrdir=str(hdrdir), geo_buffer_path=str(out), batch_size=B)
    R.relight(ds, args, tensoIR=model)
    assert len(calls) == len(ds) * n_chunks
    rs, rt = ref["rescale_ratio"]
    assert abs(float(ratios[0][0]) / float(rs) - 1) < 1e-3 and torch.allclose(ratios[0][1].cpu(), rt, rtol=1e-3)
    written = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs
                     if f.endswith(".png"))
    assert written == sorted(p for p, _ in ref["writes"])
    bad = []
    for path, want in ref["writes"]:
        got = _read(str(out / path)).reshape(want.shape).astype(np.int32)
        diff = np.abs(got - want.astype(np.int32))
        relit = path.split("/")[1].startswith("relighting")
        # the saved acc (acc.png, the alpha of the RGBA images) is the thresholded primary acc; inside the object it is
        # 1 - T with T ~ 0, i.e. exactly on the 255 step of (acc * 255).astype(uint8), where a 1-ulp difference of the
        # sum of weights flips 254 / 255.  Such flips are allowed only where the reference's acc is that close to a step.
        if path.endswith("acc.png") or want.shape[-1] == 4:
            a = ref["acc"][int(path[5:8])].reshape(H, W).double()
            a[a <= 0.9] = 0.0
            on_step = (a * 255 - torch.round(a * 255)).abs().numpy() < 1e-4
            d_acc = diff[..., -1]
            if d_acc.max() > 1 or bool(((d_acc > 0) & ~on_step).any()):
                bad.append((path, "acc", int(d_acc.max()), float((d_acc > 0).mean())))
            diff = diff[..., :3] if want.shape[-1] == 4 else np.zeros_like(diff)
        # fp32 reassociation (512-sample mean, device vs CPU primary render) moves a few values across a uint8 step
        frac = float((diff > 0).mean())
        if diff.max() > 1 or frac > (0.02 if relit else 0.01):
            bad.append((path, "rgb", int(diff.max()), frac))
    assert not bad, bad
    num = r"-?\d+\.\d+(?:e-?\d+)?"
    texts = [(out / f"test_{v:03d}" / "relighting_without_bg" / "relight_psnr.txt", ref["psnr_view"][v])
             for v in range(len(ds))] + [(out / "relight_psnr.txt", ref["psnr_all"])]
    for path, want in texts:
        got = open(path).read()
        assert re.sub(num, "#", got) == re.sub(num, "#", want), (got, want)
        for line_g, line_w in zip(got.splitlines(), want.splitlines()):
            g, w = [float(x) for x in re.findall(num, line_g)], [float(x) for x in re.findall(num, line_w)]
            assert abs(g[0] - w[0]) < 1e-3 and abs(g[1] - w[1]) < 1e-4 and g[2:] == w[2:], (line_g, line_w)
