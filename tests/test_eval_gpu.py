"""Test-view evaluation on the H100: the metric kernel (csrc/tir_eval.cu) against the fixture recorded from the reference
(tests/golden/eval_reference.pt, written by tests/golden/make_eval_golden.py) and against the oracle at full size; the
three evaluation loops end to end against the reference's returned metrics, metrics_record.txt and written images."""
import os
import re
import sys
import types

import cv2
import numpy as np
import pytest
import torch

from gpu_helpers import load_fixture, model_from_fixture, renderer_args
from oracle import eval_oracle as EO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def fx():
    import __graft_entry__ as g
    g.build()
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "eval_reference.pt"), weights_only=False)


def _views(fx, n_lights=1):
    from tensoir_b200.synthetic import SyntheticViews
    return SyntheticViews(fx["poses"], fx["H"], fx["W"], n_lights=n_lights)


def _kernel_view(H, W, maps, item, ratio=None, ssim=True):
    from tensoir_b200.evaluation import view_metrics
    d = lambda t: t.to(DEV)  # noqa: E731
    gt_rgb, gt_alb, mask = d(item["rgbs"][0]), d(item["albedo"]), d(item["rgbs_mask"]).reshape(-1)
    alb = d(maps["albedo_map"])
    if ratio is None:
        s, t = EO.view_ratios(alb, gt_alb, mask)
        ratio = torch.cat([s.reshape(1), t])
    return view_metrics(H, W, d(maps["rgb_map"]), d(maps["rgb_with_brdf_map"]), gt_rgb, alb, gt_alb, mask, ratio,
                        d(maps["normal_map"]), d(item["normals"]), ssim=ssim)


def test_kernel_on_recorded_maps(fx):
    H, W = fx["H"], fx["W"]
    ds = _views(fx)
    outs = [_kernel_view(H, W, m, ds[v])[0].cpu() for v, m in enumerate(fx["runs"]["full"]["maps"])]
    o = torch.stack(outs).numpy()
    n = H * W
    psnr = np.mean(-10 * np.log10(o[:, 0] / (n * 3)))
    psnr_b = np.mean(-10 * np.log10(o[:, 1] / (n * 3)))
    mae = o[:, 4].sum() / (len(outs) * n)
    ps = -10 * np.log10(o[:, 2].sum() / (len(outs) * n * 3))
    pt = -10 * np.log10(o[:, 3].sum() / (len(outs) * n * 3))
    want = fx["runs"]["full"]["returned"]
    for got, ref, tol in zip((psnr, psnr_b, mae, ps, pt), want, (1e-4, 1e-4, 1e-3, 1e-4, 1e-4)):
        assert abs(got - ref) < tol, (got, ref)
    ssim_ref = np.asarray(fx["runs"]["full_extra"]["ssim"]).reshape(len(outs), 4)
    assert np.abs(o[:, 5:9] - ssim_ref).max() < 1e-10


def test_kernel_ssim_on_recorded_pairs(fx):
    from tensoir_b200.evaluation import view_metrics
    for a, b, want in fx["ssim_pairs"]:
        H, W = a.shape[:2]
        out, _, _ = view_metrics(H, W, a.to(DEV), a.to(DEV), b.to(DEV))
        assert abs(float(out[5]) - want) < 1e-10


@pytest.mark.parametrize("H,W", [(800, 800), (801, 797), (11, 300)])
def test_kernel_matches_oracle_full_size(H, W):
    import test_eval_cpu as T
    for kind in ("random", "clip"):
        d = T.make_view(H, W, kind, seed=H + W)
        s, t = EO.view_ratios(d["albedo"], d["gt_albedo"], d["gt_mask"])
        ratio = torch.cat([s.reshape(1), t])
        from tensoir_b200.evaluation import view_metrics
        args = [d[k].to(DEV) for k in ("rgb", "rgb_brdf", "gt_rgb", "albedo", "gt_albedo", "gt_mask")]
        out, al1, al3 = view_metrics(H, W, *args, ratio.to(DEV), d["normal"].to(DEV), d["gt_normal"].to(DEV))
        out2, al1b, _ = view_metrics(H, W, *args, ratio.to(DEV), d["normal"].to(DEV), d["gt_normal"].to(DEV))
        assert torch.equal(out, out2) and torch.equal(al1, al1b)             # fixed-order reductions
        want = EO.view_metrics(H, W, d["rgb"], d["rgb_brdf"], d["gt_rgb"], d["albedo"], d["gt_albedo"], d["gt_mask"],
                               s, t, d["normal"], d["gt_normal"])
        assert torch.equal(al1.cpu().reshape(H, W, 3), want["aligned_single"])
        assert torch.equal(al3.cpu().reshape(H, W, 3), want["aligned_three"])
        o = out.cpu().tolist()
        # the fp32 powf / acosf of CUDA and numpy differ by an ulp on part of the inputs
        for k, (key, rel) in enumerate((("sse_rgb", 1e-9), ("sse_rgb_brdf", 1e-9), ("gse_single", 1e-6),
                                        ("gse_three", 1e-6), ("angle_sum", 1e-6))):
            assert o[k] == pytest.approx(want[key], rel=rel, abs=1e-9), (kind, key)
        for k, key in enumerate(("ssim_rgb", "ssim_rgb_brdf", "ssim_albedo_single", "ssim_albedo_three")):
            assert abs(o[5 + k] - want[key]) < 1e-12, (kind, key)


def _args(fx):
    a = renderer_args(24)
    a.N_vis, a.batch_size_test, a.relight_chunk_size = fx["N_vis"], fx["batch_size_test"], 160000
    return a


def _read(path):
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    return img[..., ::-1] if img.ndim == 3 else img


class _ConstLpips:
    """Stands in for lpips.LPIPS: a module returning a constant distance; records the constructor arguments."""

    def __init__(self, value):
        self.value, self.calls = value, []

    def __call__(self, net, version):
        self.calls.append((net, version))
        value = self.value

        class Net(torch.nn.Module):
            def forward(self, a, b, normalize=False):
                assert normalize and a.shape == b.shape and a.shape[0] == 3
                return torch.tensor(value)
        return Net()


@pytest.mark.parametrize("name", ["full", "full_all", "full_extra", "simple", "general"])
def test_loops_match_reference(fx, name, tmp_path, monkeypatch):
    import tensoir_b200.evaluation as E
    # the recording stood in 0.0 for LPIPS (no weights): the same stand-in here
    monkeypatch.setitem(sys.modules, "lpips", types.SimpleNamespace(LPIPS=_ConstLpips(0.0)))
    monkeypatch.setattr(E, "_LPIPS", {})
    from tensoir_b200 import Renderer_TensoIR_train
    rec = fx["runs"][name]
    model = model_from_fixture(load_fixture(rec["model"]), DEV)
    ds = _views(fx, rec["n_lights"])
    fn = {"full": E.evaluation_iter_TensoIR, "simple": E.evaluation_iter_TensoIR_simple,
          "general": E.evaluation_iter_TensoIR_general_multi_lights}[name.split("_")[0]]
    save = str(tmp_path / name)
    got = fn(ds, model, _args(fx), Renderer_TensoIR_train, savePath=save, prtx='7_', N_samples=-1, white_bg=True,
             device=DEV, **rec["kwargs"])
    assert len(got) == len(rec["returned"])
    tols = (0.02, 0.02, 0.05, 0.05, 0.05)
    for g, r, tol in zip(got, rec["returned"], tols):
        assert abs(g - r) < tol, (name, got, rec["returned"])
    if name == "full_all":
        s, t = E.compute_rescale_ratio(model, ds, sampled_num=20)
        rs, rt = fx["rescale_ratio"]
        assert abs(float(s) / float(rs) - 1) < 1e-3
        assert torch.allclose(t.cpu(), rt, rtol=1e-3)
    # metrics_record.txt: the same lines, numbers equal up to one unit of the last printed digit
    lines, want = open(os.path.join(save, "metrics_record.txt")).read().splitlines(), rec["metrics_record"].splitlines()
    assert len(lines) == len(want)
    num = r"-?\d+\.\d+"
    for a, b in zip(lines, want):
        assert re.sub(num, "#", a) == re.sub(num, "#", b), (a, b)
        for x, y in zip(re.findall(num, a), re.findall(num, b)):
            assert abs(float(x) - float(y)) <= 10.0 ** -len(y.split(".")[1]) + 1e-9, (a, b)
    # written files: same set, same shapes; >= 99 % of the pixels within 1 LSB
    written = sorted(os.path.relpath(os.path.join(d, f), save) for d, _, fs in os.walk(save) for f in fs
                     if f.endswith(".png"))
    assert written == sorted(p for p, _ in rec["writes"])
    for path, ref in rec["writes"]:
        img = _read(os.path.join(save, path))
        shape = tuple(ref) if isinstance(ref, (tuple, torch.Size)) else ref.shape
        assert img.shape == tuple(shape), path
        if isinstance(ref, np.ndarray):
            close = np.abs(img.astype(np.int32) - ref.astype(np.int32)) <= 1
            assert close.mean() >= 0.99, (path, close.mean())


def test_lpips_plumbing(fx, tmp_path, monkeypatch):
    import tensoir_b200.evaluation as E
    from tensoir_b200 import Renderer_TensoIR_train
    stub = _ConstLpips(0.125)
    monkeypatch.setitem(sys.modules, "lpips", types.SimpleNamespace(LPIPS=stub))
    monkeypatch.setattr(E, "_LPIPS", {})
    model = model_from_fixture(load_fixture("rotated_g24.pt"), DEV)
    save = str(tmp_path / "lp")
    E.evaluation_iter_TensoIR(_views(fx), model, _args(fx), Renderer_TensoIR_train, savePath=save, prtx='1_',
                              white_bg=True, device=DEV)
    assert sorted(stub.calls) == [("alex", "0.1"), ("vgg", "0.1")]
    txt = open(os.path.join(save, "metrics_record.txt")).read()
    assert txt.count("0.1250") == 8 and "nan" not in txt
