"""Test-view evaluation on the CPU.

The metric kernel's entry points are built for the host (tests/host_eval.cpp: the same C ABI, argument checks and
per-pixel / per-window math of csrc/tir_eval_body.h, loops instead of kernels) and driven through the real ctypes
wrapper tensoir_b200.evaluation.view_metrics; they must agree with the restated reference (oracle/eval_oracle.py).
Also: the struct mirror, the NULL / zero-size conventions, the drop-in renderer's evaluation names and the
SyntheticViews item contract."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from oracle import eval_oracle as EO
from tensoir_b200 import _lib, evaluation

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_eval"), "host_eval.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


def make_view(H, W, kind, seed):
    g = torch.Generator().manual_seed(seed)
    n = H * W
    r = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    if kind == "random":
        d = dict(rgb=r(n, 3) * 1.2 - 0.1, rgb_brdf=r(n, 3) * 1.2 - 0.1, gt_rgb=r(n, 3), albedo=r(n, 3),
                 gt_albedo=r(n, 3), gt_mask=r(n) > 0.3, normal=torch.randn(n, 3, generator=g),
                 gt_normal=torch.randn(n, 3, generator=g))
    else:
        # clip cases: constant patches (zero variance -> the sigma clip rules), exact zeros, saturated maps,
        # parallel / anti-parallel / zero normals
        rgb = torch.full((n, 3), 0.5)
        rgb[: n // 3] = 1.7
        rgb[n // 3: n // 2] = -0.2
        gt = torch.full((n, 3), 0.5)
        gt[n // 4: n // 2] = r(n // 2 - n // 4, 3)
        normal = torch.tensor([0.0, 0.0, 1.0]).repeat(n, 1)
        gtn = normal.clone()
        gtn[: n // 5] *= -1
        normal[n // 5: n // 4] = 0.0
        alb = torch.full((n, 3), 0.25)
        alb[::7] = 0.0
        d = dict(rgb=rgb, rgb_brdf=gt.clone(), gt_rgb=gt, albedo=alb, gt_albedo=torch.full((n, 3), 0.6),
                 gt_mask=torch.arange(n) % 3 != 0, normal=normal, gt_normal=gtn)
    return d


def _compare(H, W, d):
    s, t = EO.view_ratios(d["albedo"], d["gt_albedo"], d["gt_mask"])
    ratio = torch.cat([s.reshape(1), t])
    out, al1, al3 = evaluation.view_metrics(H, W, d["rgb"], d["rgb_brdf"], d["gt_rgb"], d["albedo"], d["gt_albedo"],
                                            d["gt_mask"], ratio, d["normal"], d["gt_normal"])
    want = EO.view_metrics(H, W, d["rgb"], d["rgb_brdf"], d["gt_rgb"], d["albedo"], d["gt_albedo"], d["gt_mask"], s, t,
                           d["normal"], d["gt_normal"])
    assert torch.equal(al1.reshape(H, W, 3), want["aligned_single"])
    assert torch.equal(al3.reshape(H, W, 3), want["aligned_three"])
    o = out.tolist()
    # numpy's own float32 power and arccos differ from libm's / CUDA's powf and acosf by 1 ulp on a good share of the
    # inputs (about 1/5 for the power): the gamma and angle sums agree to 1e-6 relative, the squared errors to 1e-9
    for k, (key, rel) in enumerate((("sse_rgb", 1e-9), ("sse_rgb_brdf", 1e-9), ("gse_single", 1e-6),
                                    ("gse_three", 1e-6), ("angle_sum", 1e-6))):
        assert o[k] == pytest.approx(want[key], rel=rel, abs=1e-9), key
    for k, key in enumerate(("ssim_rgb", "ssim_rgb_brdf", "ssim_albedo_single", "ssim_albedo_three")):
        assert abs(o[5 + k] - want[key]) < 1e-12, (key, o[5 + k], want[key])


@pytest.mark.parametrize("H,W", [(37, 53), (11, 40), (64, 64)])
@pytest.mark.parametrize("kind", ["random", "clip"])
def test_host_kernel_matches_oracle(host_lib, H, W, kind):
    _compare(H, W, make_view(H, W, kind, seed=H * 100 + W))


def test_host_kernel_without_optional_terms(host_lib):
    H, W = 13, 17
    d = make_view(H, W, "random", 5)
    out, al1, al3 = evaluation.view_metrics(H, W, d["rgb"], d["rgb_brdf"], d["gt_rgb"])
    want = EO.view_metrics(H, W, d["rgb"], d["rgb_brdf"], d["gt_rgb"])
    assert al1 is None and al3 is None
    o = out.tolist()
    assert o[0] == pytest.approx(want["sse_rgb"], rel=1e-9) and o[1] == pytest.approx(want["sse_rgb_brdf"], rel=1e-9)
    assert o[2:5] == [0.0, 0.0, 0.0] and o[7:9] == [0.0, 0.0]
    assert abs(o[5] - want["ssim_rgb"]) < 1e-12 and abs(o[6] - want["ssim_rgb_brdf"]) < 1e-12
    out, _, _ = evaluation.view_metrics(H, W, d["rgb"], d["rgb_brdf"], d["gt_rgb"], ssim=False)
    assert out.tolist()[5:] == [0.0] * 4


def test_eval_struct_size_matches_the_c_compiler(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "tensoir_b200.h"\n'
                   'int main(void){printf("%zu\\n",sizeof(TirEvalView));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)], check=True)
    got = int(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout)
    assert got == C.sizeof(_lib.TirEvalView)


def test_eval_null_and_empty(host_so):
    lib = host_so
    out = (C.c_double * 9)()
    work = (C.c_double * 4096)()
    assert lib.tir_eval_view(None, work, 4096, out, None) == -1
    v = _lib.TirEvalView(H=0, W=7)
    assert lib.tir_eval_view(C.byref(v), None, 0, None, None) == 0           # zero pixels: no-op
    v = _lib.TirEvalView(H=12, W=12)
    assert lib.tir_eval_view(C.byref(v), work, 4096, out, None) == -1          # no rgb
    buf = (C.c_float * (12 * 12 * 3))()
    v.rgb = v.rgb_brdf = v.gt_rgb = C.cast(buf, C.c_void_p)
    v.albedo = C.cast(buf, C.c_void_p)
    assert lib.tir_eval_view(C.byref(v), work, 4096, out, None) == -1          # albedo without gt_albedo
    v.albedo = None
    assert lib.tir_eval_view(C.byref(v), work, 1, out, None) == -4             # work too small
    v.ssim, v.H = 1, 10
    assert lib.tir_eval_view(C.byref(v), work, 4096, out, None) == -2          # SSIM needs 11x11
    n = C.c_int64(0)
    assert lib.tir_eval_work_size(12, 12, None) == -1
    assert lib.tir_eval_work_size(12, 12, C.byref(n)) == 0 and n.value > 0


def test_eval_rejects_small_images():
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    import types
    ds = SyntheticViews(hemisphere_poses(1), 10, 16)
    args = types.SimpleNamespace(N_vis=1, batch_size_test=64, relight_chunk_size=64)
    with pytest.raises(ValueError):
        evaluation.evaluation_iter_TensoIR_simple(ds, None, args, None, savePath=None)


def test_dropin_renderer_exports_native_evaluation():
    code = ("import renderer, tensoir_b200.evaluation as E\n"
            "for n in ('evaluation_iter_TensoIR', 'evaluation_iter_TensoIR_simple',\n"
            "          'evaluation_iter_TensoIR_general_multi_lights', 'compute_rescale_ratio'):\n"
            "    assert getattr(renderer, n) is getattr(E, n), n\n"
            "assert renderer.__file__.startswith(%r)\n" % os.path.join(REPO, "dropin"))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(REPO, "dropin"), REPO]))
    subprocess.run([sys.executable, "-c", code], check=True, env=env, cwd=REPO)


def test_synthetic_views_item_contract():
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    H, W, L = 24, 32, 2
    ds = SyntheticViews(hemisphere_poses(3), H, W, n_lights=L)
    assert len(ds) == 3 and ds.img_wh == (W, H) and ds.near_far == [2.0, 6.0] and ds.white_bg
    assert ds.lights_probes is None
    it = ds[1]
    shapes = {"rays": ((H * W, 6), torch.float32), "rgbs": ((L, H * W, 3), torch.float32),
              "light_idx": ((L, H * W, 1), torch.int32), "rgbs_mask": ((H * W, 1), torch.bool),
              "albedo": ((H * W, 3), torch.float32), "normals": ((H * W, 3), torch.float32),
              "c2w": ((4, 4), torch.float32), "w2c": ((4, 4), torch.float32)}
    for k, (shape, dtype) in shapes.items():
        assert tuple(it[k].shape) == shape and it[k].dtype == dtype, k
    m = it["rgbs_mask"][:, 0]
    assert 0 < m.sum() < H * W
    assert torch.equal(it["normals"][~m], torch.tensor([0.0, 0.0, 1.0]).expand(int((~m).sum()), 3))
    assert torch.allclose(it["normals"].norm(dim=-1), torch.ones(H * W))
    assert torch.equal(it["rgbs"][:, ~m], torch.ones(L, int((~m).sum()), 3))
    assert torch.equal(it["light_idx"][1], torch.ones(H * W, 1, dtype=torch.int32))
    assert torch.equal(ds[1]["rgbs"], it["rgbs"])                                   # deterministic
    assert np.isclose(float(torch.linalg.det(it["c2w"][:3, :3])), 1.0, atol=1e-5)
