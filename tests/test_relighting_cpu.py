"""Relighting evaluation on the CPU.

The relighting kernels' and tir_eval_pairs' entry points are built for the host (tests/host_relight.cpp: the same C ABI,
argument checks and per-sample / per-ray / per-window math of csrc/tir_relight_body.h and csrc/tir_eval_body.h, loops
instead of kernels) and driven through the real ctypes wrapper tensoir_b200.relighting; the density march on the
visibility list is the oracle's compute_transmittance.  They must agree with the restated reference
(oracle.tensoir_oracle.relight_chunk, oracle/eval_oracle.py) and with torch's searchsorted / grid_sample."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_host_lib, oracle_field, use_host
from oracle import eval_oracle as EO
from oracle import tensoir_oracle as O
from tensoir_b200 import _lib, relighting

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def oracle_march(f, rays_o, rays_d, *, table=None, counters=None, **kw):
    assert table.numel() == 96 and float(table[0]) == pytest.approx(0.05) and float(table[-1]) == pytest.approx(1.5)
    nerv, nerfactor = O.compute_transmittance(f, rays_o, rays_d, 96, 0.05, 1.5)
    return nerv, 1 - nerfactor, None


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_relight"), "host_relight.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so, oracle_march)
    return host_so


def midpoint_uniforms(cdf, idx):
    """u in the middle of bin idx of the CDF: searchsorted(cdf, u, right=True) gives idx back."""
    lo = torch.cat([torch.zeros(1, dtype=torch.float64), cdf])[idx]
    return (lo + cdf[idx]) / 2


def _golden_chunk(fx, vis_equation, idx=None):
    from tensoir_b200.relight import Environment_Light
    env = Environment_Light({"sunny": fx["env_rgb"].numpy()}, device='cpu')
    maps = fx["relight_maps"]
    acc = maps[5]
    idx = fx["relight_idx"] if idx is None else idx
    n, S = acc.shape[0], idx.shape[1]
    u = torch.full((1, n, S), 0.5, dtype=torch.float64)
    u[0, acc > 0.5] = midpoint_uniforms(env._cdf["sunny"], idx)
    return env, maps, u


@pytest.mark.parametrize("vis_equation", ["nerv", "nerfactor"])
def test_host_relight_chunk_matches_oracle(host_lib, golden_rotated, vis_equation):
    fx = golden_rotated
    f = oracle_field(fx)
    env, maps, u = _golden_chunk(fx, vis_equation)
    w, wo = relighting.relight_chunk_fused(f, env, ["sunny"], fx["rays"], maps, 1.7, u, 64,
                                           vis_equation=vis_equation)
    oenv = O.EnvLight({"sunny": fx["env_rgb"]})
    ow, owo = O.relight_chunk(f, oenv, "sunny", fx["rays"], maps, 1.7, fx["relight_idx"], 64,
                              vis_equation=vis_equation)
    assert (wo[0] - owo).abs().max() < 1e-4 and (w[0] - ow).abs().max() < 1e-4
    if vis_equation == "nerv":
        assert (wo[0] - fx["relight_without_bg"]).abs().max() < 1e-4
        assert (w[0] - fx["relight_with_bg"]).abs().max() < 1e-4
    miss = maps[5] <= 0.5
    assert torch.equal(wo[0][miss], torch.ones_like(wo[0][miss]))


def test_host_relight_two_maps_into_view_rows(host_lib, golden_rotated):
    """Several maps in one call, written at a row offset of larger maps; per map the same as a call of its own."""
    from tensoir_b200.relight import Environment_Light
    fx = golden_rotated
    f = oracle_field(fx)
    rgb = fx["env_rgb"].numpy()
    env = Environment_Light({"a": rgb, "b": rgb[::-1].copy() * 0.5}, device='cpu')
    n, S = fx["rays"].shape[0], 40
    u = torch.rand(2, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    out = (torch.full((2, n + 7, 3), -1.0), torch.full((2, n + 7, 3), -1.0))
    w, wo = relighting.relight_chunk_fused(f, env, ["a", "b"], fx["rays"], fx["relight_maps"], 1.3, u, S,
                                           out=out, row0=5)
    assert float(out[0][:, :5].max()) == -1.0 and float(out[1][:, 7 + n - 2:].max()) == -1.0
    for k, name in enumerate(("a", "b")):
        w1, wo1 = relighting.relight_chunk_fused(f, env, [name], fx["rays"], fx["relight_maps"], 1.3, u[k:k + 1], S)
        assert torch.equal(w[k], w1[0]) and torch.equal(wo[k], wo1[0])


def _sample_bins(host_so, cdf_rgb, u):
    """Run tir_relight_sample on one all-hit ray per row of u [m, S] and return the bins."""
    from tensoir_b200.relight import Environment_Light
    env = Environment_Light({"m": cdf_rgb}, device='cpu')
    tab, keep = relighting.env_tables(env, ["m"])
    m, S = u.shape
    rays = torch.tensor([[0.0, 0.0, 0.0, 0.0, 0.0, 1.0]]).repeat(m, 1)
    ones = torch.ones(m)
    normal = torch.tensor([[0.0, 0.0, 1.0]]).repeat(m, 1)
    bins = torch.empty(1, m, S, dtype=torch.int32)
    pos = torch.empty(1, m, S, dtype=torch.int32)
    lo, ld = torch.empty(m * S, 3), torch.empty(m * S, 3)
    cnt = torch.zeros(1, dtype=torch.int64)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert host_so.tir_relight_sample(tab, 1, p(rays), p(ones), p(normal), p(ones), m, S, 0.5, p(u.contiguous()),
                                      p(bins), p(pos), p(lo), p(ld), m * S, p(cnt), None) == 0
    assert int(cnt) == int((pos >= 0).sum())
    return env._cdf["m"], bins[0]


def test_host_bin_search_equals_searchsorted(host_lib):
    host_so = host_lib
    g = torch.Generator().manual_seed(7)
    rgb = torch.rand(8, 16, 3, generator=g)
    rgb[2, 3:9] = 0.0                                  # zero-mass bins
    rgb[0, :4] = 0.0                                   # zero-mass bins at the start of the CDF
    rgb[7, 12:] = 0.0                                  # ... and at its end
    cdf = relighting_cdf(rgb)
    steps = torch.cat([cdf, torch.zeros(1, dtype=torch.float64), torch.nextafter(cdf, torch.zeros_like(cdf)),
                       torch.nextafter(cdf, torch.ones_like(cdf))])
    u = torch.cat([torch.rand(4000, dtype=torch.float64, generator=g), steps.clamp(0, 1)])
    u = torch.cat([u, torch.zeros((-u.numel()) % 50, dtype=torch.float64)]).reshape(-1, 50)
    got_cdf, bins = _sample_bins(host_so, rgb.numpy(), u)
    assert torch.equal(got_cdf, cdf)
    want = torch.searchsorted(cdf, u, right=True).clamp(max=cdf.numel() - 1)
    assert torch.equal(bins.long(), want)
    assert not bool((rgb.sum(-1).reshape(-1)[want] == 0).any() & (u < 1).all())


def relighting_cdf(rgb):
    from tensoir_b200.relight import Environment_Light
    return Environment_Light({"m": rgb.numpy()}, device='cpu')._cdf["m"]


def test_host_background_equals_get_light(host_lib):
    """Non-hit rows (acc below the mask threshold) are white without background and the sRGB background with it."""
    host_so = host_lib
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.relight_utils import linear2srgb_torch
    g = torch.Generator().manual_seed(11)
    rgb = torch.rand(16, 32, 3, generator=g) * 0.999
    env = Environment_Light({"m": rgb.numpy()}, device='cpu')
    d = torch.randn(3000, 3, generator=g)
    d = torch.cat([d / d.norm(dim=-1, keepdim=True), torch.tensor([[0.0, 0.0, 1.0], [0.0, 0.0, -1.0],
                                                                   [1.0, 0.0, 0.0], [-1.0, 0.0, 0.0]])])
    n = d.shape[0]
    rays = torch.cat([torch.zeros(n, 3), d], 1)
    z3 = torch.zeros(n, 3)
    acc = torch.rand(n, generator=g) * 0.45                        # below 0.5: no hit, and acc_t = 0
    tab, keep = relighting.env_tables(env, ["m"])
    w, wo = torch.empty(1, n, 3), torch.empty(1, n, 3)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    i32 = torch.zeros(n, dtype=torch.int32)
    assert host_so.tir_relight_shade(tab, 1, p(rays), p(z3), p(z3), p(z3), 3, p(z3), p(acc), n, 1, 0.5,
                                     p(torch.ones(3)), p(i32), p(i32 - 1), None, 0, p(w), p(wo), n, 0, None) == 0
    assert torch.equal(wo[0], torch.ones(n, 3))
    raw = env.get_light("m", d)
    want = linear2srgb_torch(torch.clamp(raw, 0, 1))
    assert (w[0] - want).abs().max() < 1e-5        # torch's CPU grid_sample unnormalises as (x + 1) * (size - 1) / 2


@pytest.mark.parametrize("H,W,P", [(11, 11, 1), (24, 32, 3), (37, 53, 9)])
def test_host_eval_pairs_matches_oracle(host_lib, H, W, P):
    g = torch.Generator().manual_seed(H * W + P)
    a = torch.rand(P, H, W, 3, generator=g)
    b = torch.rand(P, H, W, 3, generator=g)
    a[0, 3:9, 2:8] = 0.5                                              # flat patch: the sigma clip rules
    b[0, 3:9, 2:8] = 0.25
    out = relighting.pair_metrics(a, b, H, W)
    assert out.shape == (P, 2) and out.dtype == torch.float64
    for p in range(P):
        d = a[p] - b[p]                                          # fp32 difference and square, fp64 sum
        assert float(out[p, 0]) == pytest.approx(float((d * d).double().sum()), rel=1e-12)
        assert abs(float(out[p, 1]) - EO.rgb_ssim(a[p].numpy(), b[p].numpy(), 1)) < 1e-12


def test_eval_pairs_arguments(host_so):
    lib = host_so
    n = C.c_int64(0)
    assert lib.tir_eval_pairs_work_size(2, 12, 12, None) == -1
    assert lib.tir_eval_pairs_work_size(-1, 12, 12, C.byref(n)) == -2
    assert lib.tir_eval_pairs_work_size(2, 12, 12, C.byref(n)) == 0 and n.value > 0
    buf = (C.c_float * (2 * 12 * 12 * 3))()
    out = (C.c_double * 4)()
    work = (C.c_double * n.value)()
    assert lib.tir_eval_pairs(buf, buf, 0, 12, 12, None, 0, None, None) == 0          # no pairs: no-op
    assert lib.tir_eval_pairs(buf, buf, 2, 10, 12, work, n.value, out, None) == -2    # SSIM needs 11x11
    assert lib.tir_eval_pairs(None, buf, 2, 12, 12, work, n.value, out, None) == -1
    assert lib.tir_eval_pairs(buf, buf, 2, 12, 12, work, 1, out, None) == -4          # work too small
    assert lib.tir_eval_pairs(buf, buf, 2, 12, 12, work, n.value, out, None) == 0


def test_relight_arguments(host_so):
    lib = host_so
    env = (_lib.TirEnvMap * 1)()
    assert lib.tir_relight_sample(None, 1, None, None, None, None, 4, 8, 0.5, None, None, None, None, None, 0, None,
                                  None) == -1
    assert lib.tir_relight_sample(env, 17, None, None, None, None, 4, 8, 0.5, None, None, None, None, None, 0, None,
                                  None) == -2                                     # more than TIR_RELIGHT_MAX_LIGHTS
    assert lib.tir_relight_sample(None, 1, None, None, None, None, 0, 8, 0.5, None, None, None, None, None, 0, None,
                                  None) == 0                                      # empty chunk: no-op
    env[0].H, env[0].W = 2, 2
    assert lib.tir_relight_shade(env, 1, None, None, None, None, 1, None, None, 4, 8, 0.5, None, None, None, None, 0,
                                 None, None, 4, 0, None) == -1                    # map without tables


def test_env_map_struct_layout(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tensoir_b200.h"\n'
                   'int main(void){printf("%zu %zu %zu %zu %zu %zu %d\\n",sizeof(TirEnvMap),offsetof(TirEnvMap,W),'
                   'offsetof(TirEnvMap,rgb),offsetof(TirEnvMap,dir),offsetof(TirEnvMap,pdf_return),'
                   'offsetof(TirEnvMap,cdf),TIR_RELIGHT_MAX_LIGHTS);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    T = _lib.TirEnvMap
    assert got == [C.sizeof(T), T.W.offset, T.rgb.offset, T.dir.offset, T.pdf_return.offset, T.cdf.offset,
                   _lib.RELIGHT_MAX_LIGHTS]


def test_synthetic_views_relighting_item_contract():
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    H, W = 24, 32
    names = ["bridge", "city", "night"]
    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=names)
    assert ds.split == "test" and ds.light_names == names and len(ds) == 2
    it = ds[0]
    shapes = {"rays": ((H * W, 6), torch.float32), "rgbs": ((3, H * W, 3), torch.float32),
              "light_idx": ((3, H * W, 1), torch.int32), "rgbs_mask": ((H * W, 1), torch.bool),
              "albedo": ((H * W, 3), torch.float32), "normals": ((H * W, 3), torch.float32),
              "normals_white": ((H * W, 3), torch.float32), "c2w": ((4, 4), torch.float32),
              "w2c": ((4, 4), torch.float32)}
    for k, (shape, dtype) in shapes.items():
        assert tuple(it[k].shape) == shape and it[k].dtype == dtype, k
    assert it["img_wh"] == (W, H)
    assert torch.equal(it["light_idx"], torch.zeros(3, H * W, 1, dtype=torch.int32))
    m = it["rgbs_mask"][:, 0]
    assert torch.equal(it["rgbs"][:, ~m], torch.ones(3, int((~m).sum()), 3))
    assert not torch.equal(it["rgbs"][0], it["rgbs"][1])
    assert torch.equal(it["normals_white"][~m], torch.ones(int((~m).sum()), 3))
    plain = SyntheticViews(hemisphere_poses(2), H, W)
    assert not hasattr(plain, "split") and not hasattr(plain, "light_names")


def test_host_relight_more_maps_than_one_call_takes(host_lib, golden_rotated):
    """More maps than TIR_RELIGHT_MAX_LIGHTS are relit in groups: the same as one call per map."""
    from tensoir_b200.relight import Environment_Light
    fx = golden_rotated
    f = oracle_field(fx)
    rgb = fx["env_rgb"].numpy()
    L = _lib.RELIGHT_MAX_LIGHTS + 2
    env = Environment_Light({f"m{k}": rgb * (0.5 + 0.1 * k) for k in range(L)}, device='cpu')
    names = [f"m{k}" for k in range(L)]
    n, S = fx["rays"].shape[0], 8
    u = torch.rand(L, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
    w, wo = relighting.relight_chunk_fused(f, env, names, fx["rays"], fx["relight_maps"], 1.1, u, S)
    for k in (0, _lib.RELIGHT_MAX_LIGHTS - 1, _lib.RELIGHT_MAX_LIGHTS, L - 1):
        w1, wo1 = relighting.relight_chunk_fused(f, env, [names[k]], fx["rays"], fx["relight_maps"], 1.1, u[k:k + 1], S)
        assert torch.equal(w[k], w1[0]) and torch.equal(wo[k], wo1[0]), k
