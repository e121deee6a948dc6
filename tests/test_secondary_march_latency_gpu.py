"""The dense secondary march's volume instance at 3 CTAs per SM (80 registers, 32-bit per-lane counters, the
appearance append re-reading its queue entry) and the density-volume builder with its z-dependent factor rows staged in
shared memory: the volume march against the factor march in count-parity and lean modes at several sample counts, and
the builder against float64 on boxes that cut its tiles."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from gpu_helpers import load_shrunk_state, model_from_fixture   # noqa: E402
from test_density_volume_gpu import (EPS32, W_RTOL, _compare, _d64, _factors, _grid, _lego_inputs,   # noqa: E402
                                     _shrunk_inputs)

DEV = "cuda:0"


def _march(model, pts, nrm, li, dirs, n_sample, lean, use_vol):
    """One tir_secondary_radiance(_vol) call with counters -> dict of outputs (as test_density_volume_gpu._march, plus
    the lean flag)."""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.device_field import mlp_struct
    lib = _lib.load()
    f = ops.device_field(model).refresh(model)
    keep = []
    cfg = ops.march_cfg(model, table=ops.equal_z_table(n_sample, 0.05, 1.5, DEV), keep=keep)
    if lean:
        cfg.flags |= _lib.MARCH_LEAN_COUNTERS
    mlp = mlp_struct(model, "renderModule", keep, light="index")
    n_pts, n_dirs = pts.shape[0], dirs.shape[0]
    vis = torch.zeros(n_pts, n_dirs, 1, device=DEV)
    ind = torch.zeros(n_pts, n_dirs, 3, device=DEV)
    cnt = ops.new_counters(DEV)
    sc = ops.SampleScratch(DEV, max(1 << 16, 4 * n_pts * n_dirs * -(-n_sample // 32)))
    li32 = li.reshape(-1).to(torch.int32).contiguous()
    common = (_lib.dptr(pts), _lib.dptr(nrm), _lib.dptr(li32, torch.int32), n_pts, _lib.dptr(dirs), n_dirs,
              C.byref(cfg))
    tail = (_lib.dptr(vis), _lib.dptr(ind), _lib.dptr(sc.buf, torch.uint8), _lib.dptr(sc.count, torch.int32),
            sc.capacity, _lib.dptr(cnt, torch.int64), _lib.stream_ptr())
    if use_vol:
        v = ops.density_volume(model, f)
        rc = lib.tir_secondary_radiance_vol(C.byref(f), C.byref(mlp), *common, C.byref(v), *tail)
    else:
        rc = lib.tir_secondary_radiance(C.byref(f), C.byref(mlp), *common, *tail)
    _lib.check(rc, "secondary radiance")
    torch.cuda.synchronize()
    sm = sc.samples()
    key = (sm["ray"].long() * n_sample + sm["sample"].long()).sort()
    return {"vis": vis, "ind": ind, "cnt": ops.counters_dict(cnt), "key": key.values,
            "w": sm["weight"][key.indices]}


def _compare_lean(a, b):
    """Lean counters count the queries made, and a ray stops at the first batch that leaves its transmittance at
    exactly 0: where the two paths round T differently they stop at different samples, so only the outputs compare."""
    assert a["cnt"]["rays"] == b["cnt"]["rays"] and a["cnt"]["overflow"] == b["cnt"]["overflow"] == 0
    same, same_b = torch.isin(a["key"], b["key"]), torch.isin(b["key"], a["key"])
    assert int((~same).sum()) + int((~same_b).sum()) <= 2
    assert torch.allclose(a["w"][same], b["w"][same_b], rtol=W_RTOL, atol=1e-7)
    assert float((a["vis"] - b["vis"]).abs().max()) <= 1e-5
    assert float(((a["ind"] - b["ind"]).abs() / (1 + b["ind"].abs())).max()) <= 1e-4


@pytest.fixture(scope="module", params=("lego", "B"))
def scene(request):
    if request.param == "lego":
        return _lego_inputs()
    fx = load_shrunk_state(request.param)
    m = model_from_fixture(fx, DEV)
    return (m,) + _shrunk_inputs(fx, m)


@pytest.mark.parametrize("lean", [False, True], ids=["count_parity", "lean"])
@pytest.mark.parametrize("n_sample", [96, 40, 129])
def test_volume_march_matches_factor_march(scene, n_sample, lean):
    """96 samples (the training step's), 40 and 129 (a last chunk cut by the end of the ray).  Two launches of the
    volume path agree with each other and with the factor path; in count-parity mode the mask, density and ray counters
    are exact."""
    m, pts, nrm, li, dirs = scene
    fac = _march(m, pts, nrm, li, dirs, n_sample, lean, use_vol=False)
    vol = [_march(m, pts, nrm, li, dirs, n_sample, lean, use_vol=True) for _ in range(2)]
    assert fac["cnt"]["density"] > 0
    for r in vol:
        if lean:
            _compare_lean(r, fac)
        else:
            _compare(r, fac, W_RTOL)
    if not lean:
        for k in ("mask", "density", "rays"):
            assert vol[0]["cnt"][k] == vol[1]["cnt"][k] == fac["cnt"][k], k


def _build_box(model, lo, n):
    """tir_density_volume_build over the box (lo, n) into a buffer with a NaN guard behind it -> (D [n_z, n_y, n_x],
    the guard)."""
    from tensoir_b200 import _lib, ops
    lib = _lib.load()
    f = ops.device_field(model).refresh(model)
    size = n[0] * n[1] * n[2]
    buf = torch.full((size + 4096,), float("nan"), device=DEV)
    v = _lib.TirDensityVolume()
    v.data, v.lo[:], v.n[:] = buf.data_ptr(), lo, n
    _lib.check(lib.tir_density_volume_build(C.byref(f), C.byref(v), size, _lib.stream_ptr()), "build")
    torch.cuda.synchronize()
    return buf[:size].view(n[2], n[1], n[0]).cpu(), buf[size:].cpu()


@pytest.mark.parametrize("where", ["lego", "B"])
def test_builder_on_boxes_that_cut_its_tiles(where):
    """One-vertex-thick boxes, a single vertex, boxes on the grid's faces and corners, and sizes that are no multiple of
    the 32 x 8 x 8 tile: every vertex of the box is written, against float64, and nothing behind it."""
    if where == "lego":
        m = _lego_inputs()[0]
    else:
        m = model_from_fixture(load_shrunk_state(where), DEV)
    G = _grid(m)
    boxes = [([0, 0, 0], G),
             ([0, 0, 0], [1, 1, 1]),
             ([G[0] - 1, G[1] - 1, G[2] - 1], [1, 1, 1]),
             ([3, 0, 5], [G[0] - 3, G[1], 1]),
             ([0, 2, 0], [G[0], 1, G[2]]),
             ([G[0] - 1, 0, 0], [1, G[1], G[2]]),
             ([1, 2, 3], [min(33, G[0] - 1), min(9, G[1] - 2), min(17, G[2] - 3)]),
             ([G[0] - 13, G[1] - 11, G[2] - 9], [13, 11, 9])]
    factors = _factors(m)
    for lo, n in boxes:
        got, guard = _build_box(m, lo, n)
        assert bool(torch.isfinite(got).all()), (lo, n)
        assert bool(torch.isnan(guard).all()), (lo, n)
        want, mag = _d64(factors, lo, n)
        assert bool(((got.double() - want).abs() <= EPS32 * 18 * mag).all()), (lo, n)
