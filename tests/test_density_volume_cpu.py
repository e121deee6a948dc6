"""Host-side rules of the baked density volume (include/tensoir_b200.h, TirDensityVolume): the box
tir_density_volume_extent derives from the occupied-cell box, and the argument checks of the builder and of the
secondary march that reads the volume.  None of these calls reaches the device."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import _lib
    return _lib.load()


def _field(grid=(30, 31, 29), lo=(-1.2, -1.4, -1.1), hi=(1.3, 1.0, 1.6), occ=None, mask=True):
    from tensoir_b200 import _lib
    f = _lib.TirField()
    f.dC, f.aC = 16, 48
    for k in range(3):
        f.dplane[k] = f.dline[k] = 256
        f.grid[k] = grid[k]
        f.aabb_lo[k], f.aabb_hi[k] = lo[k], hi[k]
        f.inv_aabb[k] = float(np.float32(2.0) / (np.float32(hi[k]) - np.float32(lo[k])))
    f.amask = 512 if mask else None
    for k in range(3):
        f.occ_lo[k], f.occ_hi[k] = occ[k] if occ is not None else (1.0, -1.0)
    return f


def _extent(lib, f):
    lo, n = (C.c_int32 * 3)(), (C.c_int32 * 3)()
    rc = lib.tir_density_volume_extent(C.byref(f), lo, n)
    return rc, list(lo), list(n)


def _vertex(f, a, c):
    """floor of the grid coordinate of world coordinate c: normalize_coord + unnormalize in float32, no FMA."""
    f32 = np.float32
    n = (f32(c) - f32(f.aabb_lo[a])) * f32(f.inv_aabb[a]) - f32(1)
    return int(np.floor(((n + f32(1)) * f32(0.5)) * f32(f.grid[a] - 1)))


def _want_axis(f, a, c0, c1):
    """floor(i) - 1 .. floor(i) + 2 of the two box ends, clamped to the grid."""
    lo = max(_vertex(f, a, c0) - 1, 0)
    hi = min(_vertex(f, a, c1) + 2, f.grid[a] - 1)
    return lo, max(hi - lo + 1, 0)


def test_extent_is_the_whole_grid_without_mask_or_box(lib):
    for f in (_field(mask=False), _field(mask=True), _field(mask=False, occ=((-0.5, 0.5),) * 3)):
        assert _extent(lib, f) == (0, [0, 0, 0], [30, 31, 29])


def test_extent_covers_the_taps_of_the_occupied_box(lib):
    occ = ((-0.71, 0.33), (-1.4, 0.02), (0.5, 1.6))           # y starts at the grid's first vertex, z ends at its last
    f = _field(occ=occ)
    rc, lo, n = _extent(lib, f)
    assert rc == 0
    for a in range(3):
        assert (lo[a], n[a]) == _want_axis(f, a, *occ[a]), a
    assert lo[1] == 0 and lo[2] + n[2] == 29                # clamped to the grid
    assert 0 < n[0] < 30
    # both in-grid taps of every coordinate inside the box lie in the extent (a dense sweep of each axis)
    for a in range(3):
        for c in np.linspace(occ[a][0], occ[a][1], 997, dtype=np.float32):
            i = _vertex(f, a, c)
            for t in (i, i + 1):
                if 0 <= t < f.grid[a]:
                    assert lo[a] <= t < lo[a] + n[a], (a, float(c), t)


def test_extent_of_a_box_outside_the_grid_is_empty(lib):
    f = _field(occ=((2.0, 2.5), (-0.5, 0.5), (-0.5, 0.5)))
    assert _extent(lib, f) == (0, [0, 0, 0], [0, 0, 0])


def test_extent_argument_checks(lib):
    lo, n = (C.c_int32 * 3)(), (C.c_int32 * 3)()
    assert lib.tir_density_volume_extent(None, lo, n) == -1
    assert lib.tir_density_volume_extent(C.byref(_field()), None, n) == -1
    assert lib.tir_density_volume_extent(C.byref(_field(grid=(30, 0, 29))), lo, n) == -2


def test_build_argument_checks(lib):
    from tensoir_b200 import _lib
    f = _field()
    v = _lib.TirDensityVolume()
    v.data = 1024
    v.lo[:], v.n[:] = [0, 0, 0], [30, 31, 29]
    assert lib.tir_density_volume_build(None, C.byref(v), 1 << 20, None) == -1
    assert lib.tir_density_volume_build(C.byref(f), None, 1 << 20, None) == -1
    assert lib.tir_density_volume_build(C.byref(f), C.byref(v), 30 * 31 * 29 - 1, None) == -4
    v.lo[1] = 1                                                 # leaves the grid along y
    assert lib.tir_density_volume_build(C.byref(f), C.byref(v), 1 << 20, None) == -2
    v.lo[1], v.n[2] = 0, -1
    assert lib.tir_density_volume_build(C.byref(f), C.byref(v), 1 << 20, None) == -2
    v.n[2] = 0                                                  # empty box: nothing to build, no launch
    assert lib.tir_density_volume_build(C.byref(f), C.byref(v), 0, None) == 0
    v.n[2], v.data = 29, None
    assert lib.tir_density_volume_build(C.byref(f), C.byref(v), 1 << 20, None) == -1
    v.data = 1024
    f.dC = 8
    assert lib.tir_density_volume_build(C.byref(f), C.byref(v), 1 << 20, None) == -2


def test_march_vol_argument_checks(lib):
    from tensoir_b200 import _lib
    f = _field()
    cfg = _lib.TirMarchCfg()
    cfg.sampling, cfg.n_samples, cfg.z_table = _lib.SAMPLE_TABLE, 24, 2048
    v = _lib.TirDensityVolume()
    v.data = 1024
    v.lo[:], v.n[:] = [0, 0, 0], [30, 31, 30]                  # one vertex past the grid along z
    p = C.c_void_p(4096)
    args = (p, p, 5, p, 8, C.byref(cfg))
    out = (p, p, p, 1 << 16, None, None)
    assert lib.tir_secondary_march_vol(C.byref(f), *args, None, *out) == -1
    assert lib.tir_secondary_march_vol(C.byref(f), *args, C.byref(v), *out) == -2
    assert lib.tir_secondary_radiance_vol(C.byref(f), None, p, p, p, 5, p, 8, C.byref(cfg), C.byref(v), p, p, p, p,
                                          1 << 16, None, None) == -1
    # no points: a no-op whatever the other arguments are
    assert lib.tir_secondary_march_vol(None, None, None, 0, None, 0, None, None, None, None, None, 0, None, None) == 0
