"""The VM-factor gradient scatters sum the rows of a run that hit the same tap texel in registers and issue one atomic
per run (csrc/tir_vm.cu, kScatterRows rows per thread group).  Each scatter is checked against float64 with the bound
of test_vm_kernels_fp64.py on lists whose run structure crosses the group, warp and grid-stride boundaries: runs of 1,
2, 31, 32, 33, 64 and 65 rows, alternating texels (no runs), runs with zero-weight taps inside, and the valid list of
the lego bench field in ray order and shuffled.  The fused backward's one launch of the appearance-list scatters (two
point sets and the derived normals' double backward) and the density scatter on a list whose device-side length is
below its capacity, with sentinel coordinates in the padding rows, are checked stage by stage by run_case."""
import ctypes as C

import pytest
import torch

import test_vm_kernels_fp64 as V
from oracle import tensoir_oracle as O

pytestmark = pytest.mark.gpu

DEV = V.DEV
RUNS = [1, 2, 31, 32, 33, 64, 65]
CHUNK = 1 << 16


def _cell(g, lo=0.15, hi=0.85):
    """a random point strictly inside one texel cell of every plane and line (all taps fixed for the cell)"""
    idx = [int(torch.randint(1, s - 2, (1,), generator=g)) for s in V.GRID]
    frac = lo + (hi - lo) * torch.rand(3, generator=g)
    return torch.tensor([-1 + 2 * (i + f) / (s - 1) for i, f, s in zip(idx, frac.tolist(), V.GRID)])


def _jitter_in_cell(c, n, g):
    half = torch.tensor([0.1 / (s - 1) for s in V.GRID])
    return c + (torch.rand(n, 3, generator=g) * 2 - 1) * half


def runs_list(lengths, seed, offset=3):
    """consecutive runs of the given lengths, each inside its own cell, after ``offset`` unrelated rows (so runs start
    at every position of a row group)"""
    g = torch.Generator().manual_seed(seed)
    parts = [torch.rand(offset, 3, generator=g) * 2 - 1]
    for n in lengths:
        parts.append(_jitter_in_cell(_cell(g), n, g))
    return torch.cat(parts)


def alternating(n, seed):
    g = torch.Generator().manual_seed(seed)
    a, b = _cell(g), _cell(g)
    x = torch.where((torch.arange(n) % 2 == 0)[:, None], _jitter_in_cell(a, n, g), _jitter_in_cell(b, n, g))
    return x


def zero_weight_runs(seed):
    """runs inside one cell whose rows alternate with rows on texel centres (one tap of each axis has weight 0) and
    rows just outside +-1 (zero-padding taps), so zero-weight taps sit inside the runs of the other taps"""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for n in (5, 17, 40):
        c = _cell(g)
        inner = _jitter_in_cell(c, n, g)
        centre = inner.clone()
        for a, s in enumerate(V.GRID):
            centre[:, a] = torch.round((centre[:, a] + 1) / 2 * (s - 1)) * 2 / (s - 1) - 1
        out = inner.clone()
        out[:, 0] = 1 + 0.3 / (V.GRID[0] - 1)
        rows.append(torch.stack([inner, centre, out], 1).reshape(-1, 3))
    return torch.cat(rows)


def lego_valid_list(m=None, n_rays=256):
    """the valid-sample list of ``n_rays`` rays of a training batch on the lego field ``m`` (default: the bench's lego
    field at 128^3), in ray order"""
    from tensoir_b200 import vm_autograd as vm
    from tensoir_b200.synthetic import hemisphere_poses, make_lego_model, n_samples_for, training_batch
    if m is None:
        m = make_lego_model(128, torch.device(DEV))
    rays, _ = training_batch(hemisphere_poses(100), n_rays, 0)
    rays = rays.to(DEV).float()
    ref = vm.valid_samples(m, rays[:, :3], rays[:, 3:6], n_samples=n_samples_for(int(m.gridSize[0])))
    return ref["xn"].float().cpu()


_LEGO = {}


def points(case):
    if case == "runs":
        return runs_list(RUNS, 1)
    if case == "runs-reversed":
        return runs_list(RUNS[::-1] * 3, 2, offset=5)
    if case == "alternating":
        return alternating(4096, 3)
    if case == "zero-weight":
        return zero_weight_runs(4)
    if case.startswith("lego"):
        if "x" not in _LEGO:
            _LEGO["x"] = lego_valid_list()
        x = _LEGO["x"]
        if case == "lego-shuffled":
            x = x[torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(5))]
        return x.contiguous()
    raise KeyError(case)


CASES = ["runs", "runs-reversed", "alternating", "zero-weight", "lego", "lego-shuffled"]


@pytest.fixture(scope="module")
def field():
    from tensoir_b200 import _lib
    _lib.load()
    return V.Field(0)


def scatter_reference(field, kind, x, g, gp, gl, what):
    """The density ("density": g [n]) or appearance-products ("app": g [n, 144]) scatter the kernel wrote into gp / gl
    against float64 autograd of the gather, with test_vm_kernels_fp64's bound; the reference runs in chunks of CHUNK
    rows, so lists of a training step fit.  -> the largest err / bound"""
    planes_of = (lambda f: (f.density_plane, f.density_line)) if kind == "density" else \
        (lambda f: (f.app_plane, f.app_line))
    C_ = 16 if kind == "density" else 48
    with V.f64():
        f = field.oracle(torch.float64)
        planes, lines = planes_of(f)
        for p in planes + lines:
            p.requires_grad_(True)
        mags = units = None
        for a in range(0, x.shape[0], CHUNK):
            xs = x[a:a + CHUNK].to(DEV, torch.float64)
            gc = g[a:a + CHUNK].to(DEV).double()
            if kind == "density":
                (O.density_feature(f, xs) * gc).sum().backward()
                ga = gc.abs()[:, None]

                def coef_p(k, t, j):
                    return ga * t["ptaps"][j][1][:, None] * t["AL"]

                def coef_l(k, t, j):
                    return ga * t["ltaps"][j][1][:, None] * t["AP"]
            else:
                ps, ls = O._app_products(f, xs)
                (ps * ls).t().backward(gc)
                ga = gc.abs().view(-1, 3, 48)

                def coef_p(k, t, j):
                    return ga[:, k] * t["ptaps"][j][1][:, None] * t["AL"]

                def coef_l(k, t, j):
                    return ga[:, k] * t["ltaps"][j][1][:, None] * t["AP"]
            with torch.no_grad():
                m = V.scatter(V.tap_sums(planes, lines, xs, False, False, field.grid), coef_p, coef_l, C_)
                u = V.scatter(V.tap_sums(planes, lines, xs, False, True, field.grid), coef_p, coef_l, C_)
            mags = m if mags is None else [tuple(p + q for p, q in zip(A, B)) for A, B in zip(mags, m)]
            units = u if units is None else [tuple(p + q for p, q in zip(A, B)) for A, B in zip(units, u)]
        return V.check_scatter(gp, gl, [p.grad for p in planes], [l_.grad for l_ in lines], mags, units, what,
                               field.grid)


def density_bwd(field, x, what):
    """tir_vm_density_bwd on the rows x (every 7th upstream gradient 0: skipped rows inside runs) against float64
    -> the largest err / bound"""
    from tensoir_b200 import _lib
    lib = _lib.load()
    x = x.float()
    xd = x.to(DEV).contiguous()
    n = x.shape[0]
    g = torch.randn(n, generator=torch.Generator().manual_seed(n + 1))
    g[3::7] = 0.0                                         # skipped rows inside runs
    gd = g.to(DEV)
    gp, gl, ap, al = V.grad_shadows(field, "density")
    _lib.check(lib.tir_vm_density_bwd(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(gd), ap, al,
                                      _lib.stream_ptr()), "density bwd")
    torch.cuda.synchronize()
    return scatter_reference(field, "density", x, gd, gp, gl, f"density bwd {what}")


def app_products_bwd(field, x, what):
    """tir_vm_app_products_bwd on the rows x against float64 -> the largest err / bound"""
    from tensoir_b200 import _lib
    lib = _lib.load()
    x = x.float()
    xd = x.to(DEV).contiguous()
    n = x.shape[0]
    gout = torch.randn(n, 144, generator=torch.Generator().manual_seed(n)).to(DEV)
    gp, gl, ap, al = V.grad_shadows(field, "app")
    _lib.check(lib.tir_vm_app_products_bwd(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(gout), ap, al,
                                           _lib.stream_ptr()), "app products bwd")
    torch.cuda.synchronize()
    return scatter_reference(field, "app", x, gout, gp, gl, f"app products bwd {what}")


@pytest.mark.parametrize("case", CASES)
def test_density_bwd_runs(field, case):
    density_bwd(field, points(case), case)


@pytest.mark.parametrize("case", CASES)
def test_app_products_bwd_runs(field, case):
    app_products_bwd(field, points(case), case)


@pytest.mark.parametrize("case", [c for c in CASES if c != "zero-weight"])
def test_density_grad_bwd_runs(field, case):
    """(texel centres make the spatial derivative one-sided, so the zero-weight set is left to the two scatters above)"""
    from tensoir_b200 import _lib
    lib = _lib.load()
    x = points(case).float()
    xd = x.to(DEV).contiguous()
    n = x.shape[0]
    gen = torch.Generator().manual_seed(n + 2)
    gf = torch.randn(n, generator=gen).to(DEV)
    gx = torch.randn(n, 3, generator=gen).to(DEV)
    gp, gl, ap, al = V.grad_shadows(field, "density")
    _lib.check(lib.tir_vm_density_grad_bwd(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(gf), _lib.dptr(gx),
                                           ap, al, _lib.stream_ptr()), "density grad bwd")
    torch.cuda.synchronize()
    with V.f64():
        f = field.oracle(torch.float64)
        for p in f.density_plane + f.density_line:
            p.requires_grad_(True)
        xs = x.to(DEV, torch.float64).requires_grad_(True)
        ft = O.density_feature_with_xyz_grad(f, xs)
        (d,) = torch.autograd.grad(ft.sum(), xs, create_graph=True)
        ((ft * gf.double()).sum() + (d * gx.double()).sum()).backward()
        ts = V.tap_sums(f.density_plane, f.density_line, xs.detach(), True, False)
        tu = V.tap_sums(f.density_plane, f.density_line, xs.detach(), True, True)
        agf, agx = gf.double().abs(), gx.double().abs()

        def coef_p(k, t, j):
            sx, sy, sl = t["s"]
            _, w, dwx, dwy = t["ptaps"][j]
            g0, g1, gv = agx[:, V.MAT[k][0]] * sx, agx[:, V.MAT[k][1]] * sy, agx[:, V.VEC[k]] * sl
            return (agf * w + g0 * dwx + g1 * dwy)[:, None] * t["AL"] + (gv * w)[:, None] * t["AZ"]

        def coef_l(k, t, j):
            sx, sy, sl = t["s"]
            _, w, kz = t["ltaps"][j]
            g0, g1, gv = agx[:, V.MAT[k][0]] * sx, agx[:, V.MAT[k][1]] * sy, agx[:, V.VEC[k]] * sl
            return t["AP"] * (agf * w + gv * kz)[:, None] + w[:, None] * (g0[:, None] * t["AX"] + g1[:, None] * t["AY"])
        m = V.scatter(ts, coef_p, coef_l, 16)
        u = V.scatter(tu, coef_p, coef_l, 16)
        V.check_scatter(gp, gl, [p.grad for p in f.density_plane], [l.grad for l in f.density_line], m, u,
                        f"density grad bwd {case}")


@pytest.mark.parametrize("kind", ["derived_plus_predicted", "purely_predicted"])
def test_fused_backward_with_padding_rows(kind):
    """tir_primary_backward with both lists longer than their device-side lengths, sentinel coordinates in the padding
    rows: the appearance-list launch (two point sets, plus the derived normals' double backward with
    derived_plus_predicted) and the density scatter match float64 stage by stage, so no padding row was scattered."""
    import test_primary_kernels_fp64 as P
    m, rays, li = P.rotated(kind)
    cs = P.Case(m, rays, li, -1, 1)
    probe = P.run_case(cs, stats_key=f"probe {kind}")
    res = P.run_case(cs, cap_valid=probe["total"] + 300, cap_app=probe["total_app"] + 300,
                     stats_key=f"padding {kind}")
    assert res["total"] == probe["total"] and res["total_app"] == probe["total_app"] > 100
