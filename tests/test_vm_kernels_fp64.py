"""The point-wise VM kernels and the compositing scan (csrc/tir_vm.cu), called through the C ABI, against torch autograd
of the same expressions in float64: F.grid_sample (zero padding) for tir_vm_app_products / tir_vm_density_bwd, the
oracle's grid_sample_clamped for tir_vm_density_grad / _bwd, and the oracle's raw2alpha for tir_composite_fwd / _bwd.

The field is non-cubic (grid 37 x 18 x 61: every axis has a different size - 1) with random channel-last planes, so a
swapped axis, size or scale changes the result.  The point sets cover taps on texel centres and on +-1, partial taps
just outside +-1, a cluster of thousands of points inside one texel (contending float4 atomics) and list lengths on both
sides of the first extra grid-stride pass of every scatter (derived from the device's SM count).

Tolerances come from the fp32 error of each expression, evaluated in float64 and independent of the summation order:
an entry may differ from the float64 value by

    eps32 * ((16 + 4 sqrt(n_add)) * sum|terms| + 2 (G - 1) * sum|terms with unit tap weights|)

where sum|terms| is the sum of the absolute products the entry adds up (from |values| and |tap weights|), n_add is the
number of atomic additions into the entry (the order of a float sum of n terms adds up to ~sqrt(n) roundings), and the
last part covers the fp32 rounding of the texel coordinate ((x + 1) / 2 * (G - 1) is exact to eps32 * (G - 1), and a
tap weight moves by as much; every tap weight and its derivative has modulus <= 1)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import tensoir_oracle as O        # noqa: E402

DEV = "cuda:0"
EPS32 = 2.0 ** -24 * 2          # float32 machine epsilon (unit roundoff 2^-24)
GRID = (37, 18, 61)
MAT = O.MAT_MODE
VEC = O.VEC_MODE


class Field:
    """Random VM factors in the reference's NCHW layout plus the channel-last copies and the TirField the kernels
    read.  ``model``: take the factors of that TensorVMSplit (and its grid) instead."""

    def __init__(self, seed=0, model=None):
        from tensoir_b200 import _lib
        g = torch.Generator().manual_seed(seed)
        self.dplane, self.dline, self.aplane, self.aline = [], [], [], []
        self.grid = GRID if model is None else tuple(int(x) for x in model.gridSize)
        for k in range(3):
            if model is not None:
                for name, src in (("dplane", model.density_plane), ("dline", model.density_line),
                                  ("aplane", model.app_plane), ("aline", model.app_line)):
                    getattr(self, name).append(src[k].detach().float().cpu())
                continue
            W, H, D = GRID[MAT[k][0]], GRID[MAT[k][1]], GRID[VEC[k]]
            self.dplane.append(torch.randn(1, 16, H, W, generator=g))
            self.dline.append(torch.randn(1, 16, D, 1, generator=g))
            self.aplane.append(torch.randn(1, 48, H, W, generator=g))
            self.aline.append(torch.randn(1, 48, D, 1, generator=g))
        self.cl = {name: [t[0].permute(1, 2, 0).contiguous().to(DEV) for t in getattr(self, name)]
                   for name in ("dplane", "dline", "aplane", "aline")}
        s = _lib.TirField()
        for k in range(3):
            s.dplane[k], s.dline[k] = self.cl["dplane"][k].data_ptr(), self.cl["dline"][k].data_ptr()
            s.aplane[k], s.aline[k] = self.cl["aplane"][k].data_ptr(), self.cl["aline"][k].data_ptr()
            s.grid[k] = self.grid[k]
        s.dC, s.aC = 16, 48
        self.struct = s

    def oracle(self, dtype, absolute=False):
        """OracleField of the same factors (|factors| when ``absolute``) on the GPU in ``dtype``."""
        def cp(ts):
            return [(t.abs() if absolute else t).clone() for t in ts]
        f = O.OracleField(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), grid_size=list(self.grid),
                          density_plane=cp(self.dplane), density_line=cp(self.dline), app_plane=cp(self.aplane),
                          app_line=cp(self.aline), basis_w=None, mlp_rgb=None)
        return f.to(DEV, dtype)


class f64:
    """Run oracle functions with float64 intermediates."""

    def __enter__(self):
        self.old = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)

    def __exit__(self, *exc):
        torch.set_default_dtype(self.old)


def grad_shadows(field, kind):
    planes = field.cl["dplane" if kind == "density" else "aplane"]
    lines = field.cl["dline" if kind == "density" else "aline"]
    gp, gl = [torch.zeros_like(p) for p in planes], [torch.zeros_like(l) for l in lines]
    arr_p, arr_l = (C.c_void_p * 3)(), (C.c_void_p * 3)()
    for k in range(3):
        arr_p[k], arr_l[k] = gp[k].data_ptr(), gl[k].data_ptr()
    return gp, gl, arr_p, arr_l


def as_param_layout(gp, gl):
    return [g.permute(2, 0, 1)[None] for g in gp], [g.permute(2, 0, 1)[None] for g in gl]


# ------------------------------------------------------------------------------------------------------------------
# float64 magnitudes: per-tap absolute coefficients of the gathers and scatters
# ------------------------------------------------------------------------------------------------------------------
def axis_taps(coord, size, clamped, unit):
    """The two taps of one axis: (index, |weight|, |d weight / d index|) in float64.  Zero padding drops taps outside
    the grid; the clamped sampler clamps their index.  ``unit`` replaces every kept weight by 1."""
    i = (coord + 1) / 2 * (size - 1)
    i0 = torch.floor(i)
    out = []
    for idx, w in ((i0, (i0 + 1) - i), (i0 + 1, i - i0)):
        keep = torch.ones_like(w) if clamped else ((idx >= 0) & (idx <= size - 1)).double()
        w = keep if unit else w.abs() * keep
        out.append((idx.clamp(0, size - 1).long(), w, keep))
    return out


def tap_sums(planes, lines, x, clamped, unit, grid=GRID):
    """Per orientation k: the taps and the channel sums A_P = sum_t |w_t||P_t|, AX/AY = sum_t |dw_t/dx||P_t| (x / y of
    the plane), A_L = sum_u |w_u||L_u|, AZ = sum_u |dw_u/dz||L_u|, all [n, C]."""
    res = []
    for k in range(3):
        m0, m1, v = MAT[k][0], MAT[k][1], VEC[k]
        W, H, D = grid[m0], grid[m1], grid[v]
        P = planes[k][0].reshape(planes[k].shape[1], -1).t().abs()
        L = lines[k][0, :, :, 0].t().abs()
        tx, ty, tz = axis_taps(x[:, m0], W, clamped, unit), axis_taps(x[:, m1], H, clamped, unit), \
            axis_taps(x[:, v], D, clamped, unit)
        ptaps = []
        for iy, wy, ky in ty:
            for ix, wx, kx in tx:
                # |d w / d ix| = |wy|, |d w / d iy| = |wx| (bilinear); the unit variant keeps them at 1
                ptaps.append((iy * W + ix, wx * wy, wy * kx, wx * ky))
        ltaps = [(iz, wz, kz) for iz, wz, kz in tz]
        AP = sum(w[:, None] * P[t] for t, w, _, _ in ptaps)
        AX = sum(dx[:, None] * P[t] for t, _, dx, _ in ptaps)
        AY = sum(dy[:, None] * P[t] for t, _, _, dy in ptaps)
        AL = sum(w[:, None] * L[u] for u, w, _ in ltaps)
        AZ = sum(kz[:, None] * L[u] for u, _, kz in ltaps)
        res.append(dict(ptaps=ptaps, ltaps=ltaps, AP=AP, AX=AX, AY=AY, AL=AL, AZ=AZ, HW=H * W, D=D,
                        s=(0.5 * (W - 1), 0.5 * (H - 1), 0.5 * (D - 1))))
    return res


def scatter(ts, coef_p, coef_l, C_):
    """index_add of per-tap coefficients [n, C] into [HW, C] / [D, C] tables (float64), per orientation; also counts
    the additions per entry."""
    out = []
    for k, t in enumerate(ts):
        gp = torch.zeros(t["HW"], C_, dtype=torch.float64, device=DEV)
        gl = torch.zeros(t["D"], C_, dtype=torch.float64, device=DEV)
        cp = torch.zeros(t["HW"], dtype=torch.float64, device=DEV)
        cl = torch.zeros(t["D"], dtype=torch.float64, device=DEV)
        for j, (idx, *_rest) in enumerate(t["ptaps"]):
            gp.index_add_(0, idx, coef_p(k, t, j))
            cp.index_add_(0, idx, torch.ones_like(idx, dtype=torch.float64))
        for j, (idx, *_rest) in enumerate(t["ltaps"]):
            gl.index_add_(0, idx, coef_l(k, t, j))
            cl.index_add_(0, idx, torch.ones_like(idx, dtype=torch.float64))
        out.append((gp, gl, cp, cl))
    return out


def bound(mag, unit, n_add=None, grid=GRID):
    k = 16.0 if n_add is None else 16.0 + 4.0 * n_add.sqrt()
    return EPS32 * (k * mag + 2.0 * (max(grid) - 1) * unit)


def check(got, want, bnd, what):
    """-> the largest err / bound"""
    got, want = got.detach().double().reshape(want.shape), want.detach().double()
    err = (got - want).abs()
    ratio = err / bnd.reshape(want.shape).clamp_min(1e-30)
    assert bool(torch.isfinite(got).all()), what
    worst = int(ratio.reshape(-1).argmax())
    assert float(ratio.max()) <= 1.0, (what, float(ratio.max()), float(err.reshape(-1)[worst]),
                                       float(want.reshape(-1)[worst]), float(bnd.reshape(-1)[worst]))
    return float(ratio.max())


def check_scatter(gp_got, gl_got, want_p, want_l, mags, units, what, grid=GRID):
    """Parameter gradients (channel-last [H,W,C] / [D,1,C] from the kernel) against the float64 NCHW gradients.
    -> the largest err / bound"""
    gp_n, gl_n = as_param_layout(gp_got, gl_got)
    worst = 0.0
    for k in range(3):
        mp, ml, cp, cl = mags[k]
        up, ul = units[k][0], units[k][1]
        C_ = mp.shape[1]
        H, W = want_p[k].shape[2], want_p[k].shape[3]
        D = want_l[k].shape[2]
        bp = bound(mp, up, cp[:, None], grid).t().reshape(1, C_, H, W)
        bl = bound(ml, ul, cl[:, None], grid).t().reshape(1, C_, D, 1)
        worst = max(worst, check(gp_n[k], want_p[k], bp, f"{what} plane {k}"),
                    check(gl_n[k], want_l[k], bl, f"{what} line {k}"))
    return worst


# ------------------------------------------------------------------------------------------------------------------
# point sets
# ------------------------------------------------------------------------------------------------------------------
def _threads():
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 128     # blocks_for's cap x 128 threads


def point_set(name, n=None):
    g = torch.Generator().manual_seed(sum(map(ord, name)) + (n or 0))
    if name == "random":
        return torch.rand(n, 3, generator=g) * 2 - 1
    if name == "texel":
        # texel centres of every axis (in the float32 the kernels get) and the faces +-1 exactly
        cols = []
        for a in range(3):
            s = GRID[a]
            c = torch.cat([torch.linspace(-1, 1, s), torch.tensor([-1.0, 1.0, -1.0, 1.0])])
            cols.append(c[torch.randint(0, c.numel(), (2000,), generator=g)])
        return torch.stack(cols, 1)
    if name == "outside":
        # just outside +-1 along one or more axes, within half a texel: partial zero-padding taps, full clamped taps
        x = torch.rand(3000, 3, generator=g) * 2 - 1
        sel = torch.rand(3000, 3, generator=g) < 0.5
        for a in range(3):
            d = torch.rand(3000, generator=g) * (1.0 / (GRID[a] - 1)) + 1e-6
            sgn = torch.where(torch.rand(3000, generator=g) < 0.5, -1.0, 1.0)
            x[:, a] = torch.where(sel[:, a], sgn * (1 + d), x[:, a])
        return x
    if name == "cluster":
        # 6000 points inside one texel of every plane and line
        c = torch.tensor([-1 + 2 * 11.5 / (GRID[0] - 1), -1 + 2 * 4.5 / (GRID[1] - 1), -1 + 2 * 30.5 / (GRID[2] - 1)])
        half = torch.tensor([1.0 / (g_ - 1) for g_ in GRID]) * 0.9
        return c + (torch.rand(6000, 3, generator=g) * 2 - 1) * half
    raise KeyError(name)


def sizes_for(threads_per_point):
    n = _threads() // threads_per_point
    return [1, n, n + 1, 40000, 100000]


CASES = ["random:4096", "texel", "outside", "cluster", "n:1", "n:app", "n:app+1", "n:40000", "n:100000"]


def points(case):
    name, _, arg = case.partition(":")
    if name != "n":
        return point_set(name, int(arg) if arg else None)
    n = {"app": _threads() // 36, "app+1": _threads() // 36 + 1}.get(arg) or int(arg)
    return point_set("random", n)


def _xn(case):
    x = points(case).float()
    return x, x.to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def field():
    from tensoir_b200 import _lib
    _lib.load()
    return Field(0)


def test_second_grid_stride_pass_is_reached():
    """The list lengths of CASES straddle the point where each scatter's grid-stride loop makes a second pass
    (blocks_for caps a launch at 16 CTAs of 128 threads per SM): 36 threads per point for app_products_bwd, 12 for
    density_grad_bwd, 3 for density_bwd."""
    t = _threads()
    n_app = t // 36
    assert n_app * 36 <= t < (n_app + 1) * 36
    assert 40000 * 12 > t and 100000 * 3 > t and 100000 * 36 > 2 * t


@pytest.mark.parametrize("case", CASES)
def test_app_products_fwd_bwd(field, case):
    from tensoir_b200 import _lib
    lib = _lib.load()
    x, xd = _xn(case)
    n = x.shape[0]
    out = torch.empty(n, 144, device=DEV)
    _lib.check(lib.tir_vm_app_products(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(out), _lib.stream_ptr()),
               "app products")
    gout = torch.randn(n, 144, generator=torch.Generator().manual_seed(n)).to(DEV)
    gp, gl, ap, al = grad_shadows(field, "app")
    _lib.check(lib.tir_vm_app_products_bwd(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(gout), ap, al,
                                           _lib.stream_ptr()), "app products bwd")
    torch.cuda.synchronize()
    with f64():
        f = field.oracle(torch.float64)
        for p in f.app_plane + f.app_line:
            p.requires_grad_(True)
        xs = x.to(DEV, torch.float64)
        ps, ls = O._app_products(f, xs)
        want = (ps * ls).t()                               # [n, 3C]: orientation-major, like the kernel's output
        want.backward(gout.double())
        ts = tap_sums(f.app_plane, f.app_line, xs, False, False)
        tu = tap_sums(f.app_plane, f.app_line, xs, False, True)
        mag = torch.cat([t["AP"] * t["AL"] for t in ts], 1)
        unit = torch.cat([t["AP"] * t["AL"] for t in tu], 1)
        check(out, want.detach(), bound(mag, unit), f"app products {case}")
        ga = gout.double().abs().view(n, 3, 48)
        m = scatter(ts, lambda k, t, j: ga[:, k] * t["ptaps"][j][1][:, None] * t["AL"],
                    lambda k, t, j: ga[:, k] * t["ltaps"][j][1][:, None] * t["AP"], 48)
        u = scatter(tu, lambda k, t, j: ga[:, k] * t["ptaps"][j][1][:, None] * t["AL"],
                    lambda k, t, j: ga[:, k] * t["ltaps"][j][1][:, None] * t["AP"], 48)
        check_scatter(gp, gl, [p.grad for p in f.app_plane], [l.grad for l in f.app_line], m, u,
                      f"app products bwd {case}")


@pytest.mark.parametrize("case", CASES)
def test_density_bwd(field, case):
    from tensoir_b200 import _lib
    lib = _lib.load()
    x, xd = _xn(case)
    n = x.shape[0]
    g = torch.randn(n, generator=torch.Generator().manual_seed(n + 1))
    g[::5] = 0.0                                         # the kernel skips zero upstream gradients
    gd = g.to(DEV)
    gp, gl, ap, al = grad_shadows(field, "density")
    _lib.check(lib.tir_vm_density_bwd(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(gd), ap, al,
                                      _lib.stream_ptr()), "density bwd")
    torch.cuda.synchronize()
    with f64():
        f = field.oracle(torch.float64)
        for p in f.density_plane + f.density_line:
            p.requires_grad_(True)
        xs = x.to(DEV, torch.float64)
        (O.density_feature(f, xs) * gd.double()).sum().backward()
        ts = tap_sums(f.density_plane, f.density_line, xs, False, False)
        tu = tap_sums(f.density_plane, f.density_line, xs, False, True)
        ga = gd.double().abs()[:, None]
        m = scatter(ts, lambda k, t, j: ga * t["ptaps"][j][1][:, None] * t["AL"],
                    lambda k, t, j: ga * t["ltaps"][j][1][:, None] * t["AP"], 16)
        u = scatter(tu, lambda k, t, j: ga * t["ptaps"][j][1][:, None] * t["AL"],
                    lambda k, t, j: ga * t["ltaps"][j][1][:, None] * t["AP"], 16)
        check_scatter(gp, gl, [p.grad for p in f.density_plane], [l.grad for l in f.density_line], m, u,
                      f"density bwd {case}")


def _grad_mags(ts, x):
    """sum|terms| of feature [n] and of d feature / d x_hat [n, 3] under the clamped sampler."""
    feat = sum((t["AP"] * t["AL"]).sum(1) for t in ts)
    d = torch.zeros(x.shape[0], 3, dtype=torch.float64, device=DEV)
    for k, t in enumerate(ts):
        sx, sy, sl = t["s"]
        d[:, MAT[k][0]] += sx * (t["AX"] * t["AL"]).sum(1)
        d[:, MAT[k][1]] += sy * (t["AY"] * t["AL"]).sum(1)
        d[:, VEC[k]] += sl * (t["AP"] * t["AZ"]).sum(1)
    return feat, d


@pytest.mark.parametrize("inputs", ["both", "feature", "dfdx"])
@pytest.mark.parametrize("case", CASES)
def test_density_grad_fwd_bwd(field, case, inputs):
    """Feature and d feature / d x_hat with the clamped sampler, and their backward with g_feature and g_dfdx, each
    alone and together (the reference's create_graph=True double backward)."""
    from tensoir_b200 import _lib
    lib = _lib.load()
    if inputs != "both" and case not in ("random:4096", "outside", "cluster", "n:40000", "texel"):
        pytest.skip("one upstream gradient alone: a subset of the point sets")
    # On a texel centre the interpolant has a kink: d feature / d x_hat is one-sided, and which side the kernel takes
    # depends on how the fp32 coordinate rounds (floor of a value within eps32 (G - 1) of an integer).  There only the
    # feature and its g_feature backward (continuous tap weights) have one right answer.
    kink = case == "texel"
    if kink and inputs != "feature":
        pytest.skip("the spatial derivative is one-sided on texel centres")
    x, xd = _xn(case)
    n = x.shape[0]
    feat = torch.empty(n, device=DEV)
    dfdx = torch.empty(n, 3, device=DEV)
    _lib.check(lib.tir_vm_density_grad(C.byref(field.struct), _lib.dptr(xd), n, _lib.dptr(feat), _lib.dptr(dfdx),
                                       _lib.stream_ptr()), "density grad")
    gen = torch.Generator().manual_seed(n + 2)
    gf = torch.randn(n, generator=gen).to(DEV) if inputs in ("both", "feature") else None
    gx = torch.randn(n, 3, generator=gen).to(DEV) if inputs in ("both", "dfdx") else None
    gp, gl, ap, al = grad_shadows(field, "density")
    _lib.check(lib.tir_vm_density_grad_bwd(C.byref(field.struct), _lib.dptr(xd), n,
                                           None if gf is None else _lib.dptr(gf), None if gx is None else _lib.dptr(gx),
                                           ap, al, _lib.stream_ptr()), "density grad bwd")
    torch.cuda.synchronize()
    with f64():
        f = field.oracle(torch.float64)
        for p in f.density_plane + f.density_line:
            p.requires_grad_(True)
        xs = x.to(DEV, torch.float64).requires_grad_(True)
        ft = O.density_feature_with_xyz_grad(f, xs)
        (d,) = torch.autograd.grad(ft.sum(), xs, create_graph=True)
        ts = tap_sums(f.density_plane, f.density_line, xs.detach(), True, False)
        tu = tap_sums(f.density_plane, f.density_line, xs.detach(), True, True)
        mf, md = _grad_mags(ts, xs)
        uf, ud = _grad_mags(tu, xs)
        check(feat, ft.detach(), bound(mf, uf), f"feature {case}")
        if not kink:
            check(dfdx, d.detach(), bound(md, ud), f"dfdx {case}")
        loss = 0
        if gf is not None:
            loss = loss + (ft * gf.double()).sum()
        if gx is not None:
            loss = loss + (d * gx.double()).sum()
        loss.backward()
        agf = gf.double().abs() if gf is not None else torch.zeros(n, dtype=torch.float64, device=DEV)
        agx = gx.double().abs() if gx is not None else torch.zeros(n, 3, dtype=torch.float64, device=DEV)

        def coef_p(k, t, j):
            sx, sy, sl = t["s"]
            _, w, dwx, dwy = t["ptaps"][j]
            g0, g1, gv = agx[:, MAT[k][0]] * sx, agx[:, MAT[k][1]] * sy, agx[:, VEC[k]] * sl
            return (agf * w + g0 * dwx + g1 * dwy)[:, None] * t["AL"] + (gv * w)[:, None] * t["AZ"]

        def coef_l(k, t, j):
            sx, sy, sl = t["s"]
            _, w, kz = t["ltaps"][j]
            g0, g1, gv = agx[:, MAT[k][0]] * sx, agx[:, MAT[k][1]] * sy, agx[:, VEC[k]] * sl
            return t["AP"] * (agf * w + gv * kz)[:, None] + w[:, None] * (g0[:, None] * t["AX"] + g1[:, None] * t["AY"])
        m = scatter(ts, coef_p, coef_l, 16)
        u = scatter(tu, coef_p, coef_l, 16)
        check_scatter(gp, gl, [p.grad for p in f.density_plane], [l.grad for l in f.density_line], m, u,
                      f"density grad bwd {case} {inputs}")


# ------------------------------------------------------------------------------------------------------------------
# compositing: raw2alpha over ray segments and its backward
# ------------------------------------------------------------------------------------------------------------------
SCALE = 25.0


def composite_case():
    """Ray segments of a flat sample list: empty and one-sample segments, runs of sigma = 0, near-opaque samples whose
    fp32 alpha rounds to 1 (sigma * dist * scale > 17.4: exp < 2^-25), transmittance underflowing to 0 after a few of
    them, ordinary rays; with z for the depth sum."""
    g = torch.Generator().manual_seed(5)
    lens = [0, 1, 1, 7, 0, 40, 60, 3, 25, 0, 12, 60, 33, 1, 48, 20] * 4
    rows = []
    for r, L in enumerate(lens):
        s = torch.rand(L, generator=g) * 3
        kind = r % 8
        if kind == 1 and L > 4:
            s[L // 4: L // 2] = 0.0                          # a run of empty space
        if kind == 2 and L > 2:
            s[L // 2] = 2000.0                               # one near-opaque sample (sigma d >= 50)
        if kind == 3 and L > 8:
            s[2:8] = 1500.0                                  # several: T = prod(1e-10) underflows to 0
        if kind == 5:
            s[:] = 0.0
        d = torch.rand(L, generator=g) * 0.02 + 0.001
        z = torch.cumsum(d, 0) + 2.0
        rows.append((s, d, z))
    offsets = torch.tensor([0] + lens).cumsum(0)
    return rows, offsets


def padded(rows, dtype, limit=None, offsets=None):
    S = max(1, max(r[0].numel() for r in rows))
    sig = torch.zeros(len(rows), S, dtype=dtype)
    dist = torch.zeros(len(rows), S, dtype=dtype)
    z = torch.zeros(len(rows), S, dtype=dtype)
    valid = torch.zeros(len(rows), S, dtype=torch.bool)
    for r, (s, d, zz) in enumerate(rows):
        L = s.numel()
        if limit is not None:
            L = max(0, min(L, limit - int(offsets[r])))
        sig[r, :L], dist[r, :L], z[r, :L] = s[:L].to(dtype), d[:L].to(dtype), zz[:L].to(dtype)
        valid[r, :L] = True
    return sig, dist, z, valid


def reference(rows, dtype, g_w, g_acc, g_depth, limit=None, offsets=None):
    """raw2alpha on padded per-ray rows (padding: sigma = dist = 0, alpha = 0) in ``dtype``, with acc / depth and the
    gradient of sum(g_w w) + sum(g_acc acc) + sum(g_depth depth) w.r.t. sigma."""
    sig, dist, z, valid = padded(rows, dtype, limit, offsets)
    sig = sig.to(DEV).requires_grad_(True)
    dist, z, valid = dist.to(DEV) * SCALE, z.to(DEV), valid.to(DEV)
    alpha, w, T_last = O.raw2alpha(sig, dist)
    with torch.no_grad():                 # the transmittance in front of each sample (raw2alpha's T[:, :-1])
        T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1. - alpha + 1e-10], -1), -1)[:, :-1]
    acc = w.sum(1)
    depth = (w * z).sum(1)
    gw = torch.zeros_like(w)
    gw[valid] = g_w[:int(valid.sum())].to(DEV, dtype)
    loss = (w * gw).sum() + (acc * g_acc.to(DEV, dtype)).sum() + (depth * g_depth.to(DEV, dtype)).sum()
    (gs,) = torch.autograd.grad(loss, sig)
    return dict(alpha=alpha.detach(), w=w.detach(), T=T, T_last=T_last.detach().reshape(-1), acc=acc.detach(),
                depth=depth.detach(), g_sigma=gs, valid=valid, gw=gw, z=z, dist=dist, sigma=sig.detach())


def regimes(r64):
    """fp64 regime: the samples of a ray before its first sample whose fp32 alpha rounds to 1 (fp64 1 - alpha < 2^-24);
    those from there on are in the fp32 regime."""
    valid = r64["valid"]
    opaque = valid & ((1 - r64["alpha"]) < 2.0 ** -24)
    n_rays, S = valid.shape
    first = torch.where(opaque.any(1), opaque.float().argmax(1), torch.full((n_rays,), S, device=DEV))
    idx = torch.arange(S, device=DEV)[None]
    return valid & (idx < first[:, None]), valid & (idx >= first[:, None]), opaque.any(1)


def forward_bounds(r64, fp64_ok):
    """Per sample: eps32 * 8 (i + 1) T_i (sample i of its ray multiplies i rounded factors into T, and alpha_i is
    exact to eps32 in absolute terms), plus the smallest normal float32 for a T that underflows."""
    pos = r64["valid"].cumsum(1).double()
    return torch.where(fp64_ok, EPS32 * 8 * (pos + 1) * r64["T"] + 2.0 ** -126, torch.zeros_like(pos))


def run_composite(rows, offsets, g_w, g_acc, g_depth, limit=0):
    from tensoir_b200 import _lib
    lib = _lib.load()
    sig = torch.cat([r[0] for r in rows]).to(DEV)
    dist = torch.cat([r[1] for r in rows]).to(DEV)
    z = torch.cat([r[2] for r in rows]).to(DEV)
    n_rays, N = len(rows), sig.numel()
    sentinel = -3.0
    weight, trans = torch.full((N,), sentinel, device=DEV), torch.full((N,), sentinel, device=DEV)
    t_last, acc, depth = (torch.full((n_rays,), sentinel, device=DEV) for _ in range(3))
    off = offsets.to(DEV)
    _lib.check(lib.tir_composite_fwd(_lib.dptr(sig), _lib.dptr(dist), _lib.dptr(off, torch.int64), n_rays, SCALE,
                                     _lib.dptr(weight), _lib.dptr(trans), _lib.dptr(t_last), limit, _lib.dptr(z),
                                     _lib.dptr(acc), _lib.dptr(depth), _lib.stream_ptr()), "composite fwd")
    g_sigma = torch.full((N,), sentinel, device=DEV)
    gw, ga, gd = (t.to(DEV).contiguous() for t in (g_w, g_acc, g_depth))
    _lib.check(lib.tir_composite_bwd(_lib.dptr(sig), _lib.dptr(dist), _lib.dptr(off, torch.int64), n_rays, SCALE,
                                     _lib.dptr(weight), _lib.dptr(trans), _lib.dptr(gw), _lib.dptr(g_sigma), limit,
                                     _lib.dptr(z), _lib.dptr(ga), _lib.dptr(gd), _lib.stream_ptr()), "composite bwd")
    torch.cuda.synchronize()
    return dict(w=weight, T=trans, T_last=t_last, acc=acc, depth=depth, g_sigma=g_sigma)


@pytest.mark.parametrize("terms", ["all", "weight", "acc", "depth"])
def test_composite_vs_fp64(terms):
    """Two regimes per ray (see ``regimes``):
      * before a ray's first sample whose fp32 alpha rounds to 1, fp32 represents the scan: weights, transmittance and
        the sigma gradient are compared with float64.  Forward bound: ``forward_bounds``.  Gradient bound:
        eps32 * c_i * sum|terms| with sum|terms| = d e^{-sigma d} (|g_i| T_i + sum_{j>i} |g_j| w_j / om_i) and
        c_i = 16 (S + sum_{k<=i} 1 / om_k): every om_k = 1 - alpha_k + 1e-10 is exact to eps32 in absolute terms, i.e. to
        eps32 / om_k relative, and enters the products of every later sample (S = samples of the ray).  acc / depth /
        T_last of rays without such a sample: the sum of the per-sample bounds plus eps32 (S + 1) of the value;
      * from that sample on, fp32 has replaced e^{-sigma d} + 1e-10 by 1e-10 and T may underflow to 0: every output and
        gradient must be finite and equal the fp32 autograd of the same expression (torch on the padded rows) within
        1e-4 of the ray's largest |value|."""
    rows, offsets = composite_case()
    n_rays, N = len(rows), int(offsets[-1])
    g = torch.Generator().manual_seed(8)
    g_w = torch.randn(N, generator=g) if terms in ("all", "weight") else torch.zeros(N)
    g_acc = torch.randn(n_rays, generator=g) if terms in ("all", "acc") else torch.zeros(n_rays)
    g_depth = torch.randn(n_rays, generator=g) if terms in ("all", "depth") else torch.zeros(n_rays)
    got = run_composite(rows, offsets, g_w, g_acc, g_depth)
    r64 = reference(rows, torch.float64, g_w, g_acc, g_depth)
    r32 = reference(rows, torch.float32, g_w, g_acc, g_depth)
    valid = r64["valid"]
    fp64_ok, fp32_reg, has_opaque = regimes(r64)
    assert int(fp32_reg.sum()) > 0 and int(fp64_ok.sum()) > 100
    S = valid.sum(1).double()

    def pad(flat_t):
        out = torch.zeros(valid.shape, dtype=torch.float64, device=DEV)
        out[valid] = flat_t.double()
        return out
    fb = forward_bounds(r64, fp64_ok)
    for k in ("w", "T"):
        check(pad(got[k])[fp64_ok], r64[k][fp64_ok], fb[fp64_ok], f"{k} fp64 regime")
        scale = r32[k].abs().amax(1, keepdim=True).double().expand_as(fb)
        check(pad(got[k])[fp32_reg], r32[k].double()[fp32_reg], 1e-4 * scale[fp32_reg] + 1e-30, f"{k} fp32 regime")
    clear = ~has_opaque
    for k, extra in (("acc", fb.sum(1)), ("depth", (fb * r64["z"]).sum(1)), ("T_last", fb.amax(1) * (S + 1))):
        b = extra + EPS32 * (S + 1) * r64[k].abs() + 2.0 ** -126
        check(got[k][clear], r64[k][clear], b[clear], f"{k} fp64 regime")
        check(got[k][~clear], r32[k].double()[~clear], 1e-4 * (1 + r32[k].double().abs()[~clear]), f"{k} fp32 regime")
    # backward
    om = 1 - r64["alpha"] + 1e-10
    gw_all = (r64["gw"] + g_acc.to(DEV).double()[:, None] + g_depth.to(DEV).double()[:, None] * r64["z"]) * valid
    tail = (gw_all.abs() * r64["w"]).flip(1).cumsum(1).flip(1) - gw_all.abs() * r64["w"]      # sum_{j>i}
    d = r64["dist"]
    mag = d * torch.exp(-r64["sigma"] * d) * (gw_all.abs() * r64["T"] + tail / om)
    c = 16 * (S[:, None] + torch.where(fp64_ok, 1.0 / om, torch.zeros_like(om)).cumsum(1))
    gs = pad(got["g_sigma"])
    assert bool(torch.isfinite(got["g_sigma"]).all())
    check(gs[fp64_ok], r64["g_sigma"][fp64_ok], (EPS32 * c * mag)[fp64_ok] + 1e-300, f"g_sigma fp64 regime {terms}")
    scale32 = r32["g_sigma"].abs().amax(1, keepdim=True).double().expand_as(gs)
    check(gs[fp32_reg], r32["g_sigma"].double()[fp32_reg], 1e-4 * scale32[fp32_reg] + 1e-30,
          f"g_sigma fp32 regime {terms}")
    # the cases the list was built for are really there
    assert bool((r32["alpha"][valid] == 1.0).any())                        # fp32 alpha rounds to 1
    assert bool(((r32["T"] == 0) & valid).any())                          # transmittance underflows to 0
    assert bool(((r32["sigma"] == 0) & valid).any())                      # empty space inside segments
    assert (offsets[1:] - offsets[:-1]).eq(0).any() and (offsets[1:] - offsets[:-1]).eq(1).any()


def test_composite_limit_cuts_a_segment():
    """A static-capacity list shorter than the real total: the scan stops at ``limit`` in the middle of a segment, the
    rows at and past it are left untouched, and what is computed equals the float64 scan of the truncated segments."""
    rows, offsets = composite_case()
    n_rays = len(rows)
    limit = int(offsets[6]) + 17                   # inside ray 6's 60 samples
    assert int(offsets[6]) < limit < int(offsets[7])
    N = int(offsets[-1])
    g = torch.Generator().manual_seed(9)
    g_w, g_acc, g_depth = torch.randn(N, generator=g), torch.randn(n_rays, generator=g), torch.randn(n_rays, generator=g)
    got = run_composite(rows, offsets, g_w, g_acc, g_depth, limit=limit)
    for k in ("w", "T", "g_sigma"):
        assert bool((got[k][limit:] == -3.0).all()), k                # untouched past the limit
    r64 = reference(rows, torch.float64, g_w, g_acc, g_depth, limit=limit, offsets=offsets)
    valid = r64["valid"]
    assert int(valid.sum()) == limit
    fp64_ok, _, has_opaque = regimes(r64)
    fb = forward_bounds(r64, fp64_ok)
    assert bool(fp64_ok[6].any())
    w = torch.zeros(valid.shape, dtype=torch.float64, device=DEV)
    w[valid] = got["w"][:limit].double()
    check(w[fp64_ok], r64["w"][fp64_ok], fb[fp64_ok], "weight with limit")
    clear = ~has_opaque
    b = fb.sum(1) + EPS32 * (valid.sum(1) + 1) * r64["acc"].abs() + 2.0 ** -126
    check(got["acc"][clear], r64["acc"][clear], b[clear], "acc with limit")
    r32 = reference(rows, torch.float32, g_w, g_acc, g_depth, limit=limit, offsets=offsets)
    scale = r32["g_sigma"].abs().amax(1, keepdim=True).double().expand_as(valid)
    check(got["g_sigma"][:limit], r32["g_sigma"].double()[valid], 1e-4 * scale[valid] + 1e-30, "g_sigma with limit")
