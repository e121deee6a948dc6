"""The secondary path of the training step against float64: the march (csrc/tir_march.cu: the dense secondary instances
behind tir_secondary_radiance(_vol) and the explicit-ray instances behind tir_march_density / tir_march_radiance) and
the list MLP that follows it (csrc/tir_mlp_wgmma.cu, tir_app_mlp), called through the C ABI at the sizes where the
kernels change behaviour: several surface points per CTA (both slots of the point double buffer), several rays per
warp (the carried transmittance of a ray that straddles two gather batches), a second grid-stride pass, list MLP
tiles past the first wave, an appearance list longer than its capacity, and consecutive launches of different sizes.

Reference of the march, per ray and sample:
  * what the kernel decides in float32 is decided in float32 with the kernel's operations: the sample z (table, or
    t_min + step (s + jitter)), the position o + d z, the aabb test and the alpha-mask test (the oracle's functions)
    and the normalised coordinate.  The cosine test is decided in float64: a ray whose float64 cosine lies within
    COS_BAND of 1e-6 may take either branch, but must take it entirely;
  * everything after that is float64: the density feature (the VM gather; for the volume instance the same value,
    since the trilinear interpolation of the vertex sums equals the sum of the factor products), softplus, alpha,
    the transmittance (an invalid sample contributes the factor 1 - 0 + 1e-10, which is 1 in float32, so 1 here),
    the weights, t_last, acc and depth.

Bounds, per entry, in float64 and independent of the order of the scans and atomics:
  * feature: test_vm_kernels_fp64.bound of the gather's tap sums; volume instance: the vertex volume's own fp32 build
    error (18 eps32 of sum|P L| per vertex) interpolated, plus 16 eps32 of the interpolated |D| and the texel
    coordinate's rounding (2 (G - 1) eps32 per axis of the unit-weight tap sum);
  * sigma: sigmoid(x) (|feature error| + eps32 |x|) + 4 eps32 sigma, x = feature + shift;
  * every transmittance factor om = 1 - alpha + 1e-10 is off by eps32 (4 + 2 sigma d + 1 / om) relative (expf of a
    rounded argument, the rounding of 1 - e) plus d e^(-sigma d) / om of the sigma error; T_i gets
    test_vm_kernels_fp64.forward_bounds plus T_i expm1(sum of those over the samples in front of it), and w_i gets
    alpha_i times that plus T_i (eps32 ((2 + sigma d) e^(-sigma d) + 2 alpha) + d e^(-sigma d) |sigma error|);
  * the fp32 regime (test_vm_kernels_fp64.regimes: from a ray's first sample whose fp32 alpha rounds to 1 on, where T
    may underflow to exactly 0): every weight and t_last of the ray is within the bound of T at that sample plus
    2^-21 T there.
Appearance list: unique (ray, sample) pairs, each a valid sample of a marched ray, its coordinate the reference's
float32 one exactly, its weight within bound; membership is w64 > rayMarch_weight_thres except where w64 lies within
its bound of the threshold (counted, reported, and at most 5 % of the valid samples).  Count-parity mode: the mask, density, appearance and
ray counters equal the reference's counts.  Lean mode: the outputs only.

Reference of the list MLP: sum over the kernel's own list rows of w * sigmoid(MLP64(products x light row, view
direction)) per ray, with the split-BF16 bounds of test_heads_kernels_fp64 (gemm_bound) chained through the gather,
basis, PE, W0, ReLU, W1, ReLU, W2 and sigmoid stages (a ReLU pre-activation within its bound of 0 keeps its whole
term), plus the atomics into a prefilled output."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import tensoir_oracle as O                                       # noqa: E402
import test_heads_kernels_fp64 as H                                          # noqa: E402
import test_vm_kernels_fp64 as V                                             # noqa: E402
from test_density_volume_gpu import EPS32, _d64, _factors, _lego_inputs     # noqa: E402

DEV = "cuda:0"
COS_BAND = 4 * EPS32        # float64 cosines this close to 1e-6 may take either branch of the fp32 test
VIS_SENTINEL = -7.0
NEAR, FAR = 0.05, 1.5       # the secondary march's z table (ops.secondary_radiance)
CHUNK = 1 << 19


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dense_grid(vol):
    """CTAs of the dense instance: 3 per SM for the volume instance with a z table, 2 otherwise (launch_instance)."""
    return sms() * (3 if vol else 2)


# ------------------------------------------------------------------------------------------------------------------
# scenes
# ------------------------------------------------------------------------------------------------------------------
class Scene:
    """A TensorVMSplit on the device with the float32 / float64 oracle fields of its density, alpha mask and
    appearance factors."""

    def __init__(self, m, name):
        self.m, self.name = m, name
        self.grid = [int(g) for g in m.gridSize]
        am = m.alphaMask

        def field(dtype):
            f = O.OracleField(aabb=m.aabb.detach().float(), grid_size=self.grid,
                              density_plane=[p.detach().clone() for p in m.density_plane],
                              density_line=[p.detach().clone() for p in m.density_line],
                              app_plane=[p.detach().clone() for p in m.app_plane],
                              app_line=[p.detach().clone() for p in m.app_line], basis_w=None, mlp_rgb=None,
                              alpha_volume=None if am is None else am.alpha_volume.detach().float(),
                              alpha_aabb=None if am is None else am.aabb.detach().float())
            f.to(DEV, dtype)
            f.aabb = m.aabb.detach().float()                  # the decisions stay in float32
            if am is not None:
                f.alpha_volume, f.alpha_aabb = am.alpha_volume.detach().float(), am.aabb.detach().float()
            return f
        self.o32, self.o64 = field(torch.float32), field(torch.float64)
        self.shift, self.scale = float(m.density_shift), float(m.distance_scale)
        self.thres = float(m.rayMarch_weight_thres)
        mlp = m.renderModule.mlp
        self.W = [mlp[i].weight.detach().double() for i in (0, 2, 4)]
        self.B = [mlp[i].bias.detach().double() for i in (0, 2, 4)]
        self.basis = m.basis_mat.weight.detach().double()
        self.ll = m.light_line.weight.detach().double()
        self.box = None


def _random_model(opaque):
    """37 x 18 x 61 on an off-centre box (no axis size repeats) with random factors and a random 23 x 29 x 31 alpha
    mask with empty cells.  ``opaque``: positive factors near 1.5 (features near 108, sigma d near 37), so an occupied
    sample has fp32 alpha 1 and T underflows to exactly 0 after a few of them."""
    from tensoir_b200 import AlphaGridMask, TensorVMSplit
    torch.manual_seed(21 + opaque)
    aabb = torch.tensor([[-1.0, -0.7, -1.3], [1.1, 0.8, 1.2]], device=DEV)
    m = TensorVMSplit(aabb, [37, 18, 61], DEV, density_n_comp=[16] * 3, appearance_n_comp=[48] * 3, app_dim=27,
                      near_far=[2.0, 6.0], shadingMode='MLP_Fea', density_shift=-10, distance_scale=25, pos_pe=2,
                      view_pe=2, fea_pe=2, featureC=128, step_ratio=0.5, fea2denseAct='softplus',
                      normals_kind='derived_plus_predicted', light_rotation=["000", "120"], light_kind='sg',
                      numLgtSGs=128)
    with torch.no_grad():
        for p in list(m.density_plane) + list(m.density_line):
            if opaque:
                p.normal_().mul_(0.1).add_(1.5)
            else:
                p.normal_().mul_(0.9)
        for p in list(m.app_plane) + list(m.app_line):
            p.normal_().mul_(0.3)
    g = torch.Generator().manual_seed(5 + opaque)
    av = torch.rand(1, 1, 31, 29, 23, generator=g)
    av = torch.where(torch.rand(av.shape, generator=g) < 0.35, torch.zeros_like(av), av)
    m.alphaMask = AlphaGridMask(DEV, aabb.clone(), av.to(DEV))
    return m


_SCENES = {}


def scene(name, lego=None):
    """-> (Scene, surface points, normals, light indices) with at least 3x the largest dense grid of points.  ``lego``:
    the lego model of the "lego" scene (default: make_lego_model(128)); its surface points come from its own forward."""
    key = name if lego is None else (name, id(lego))
    if key not in _SCENES:
        from gpu_helpers import load_shrunk_state, model_from_fixture
        n = 3 * dense_grid(True) + 64
        if name == "lego":
            m, surf, nrm, li, _ = _lego_inputs(n_rays=4096, m=lego)
            reps = -(-n // surf.shape[0])
            pts, nrm, li = surf.repeat(reps, 1)[:n], nrm.repeat(reps, 1)[:n], li.repeat(reps)[:n]
        else:
            m = model_from_fixture(load_shrunk_state("B"), DEV) if name == "B" else _random_model(name == "opaque")
            g = torch.Generator().manual_seed(len(name))
            lo, hi = m.aabb[0].cpu(), m.aabb[1].cpu()
            pts = ((lo + hi) / 2 + (hi - lo) / 2 * (torch.rand(n, 3, generator=g) * 2 - 1) * 0.9).to(DEV)
            nrm = F.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV)
            li = (torch.arange(n) % 2).to(DEV, torch.int32)
        pts, nrm = pts.clone().float(), nrm.clone().float()
        # runs of zero normals (non-hit rays), the first and the last point among them, and points outside the aabb
        for a, b in ((0, 3), (n // 2, n // 2 + 5), (n - 2, n)):
            nrm[a:b] = 0.0
        pts[7:12] = m.aabb[1].float() * 1.3
        pts[12] = m.aabb[0].float() * 1.1
        _SCENES[key] = (Scene(m, name), pts.contiguous(), nrm.contiguous(), li.reshape(-1).to(torch.int32).contiguous())
    return _SCENES[key]


def stratified_dirs(sc, n_dirs):
    if n_dirs == 512:
        return sc.m.gen_light_incident_dirs(method='stratified_sampling').to(DEV).float().contiguous()
    g = torch.Generator().manual_seed(n_dirs)
    return F.normalize(torch.randn(n_dirs, 3, generator=g), dim=-1).to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------------------------
# float64 reference of the march
# ------------------------------------------------------------------------------------------------------------------
def _coordinate_term(sc, x):
    """The kernel rounds the texel coordinate (x + 1) / 2 (G - 1) of the float32 coordinate the reference uses as well:
    at most 4 eps32 of x, times |d feature / d x| (test_vm_kernels_fp64._grad_mags), plus 2 eps32 of the unit-weight
    tap sum for the rounding of the tap weights."""
    ts = V.tap_sums(sc.o64.density_plane, sc.o64.density_line, x, False, False, sc.grid)
    tu = V.tap_sums(sc.o64.density_plane, sc.o64.density_line, x, False, True, sc.grid)
    mag, d = V._grad_mags(ts, x)
    unit = sum((t["AP"] * t["AL"]).sum(1) for t in tu)
    return mag, EPS32 * (4 * d.sum(1) + 2 * unit)


def _feature_bound_factor(sc, x):
    mag, coord = _coordinate_term(sc, x)
    return EPS32 * 16 * mag + coord


def _trilerp(vol, lo, n, grid, x, unit):
    """sum over the 8 zero-padded taps of |w| vol (or vol at unit weights) on the box [lo, lo + n) of vertices."""
    taps = [V.axis_taps(x[:, a], grid[a], False, unit) for a in range(3)]
    out = torch.zeros(x.shape[0], dtype=torch.float64, device=DEV)
    for iz, wz, kz in taps[2]:
        for iy, wy, ky in taps[1]:
            for ix, wx, kx in taps[0]:
                keep = (kx * ky * kz) > 0
                lx, ly, lz = ix - lo[0], iy - lo[1], iz - lo[2]
                inside = (lx >= 0) & (lx < n[0]) & (ly >= 0) & (ly < n[1]) & (lz >= 0) & (lz < n[2])
                assert bool((inside | ~keep).all()), "a valid sample reads a vertex outside the volume's box"
                v = vol[lz.clamp(0, n[2] - 1), ly.clamp(0, n[1] - 1), lx.clamp(0, n[0] - 1)]
                out += wx * wy * wz * v * keep
    return out


def _feature_bound_vol(sc, box, x):
    lo, n, D, mag = box
    _, coord = _coordinate_term(sc, x)
    return EPS32 * (18 * _trilerp(mag, lo, n, sc.grid, x, False) + 16 * _trilerp(D.abs(), lo, n, sc.grid, x, False)) \
        + coord


def volume_box(sc):
    """The density volume's box as tir_density_volume_extent gives it, with its float64 vertex sums."""
    from tensoir_b200 import _lib, ops
    if sc.box is None:
        lo, n = (C.c_int32 * 3)(), (C.c_int32 * 3)()
        f = ops.device_field(sc.m).refresh(sc.m)
        _lib.check(_lib.load().tir_density_volume_extent(C.byref(f), lo, n), "extent")
        lo, n = list(lo), list(n)
        D, mag = _d64(_factors(sc.m), lo, n)
        sc.box = (lo, n, D.to(DEV), mag.to(DEV))
    return sc.box


def reference_march(sc, o, d, z, dtype=torch.float64, box=None, bounds=True):
    """March the rays (o, d) [R, 3] through the samples z [R, N] (float32).  -> dict of [R, N] / [R] tensors."""
    R, N = z.shape
    pos = o[:, None, :] + d[:, None, :] * z[..., None]            # float32, the kernel's o + d z
    aabb = sc.o32.aabb
    inbox = ~((aabb[0] > pos) | (pos > aabb[1])).any(dim=-1)
    valid = inbox.clone()
    if sc.o32.alpha_volume is not None:
        valid[inbox] = O.sample_alpha(sc.o32, pos[inbox]) > 0
    dist = torch.cat((z[:, 1:] - z[:, :-1], torch.zeros_like(z[:, :1])), dim=-1)
    xn = O.normalize_coord(sc.o32, pos[valid])
    fld = sc.o64 if dtype == torch.float64 else sc.o32
    feat = torch.zeros(xn.shape[0], dtype=dtype, device=o.device)
    efeat = torch.zeros(xn.shape[0], dtype=torch.float64, device=o.device)
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        for a in range(0, xn.shape[0], CHUNK):
            x = xn[a:a + CHUNK].to(dtype)
            feat[a:a + CHUNK] = O.density_feature(fld, x)
            if bounds:
                efeat[a:a + CHUNK] = (_feature_bound_factor(sc, x) if box is None else _feature_bound_vol(sc, box, x))
    finally:
        torch.set_default_dtype(old)
    x = feat + sc.shift
    sig = torch.zeros(R, N, dtype=dtype, device=o.device)
    sig[valid] = F.softplus(x)
    dd = dist.to(dtype) * sc.scale
    alpha = 1. - torch.exp(-sig * dd)
    om = torch.where(valid, 1. - alpha + 1e-10, torch.ones_like(alpha))
    T_incl = torch.cumprod(om, 1)
    T = torch.cat([torch.ones_like(T_incl[:, :1]), T_incl[:, :-1]], 1)
    r = dict(z=z, pos=pos, inbox=inbox, valid=valid, alpha=alpha, T=T, w=alpha * T, T_last=T_incl[:, -1])
    if not bounds:
        return r
    esig = torch.zeros_like(sig)
    esig[valid] = torch.sigmoid(x) * (efeat + EPS32 * x.abs()) + 4 * EPS32 * F.softplus(x) + 3e-9
    e = torch.exp(-sig * dd)
    rel = torch.where(valid, EPS32 * (4 + 2 * sig * dd + 1 / om) + dd * e / om * esig, torch.zeros_like(om))
    R_excl = torch.cumsum(rel, 1) - rel
    fp64_ok, fp32_reg, opaque = V.regimes(r)
    fb = V.forward_bounds(r, fp64_ok)
    bT = fb + T * torch.expm1(R_excl)
    # w = alpha T: alpha is 1 - expf(-sigma d), off by eps32 ((2 + sigma d) e + 2 alpha) plus d e |sigma error|
    bw = alpha * bT + T * (EPS32 * ((2 + sig * dd) * e + 2 * alpha) + dd * e * esig) + 2.0 ** -126
    S = valid.sum(1).double()
    R_all = rel.sum(1)
    bTl = EPS32 * 8 * (S + 2) * r["T_last"] + r["T_last"] * torch.expm1(R_all) + 2.0 ** -126
    # fp32 regime: from the first sample whose fp32 alpha rounds to 1 on
    first = fp32_reg.float().argmax(1)
    rows = torch.arange(R, device=DEV)
    Tf = T[rows, first]
    pos_f = valid.cumsum(1)[rows, first].double()
    b32 = Tf * (EPS32 * 8 * (pos_f + 1) + torch.expm1(R_excl[rows, first]) + 2.0 ** -21) + 2.0 ** -125
    bw = torch.where(fp64_ok, bw, torch.where(fp32_reg, b32[:, None], torch.zeros_like(bw)))
    bTl = torch.where(opaque, b32, bTl)
    r.update(bw=bw, bT_last=bTl, opaque=opaque, fp32_reg=fp32_reg)
    return r


def table_z(n_rays, n_sample, near=NEAR, far=FAR):
    from tensoir_b200 import ops
    t = ops.equal_z_table(n_sample, near, far, DEV)
    return t, t[None].expand(n_rays, n_sample)


def step_z(sc, cfg, o, d, n_sample, jitter):
    """TensorBase.sample_ray's z in float32 (tensorBase:705-724), with the kernel's step, near and far."""
    aabb = sc.o32.aabb
    vec = torch.where(d == 0, torch.full_like(d, 1e-6), d)
    t_min = torch.minimum((aabb[1] - o) / vec, (aabb[0] - o) / vec).amax(-1).clamp(min=cfg.near, max=cfg.far)
    rng = torch.arange(n_sample, device=DEV, dtype=torch.float32)[None].expand(o.shape[0], -1)
    if jitter is not None:
        rng = rng + jitter[:, None]
    return t_min[:, None] + cfg.step * rng


# ------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------
def ratio(got, want, bnd):
    """largest |got - want| / bound (entries with a zero bound must be exact)"""
    got, want = got.double(), want.double()
    assert bool(torch.isfinite(got).all())
    if got.numel() == 0:
        return 0.0
    err = (got - want).abs()
    assert bool((err[bnd <= 0] == 0).all())
    return float((err / bnd.clamp_min(1e-300)).max())


def decode(buf, n):
    from tensoir_b200 import _lib
    raw = buf[: n * _lib.APP_SAMPLE_BYTES].view(n, _lib.APP_SAMPLE_BYTES)
    fl = raw[:, :16].contiguous().view(torch.float32).view(n, 4)
    it = raw[:, 16:].contiguous().view(torch.int32).view(n, 2)
    return {"xn": fl[:, :3], "weight": fl[:, 3], "ray": it[:, 0].long(), "sample": it[:, 1].long()}


def check_list(sc, ref, lst, row_of, N, what, stats):
    """The appearance list against the reference; ``row_of`` maps the kernel's ray id to the reference row (-1: the
    ray was not marched)."""
    r = row_of[lst["ray"]]
    s = lst["sample"]
    assert bool((r >= 0).all()), f"{what}: listed sample of a ray that was not marched"
    assert bool(((s >= 0) & (s < N)).all()), what
    key = r * N + s
    assert key.unique().numel() == key.numel(), f"{what}: a (ray, sample) pair is listed twice"
    assert bool(ref["valid"][r, s].all()), f"{what}: listed sample is not valid"
    # the coordinate is the reference's float32 one, bit for bit
    pos = ref["pos"][r, s]
    assert torch.equal(lst["xn"], O.normalize_coord(sc.o32, pos)), f"{what}: coordinates"
    q = ratio(lst["weight"], ref["w"][r, s], ref["bw"][r, s])
    assert q <= 1.0, (what, "weights", q)
    listed = torch.zeros_like(ref["valid"])
    listed[r, s] = True
    want = ref["valid"] & (ref["w"] > sc.thres) & ref["marched"][:, None]
    amb = ref["valid"] & ((ref["w"] - sc.thres).abs() <= ref["bw"]) & ref["marched"][:, None]
    bad = (listed != want) & ~amb
    assert not bool(bad.any()), (what, "membership", int(bad.sum()))
    n_amb = int(amb.sum())
    n_dec = int((ref["valid"] & ref["marched"][:, None]).sum())           # samples the threshold is decided on
    assert n_amb <= max(8, n_dec // 20), (what, "ambiguous threshold samples", n_amb, n_dec)
    stats["w"] = max(stats.get("w", 0.0), q)
    stats["amb_thres"] = stats.get("amb_thres", 0) + n_amb
    stats["decided"] = stats.get("decided", 0) + n_dec
    return want, amb


def report(what, stats):
    print(f"{what}: " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in stats.items()))


# ------------------------------------------------------------------------------------------------------------------
# the list MLP reference
# ------------------------------------------------------------------------------------------------------------------
def mlp_reference(planes, lines, grid, W, B, basis, ll, xn, vdir, light, wgt, ray, n_rays):
    """-> (per-ray sum of w * MLP64 [n_rays, 3], per-ray error bound before the atomics, per-ray sum |w * out|,
    rows per ray).  planes / lines: float64 appearance factors (NCHW); ll None: no light row."""
    K0, NF = H.K0, H.NF
    acc = torch.zeros(n_rays, 3, dtype=torch.float64, device=DEV)
    err = torch.zeros_like(acc)
    mag = torch.zeros_like(acc)
    cnt = torch.zeros(n_rays, dtype=torch.float64, device=DEV)
    aW = [w.abs() for w in W]
    ab = basis.abs()
    f = O.OracleField(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), grid_size=list(grid), density_plane=planes,
                      density_line=lines, app_plane=planes, app_line=lines, basis_w=None, mlp_rgb=None)
    with V.f64():
        for a in range(0, xn.shape[0], 1 << 16):
            x = xn[a:a + (1 << 16)].double()
            ps, ls = O._app_products(f, x)
            x0 = (ps * ls).t()
            ts = V.tap_sums(planes, lines, x, False, False, grid)
            tu = V.tap_sums(planes, lines, x, False, True, grid)
            e_x0 = V.bound(torch.cat([t["AP"] * t["AL"] for t in ts], 1),
                           torch.cat([t["AP"] * t["AL"] for t in tu], 1), grid=grid)
            if ll is not None:
                lrow = ll[light[a:a + (1 << 16)].long()]
            else:
                lrow = torch.ones_like(x0)
            xl = x0 * lrow
            e_xl = (e_x0 + EPS32 * x0.abs()) * lrow.abs()
            feat = xl @ basis.t()
            e_feat = H.gemm_bound((xl.abs() + e_xl) @ ab.t(), K0) + e_xl @ ab.t()
            v = vdir[a:a + (1 << 16)].double()
            inp = torch.cat([feat, v, H.pe(feat), H.pe(v)], 1)
            band = torch.tensor([1.0, 2.0], dtype=torch.float64, device=DEV).repeat(NF)
            e_pe = e_feat.repeat_interleave(2, 1) * band
            e_inp = torch.cat([e_feat, torch.zeros_like(v), e_pe + 4 * EPS32, e_pe + 4 * EPS32,
                               torch.full((v.shape[0], 12), 4 * EPS32, dtype=torch.float64, device=DEV)], 1)
            h, e_h = inp, e_inp
            for k in range(2):
                z = h @ W[k].t() + B[k]
                e_z = (H.gemm_bound((h.abs() + e_h) @ aW[k].t(), h.shape[1] if k else 160) + e_h @ aW[k].t()
                       + EPS32 * (z.abs() + B[k].abs()))
                h, e_h = torch.relu(z), e_z              # ReLU is 1-Lipschitz; |h| + e_h feeds the next magnitude
            z3 = h @ W[2].t() + B[2]
            e_z3 = (e_h @ aW[2].t() + EPS32 * (16 + 4 * math.sqrt(H.HID)) * ((h.abs() + e_h) @ aW[2].t())
                    + 2 * EPS32 * B[2].abs())
            y = torch.sigmoid(z3)
            e_y = e_z3 * (y * (1 - y) + e_z3) + 4 * EPS32 * y
            w = wgt[a:a + (1 << 16)].double()[:, None]
            c = w * y
            rr = ray[a:a + (1 << 16)].long()
            acc.index_add_(0, rr, c)
            err.index_add_(0, rr, w.abs() * e_y + EPS32 * c.abs())
            mag.index_add_(0, rr, c.abs())
            cnt.index_add_(0, rr, torch.ones_like(w[:, 0]))
    return acc, err, mag, cnt


def check_mlp(got, prefill, ref, what, stats):
    """got - prefill against the float64 sum; rays without rows must keep their prefill exactly."""
    acc, err, mag, cnt = ref
    # the atomics add the rows of a ray to its prefill: an fp32 sum of cnt + 1 terms (test_heads_kernels_fp64.sum_bound)
    bnd = err + EPS32 * (16.0 + 4.0 * (cnt[:, None] + 1).sqrt()) * (mag + prefill.double().abs().reshape(mag.shape))
    bnd = torch.where(cnt[:, None] > 0, bnd, torch.zeros_like(bnd))
    got = got.double().reshape(acc.shape)
    q = ratio(got - prefill.double().reshape(acc.shape), acc, bnd)
    # rays without a row: untouched, bit for bit
    assert torch.equal(got[cnt == 0], prefill.double().reshape(acc.shape)[cnt == 0]), what
    assert q <= 1.0, (what, "indirect light", q)
    stats["mlp"] = max(stats.get("mlp", 0.0), q)


# ------------------------------------------------------------------------------------------------------------------
# the dense secondary march
# ------------------------------------------------------------------------------------------------------------------
def launch_dense(sc, pts, nrm, li, dirs, N, use_vol, lean=False, capacity=None, guard=0):
    """One tir_secondary_radiance(_vol) call (vis prefilled with a sentinel, indirect with random values) -> dict."""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.device_field import mlp_struct
    lib = _lib.load()
    m = sc.m
    f = ops.device_field(m).refresh(m)
    keep = []
    table, _ = table_z(1, N)
    cfg = ops.march_cfg(m, table=table, keep=keep)
    if lean:
        cfg.flags |= _lib.MARCH_LEAN_COUNTERS
    mlp = mlp_struct(m, "renderModule", keep, light="index")
    n_pts, n_dirs = pts.shape[0], dirs.shape[0]
    vis = torch.full((n_pts, n_dirs), VIS_SENTINEL, device=DEV)
    g = torch.Generator().manual_seed(n_pts * 7 + n_dirs)
    prefill = (torch.rand(n_pts, n_dirs, 3, generator=g) * 2 - 1).to(DEV)
    ind = prefill.clone()
    cnt = ops.new_counters(DEV)
    cap = capacity if capacity is not None else max(1 << 16, 4 * n_pts * n_dirs * -(-N // 32))
    buf = torch.full(((cap + guard) * _lib.APP_SAMPLE_BYTES,), 0xAB, dtype=torch.uint8, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    common = (_lib.dptr(pts), _lib.dptr(nrm), _lib.dptr(li, torch.int32), n_pts, _lib.dptr(dirs), n_dirs,
              C.byref(cfg))
    tail = (_lib.dptr(vis), _lib.dptr(ind), _lib.dptr(buf, torch.uint8), _lib.dptr(count, torch.int32), cap,
            _lib.dptr(cnt, torch.int64), _lib.stream_ptr())
    if use_vol:
        v = ops.density_volume(m, f)
        rc = lib.tir_secondary_radiance_vol(C.byref(f), C.byref(mlp), *common, C.byref(v), *tail)
    else:
        rc = lib.tir_secondary_radiance(C.byref(f), C.byref(mlp), *common, *tail)
    _lib.check(rc, "secondary radiance")
    return dict(vis=vis, ind=ind, prefill=prefill, cnt=cnt, buf=buf, count=count, cap=cap, keep=keep)


def dense_reference(sc, pts, nrm, dirs, N, use_vol):
    """Rays of every (point, direction) whose float64 cosine may pass the test -> (reference, ray ids, certain)."""
    n_dirs = dirs.shape[0]
    cos = nrm.double() @ dirs.double().t()
    cand = (cos > 1e-6 - COS_BAND).reshape(-1)
    certain = (cos > 1e-6 + COS_BAND).reshape(-1)
    ids = cand.nonzero()[:, 0]
    p, dj = ids // n_dirs, ids % n_dirs
    o, d = pts[p].contiguous(), dirs[dj].contiguous()
    _, z = table_z(ids.numel(), N)
    ref = reference_march(sc, o, d, z, box=volume_box(sc) if use_vol else None)
    return ref, ids, certain[ids], cand


def check_dense(sc, pts, nrm, li, dirs, N, use_vol, lean, out, what, ref=None, mlp=True):
    """Every output of one dense launch against the reference; -> stats."""
    n_pts, n_dirs = pts.shape[0], dirs.shape[0]
    if ref is None:
        ref = dense_reference(sc, pts, nrm, dirs, N, use_vol)
    r, ids, certain, cand = ref
    stats = {}
    vis = out["vis"].reshape(-1)
    wrote = vis != VIS_SENTINEL
    # cosine test: a ray outside the band takes the float64 branch; one inside takes either, as a whole
    assert not bool(wrote[~cand].any()), f"{what}: a ray that fails the cosine test was marched"
    amb = ~certain
    marched = certain | (amb & wrote[ids])
    assert bool(wrote[ids][certain].all()), f"{what}: a ray that passes the cosine test has no visibility"
    stats["amb_cos"] = int(amb.sum())
    r["marched"] = marched
    row_of = torch.full((n_pts * n_dirs,), -1, dtype=torch.long, device=DEV)
    row_of[ids[marched]] = torch.nonzero(marched)[:, 0]
    q = ratio(vis[ids][marched], r["T_last"][marched], r["bT_last"][marched])
    assert q <= 1.0, (what, "visibility", q)
    stats["vis"] = q
    stats["T0_rays"] = int((vis[ids][marched] == 0).sum())
    n = int(out["count"])
    assert n <= out["cap"], f"{what}: overflowed"
    lst = decode(out["buf"], n)
    want, _ = check_list(sc, r, lst, row_of, N, what, stats)
    from tensoir_b200 import ops
    c = ops.counters_dict(out["cnt"])
    assert c["overflow"] == 0 and c["rays"] == int(marched.sum()), (what, c)
    assert c["app"] == n, (what, c)
    if not lean:
        mk = marched[:, None]
        if sc.o32.alpha_volume is not None:
            assert c["mask"] == int((r["inbox"] & mk).sum()), (what, "mask counter", c)
        assert c["density"] == int((r["valid"] & mk).sum()), (what, "density counter", c)
        assert abs(c["app"] - int(want.sum())) <= stats["amb_thres"], (what, "app counter", c)
    nv = r["valid"][marched].sum(1)
    stats["max_valid"], stats["rays_no_valid"] = int(nv.max()) if nv.numel() else 0, int((nv == 0).sum())
    if mlp:
        ref_mlp = mlp_reference(sc.o64.app_plane, sc.o64.app_line, sc.grid, sc.W, sc.B, sc.basis, sc.ll, lst["xn"],
                                dirs[lst["ray"] % n_dirs], li[lst["ray"] // n_dirs], lst["weight"], lst["ray"],
                                n_pts * n_dirs)
        check_mlp(out["ind"].reshape(-1, 3), out["prefill"].reshape(-1, 3), ref_mlp, what, stats)
    return stats


# (scene, volume instance, directions, points as "k*grid+e", n_sample, lean)
DENSE_CASES = [
    ("lego", True, 512, "1g+5", 96, False),      # the training step's secondary march
    ("lego", True, 7, "3g+11", 96, False),
    ("random", True, 1, "3g+1", 129, True),
    ("lego", False, 33, "3g+7", 40, False),
    ("lego", False, 512, "1g+3", 96, True),
    ("B", True, 33, "3g+5", 32, False),
    ("B", False, 7, "3g+2", 33, False),
    ("random", True, 33, "3g+9", 129, False),
    ("random", False, 512, "1g+1", 96, False),
    ("opaque", True, 33, "3g+4", 96, False),
    ("opaque", True, 7, "3g+3", 96, True),
    ("opaque", False, 7, "3g+6", 129, False),
]


def _n_pts(spec, vol):
    k, e = spec.split("g+")
    return int(k) * dense_grid(vol) + int(e)


@pytest.mark.parametrize("name,vol,n_dirs,pts_spec,N,lean", DENSE_CASES)
def test_dense_march_and_list_mlp(name, vol, n_dirs, pts_spec, N, lean):
    sc, pts, nrm, li = scene(name)
    n = _n_pts(pts_spec, vol)
    assert pts.shape[0] >= n
    pts, nrm, li = pts[:n].contiguous(), nrm[:n].contiguous(), li[:n].contiguous()
    nrm = nrm.clone()
    nrm[-2:] = 0.0                                     # the last point of this run has a zero normal as well
    dirs = stratified_dirs(sc, n_dirs)
    out = launch_dense(sc, pts, nrm, li, dirs, N, vol, lean)
    torch.cuda.synchronize()
    what = f"{name} {'vol' if vol else 'factor'} dirs {n_dirs} pts {n} N {N} {'lean' if lean else 'count'}"
    st = check_dense(sc, pts, nrm, li, dirs, N, vol, lean, out, what)
    report(what, st)
    if name == "opaque":
        assert st["T0_rays"] >= 20, (what, "rays whose transmittance reaches exactly 0", st["T0_rays"])
    if N >= 96 and name == "random" and n_dirs >= 7:
        # rays whose valid samples straddle the 64-entry queue twice, and rays without any between them
        assert st["max_valid"] > 64 and st["rays_no_valid"] > 0, (what, st)


def test_dense_march_consecutive_launches_reset_the_work_counter():
    """n_pts = large, 1, large on one stream: each launch starts from a zeroed point counter."""
    sc, pts, nrm, li = scene("random")
    n = 3 * dense_grid(True) + 9
    dirs = stratified_dirs(sc, 7)
    for k, m in enumerate((n, 1, n - 5)):
        p, q, l_ = pts[13:13 + m].contiguous(), nrm[13:13 + m].contiguous(), li[13:13 + m].contiguous()
        if m == 1:
            q = F.normalize(torch.ones(1, 3, device=DEV), dim=-1)
        out = launch_dense(sc, p, q, l_, dirs, 96, True)
        torch.cuda.synchronize()
        st = check_dense(sc, p, q, l_, dirs, 96, True, False, out, f"launch {k} ({m} points)")
        report(f"launch {k}", st)


def test_dense_march_overflow():
    """A list capacity below the list length, with a guard behind it: nothing written at or past capacity, the count
    is the full count, the overflow counter is count - capacity, and the stored rows are rows of the full list."""
    from tensoir_b200 import _lib, ops
    sc, pts, nrm, li = scene("lego")
    n = 3 * dense_grid(True) + 11
    pts, nrm, li = pts[:n].contiguous(), nrm[:n].contiguous(), li[:n].contiguous()
    dirs = stratified_dirs(sc, 7)
    full = launch_dense(sc, pts, nrm, li, dirs, 96, True)
    torch.cuda.synchronize()
    total = int(full["count"])
    ref = dense_reference(sc, pts, nrm, dirs, 96, True)
    check_dense(sc, pts, nrm, li, dirs, 96, True, False, full, "full list", ref=ref, mlp=False)
    cap, guard = total // 2, 64
    out = launch_dense(sc, pts, nrm, li, dirs, 96, True, capacity=cap, guard=guard)
    torch.cuda.synchronize()
    B = _lib.APP_SAMPLE_BYTES
    assert bool((out["buf"][cap * B:] == 0xAB).all()), "written at or past capacity"
    assert int(out["count"]) == total
    c = ops.counters_dict(out["cnt"])
    assert c["overflow"] == total - cap and c["app"] == cap, c
    stored, whole = decode(out["buf"], cap), decode(full["buf"], total)
    N = 96
    k_s, k_w = stored["ray"] * N + stored["sample"], whole["ray"] * N + whole["sample"]
    assert bool(torch.isin(k_s, k_w).all()) and k_s.unique().numel() == cap
    # the stored weights are within bound of the float64 weights (vis and the counts: as in the full launch)
    r, ids, _, _ = ref
    row_of = torch.full((pts.shape[0] * dirs.shape[0],), -1, dtype=torch.long, device=DEV)
    row_of[ids] = torch.arange(ids.numel(), device=DEV)
    rr = row_of[stored["ray"]]
    assert ratio(stored["weight"], r["w"][rr, stored["sample"]], r["bw"][rr, stored["sample"]]) <= 1.0


# ------------------------------------------------------------------------------------------------------------------
# explicit rays
# ------------------------------------------------------------------------------------------------------------------
def explicit_rays(sc, n, seed):
    """n rays from a sphere around the box toward random points inside it"""
    g = torch.Generator().manual_seed(seed)
    lo, hi = sc.o32.aabb[0].cpu(), sc.o32.aabb[1].cpu()
    c, half = (lo + hi) / 2, (hi - lo) / 2
    o = c + F.normalize(torch.randn(n, 3, generator=g), dim=-1) * 3.5
    t = c + half * (torch.rand(n, 3, generator=g) * 2 - 1) * 0.8
    d = F.normalize(t - o, dim=-1)
    d[:5, 1] = 0.0                                     # axis-parallel components (the 1e-6 substitute of sample_ray)
    d[:5] = F.normalize(d[:5], dim=-1)
    return o.to(DEV).contiguous(), d.to(DEV).contiguous()


@pytest.mark.parametrize("entry", ["density", "radiance"])
@pytest.mark.parametrize("sampling", ["table", "step", "step_jitter"])
@pytest.mark.parametrize("name", ["random", "opaque"])
def test_explicit_march(name, sampling, entry):
    """tir_march_density / tir_march_radiance on more than two grid-stride passes of rays (num_sms x 2 CTAs x 8
    warps per pass), consecutive rays of a warp sharing gather batches."""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.device_field import mlp_struct
    lib = _lib.load()
    sc = scene(name)[0]
    m = sc.m
    n = 2 * sms() * 2 * 8 * 2 + 37
    o, d = explicit_rays(sc, n, 3 + len(sampling))
    f = ops.device_field(m).refresh(m)
    keep = []
    N = 96 if sampling == "table" else 0
    if sampling == "table":
        table, z = table_z(n, 96, 2.0, 6.0)
        cfg = ops.march_cfg(m, table=table, keep=keep)
    else:
        jit = torch.rand(n, generator=torch.Generator().manual_seed(2)).to(DEV) if sampling == "step_jitter" else None
        cfg = ops.march_cfg(m, n_samples=-1, jitter=jit, keep=keep)
        N = cfg.n_samples
        z = step_z(sc, cfg, o, d, N, jit)
    t_last, acc, depth = (torch.full((n,), VIS_SENTINEL, device=DEV) for _ in range(3))
    cnt = ops.new_counters(DEV)
    if entry == "density":
        _lib.check(lib.tir_march_density(C.byref(f), _lib.dptr(o), _lib.dptr(d), n, C.byref(cfg), _lib.dptr(t_last),
                                         _lib.dptr(acc), _lib.dptr(depth), _lib.dptr(cnt, torch.int64),
                                         _lib.stream_ptr()), "march density")
    else:
        mlp = mlp_struct(m, "renderModule", keep, light="index")
        li = (torch.arange(n, device=DEV) % 2).to(torch.int32)
        prefill = (torch.rand(n, 3, generator=torch.Generator().manual_seed(4)) * 2 - 1).to(DEV)
        rgb = prefill.clone()
        cap = 8 * n * 8
        buf = torch.empty(cap * _lib.APP_SAMPLE_BYTES, dtype=torch.uint8, device=DEV)
        count = torch.zeros(1, dtype=torch.int32, device=DEV)
        _lib.check(lib.tir_march_radiance(C.byref(f), C.byref(mlp), _lib.dptr(o), _lib.dptr(d),
                                          _lib.dptr(li, torch.int32), n, C.byref(cfg), _lib.dptr(t_last),
                                          _lib.dptr(acc), _lib.dptr(depth), _lib.dptr(rgb),
                                          _lib.dptr(buf, torch.uint8), _lib.dptr(count, torch.int32), cap,
                                          _lib.dptr(cnt, torch.int64), _lib.stream_ptr()), "march radiance")
    torch.cuda.synchronize()
    r = reference_march(sc, o, d, z)
    r["marched"] = torch.ones(n, dtype=torch.bool, device=DEV)
    what = f"{name} {sampling} {entry} {n} rays"
    stats = {"vis": ratio(t_last, r["T_last"], r["bT_last"])}
    S = r["valid"].sum(1).double()
    for k, val, extra in (("acc", r["w"].sum(1), r["bw"].sum(1)),
                          ("depth", (r["w"] * r["z"].double()).sum(1), (r["bw"] * r["z"].double().abs()).sum(1))):
        b = extra + EPS32 * (S + 1) * val.abs() + 2.0 ** -126
        stats[k] = ratio(acc if k == "acc" else depth, val, b)
    assert max(stats["vis"], stats["acc"], stats["depth"]) <= 1.0, (what, stats)
    c = ops.counters_dict(cnt)
    assert c["rays"] == n and c["mask"] == int(r["inbox"].sum()) and c["density"] == int(r["valid"].sum()), (what, c)
    stats["T0_rays"] = int((t_last == 0).sum())
    if entry == "radiance":
        nl = int(count)
        lst = decode(buf, nl)
        check_list(sc, r, lst, torch.arange(n, device=DEV), N, what, stats)
        assert c["app"] == nl and c["overflow"] == 0
        ref_mlp = mlp_reference(sc.o64.app_plane, sc.o64.app_line, sc.grid, sc.W, sc.B, sc.basis, sc.ll, lst["xn"],
                                d[lst["ray"]], li[lst["ray"]], lst["weight"], lst["ray"], n)
        check_mlp(rgb, prefill, ref_mlp, what, stats)
    report(what, stats)
    if name == "opaque":
        assert stats["T0_rays"] >= 20, (what, stats)


# ------------------------------------------------------------------------------------------------------------------
# the list MLP on hand-built lists
# ------------------------------------------------------------------------------------------------------------------
def _lengths():
    w = 2 * 64 * sms()                                 # rows of one wave: 2 warpgroups x 64 rows x every SM
    return {"1": 1, "63": 63, "64": 64, "65": 65, "wave-1": w - 1, "wave+1": w + 1, "3wave+17": 3 * w + 17}


@pytest.fixture(scope="module")
def vm_field():
    from tensoir_b200 import _lib
    _lib.load()
    return V.Field(0)


@pytest.mark.parametrize("light", ["index", "none"])
@pytest.mark.parametrize("cap", ["above", "equal", "below"])
@pytest.mark.parametrize("length", ["1", "63", "64", "65", "wave-1", "wave+1", "3wave+17"])
def test_list_mlp_rows(vm_field, length, cap, light):
    """One row per ray at weight 1, so each row is checked alone; max_samples above the count (full grid, the count
    read on the device), equal to it, and one below it (the last row is not evaluated and its ray keeps its prefill)."""
    from tensoir_b200 import _lib
    lib = _lib.load()
    n = _lengths()[length]
    g = torch.Generator().manual_seed(n * 3 + len(cap) + len(light))
    L = 5
    ll = torch.randn(L, H.K0, generator=g).to(DEV)
    basis = (torch.randn(H.NF, H.K0, generator=g) / 12).to(DEV)
    head = H.Head(g, 3, basis, ll if light == "index" else None, 1 if light == "index" else 0)
    xn = (torch.rand(n, 3, generator=g) * 2.1 - 1.05).to(DEV)             # some taps just outside +-1
    fl = torch.cat([xn, torch.ones(n, 1, device=DEV)], 1).contiguous()
    it = torch.stack([torch.arange(n), torch.full((n,), 5)], 1).to(DEV, torch.int32).contiguous()
    rows = torch.cat([fl.view(torch.uint8), it.view(torch.uint8)], 1).reshape(-1)
    max_samples = {"above": max(2 * n, 4 * 64 * sms()), "equal": n, "below": n - 1}[cap]
    buf = torch.zeros(max(max_samples, n) * _lib.APP_SAMPLE_BYTES, dtype=torch.uint8, device=DEV)
    buf[:rows.numel()] = rows
    count = torch.tensor([n], dtype=torch.int32, device=DEV)
    vd = F.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV).contiguous()
    li = torch.randint(0, L, (n,), generator=g, dtype=torch.int32).to(DEV)
    prefill = (torch.rand(n, 3, generator=g) * 2 - 1).to(DEV)
    rgb = prefill.clone()
    _lib.check(lib.tir_app_mlp(C.byref(vm_field.struct), C.byref(head.mlp), _lib.dptr(buf, torch.uint8),
                               _lib.dptr(count, torch.int32), max_samples, _lib.dptr(vd), 0,
                               _lib.dptr(li, torch.int32) if light == "index" else None, _lib.dptr(rgb),
                               _lib.stream_ptr()), "tir_app_mlp")
    torch.cuda.synchronize()
    k = min(n, max(max_samples, 0))
    W, B = head.w64()
    ref = mlp_reference([p.to(DEV).double() for p in vm_field.aplane], [p.to(DEV).double() for p in vm_field.aline],
                        V.GRID, W, B, basis.double(), ll.double() if light == "index" else None, xn[:k], vd[:k],
                        li[:k], torch.ones(k, device=DEV), torch.arange(k, device=DEV), n)
    stats = {}
    check_mlp(rgb, prefill, ref, f"{n} rows, max_samples {max_samples}, light {light}", stats)
    report(f"{n} rows, max_samples {max_samples}, light {light}", stats)
