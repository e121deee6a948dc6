"""The environment-map relighting kernels against float64: tir_relight_sample and tir_relight_shade (csrc/tir_relight.cu,
per-sample math in csrc/tir_relight_body.h, GGX terms in csrc/tir_ggx.h), and the indirect bounce's
tir_indirect_radiance and tir_indirect_shade (csrc/tir_indirect.cu), called through relighting.py and indirect.py.
The reference starts from the kernel's own fp32 inputs at every stage, so a failure names the stage that made it.

Stage 1, tir_relight_sample: exact, no tolerance.
  * bin == torch.searchsorted(cdf, u, right=True).clamp(max=H*W-1) for every (map, ray, sample) of a hit ray; both
    search the same float64 CDF, so they agree exactly.  The draws include the CDF entries themselves, their float64
    neighbours, 0, and the plateaus of zero-radiance texels.
  * the cosine test: rl_cosine is built from ev_* ops, which the compiler does not contract, so its numpy float32
    restatement decides ``> 1e-6`` exactly as the kernel does; pos >= 0 on exactly the hit samples that pass it.
  * every appended row is rl_surface(ray, depth) (float32 restatement) and dir[bin], bit for bit; the slots are
    distinct and cover [0, count); rows past the capacity are not written but are counted.

Stage 2, tir_relight_shade: per-entry float64 bounds, with the error-carrying arithmetic ``R`` and the GGX reference
``ggx_ref`` of test_shade_kernels_fp64.py (the same tir_ggx.h), on the kernel's own bins, slot map and visibility list.
  * each sample's term (albedo rescale / pi + frac / nom) (vis rgb[bin]) cosr / pdf[bin] follows R's per-operation
    rules (eps32 = 2^-23 per rounding; exp2f 2 ulp); an FMA contraction in rl_contrib rounds once where the rules
    round twice, so it stays inside them;
  * the mean: lane-strided partial sums over ceil(S/32) samples then the 5-level butterfly, a chain of
    ceil(S/32) + 5 additions (R.sum), and one rounded division by S;
  * tone: clamp (1-Lipschitz) and powf's 4 ulp; where the linear value lies within its bound of the sRGB threshold
    the jump between the branches is added (counted as the ``tone`` gate);
  * sign(NoV): a row whose nov lies within its bound of 0 is evaluated again with the other signs and the largest
    difference plus that evaluation's bound is added (the ``sign`` gate);
  * background (rl_background): acosf and atan2f carry the CUDA Math API's maximum errors, 2 and 3 ulp; R carries
    them through phi - 1e-6, the scales by 2 / pi and 1 / pi and the unnormalisation by (H-1) / 2 and (W-1) / 2 to
    a bound e_x, e_y on the texel coordinate.  Bilinear interpolation with zero padding is continuous, and within a
    coordinate error below half a texel its slope along x (y) is at most the largest difference Dx (Dy) of
    horizontally (vertically) adjacent texels of the 4x4 window around the lookup, so the lookup error is at most
    e_x Dx + e_y Dy, plus 8 eps32 sum |w_k rgb_k| for the fp32 weights and the 4-term sum.  At the sun's rim of the
    synthetic map that difference is 400;
  * the composite reads the kernel's own without_bg and acc; acc > thr and acc <= 0.9 are fp32 comparisons of the
    kernel's own acc, so they are exact.
Every bound handed to the comparison must be finite.  Each case reports its ambiguous gates and asserts they stay a
small fraction: sign rows at most 1 % of the hit rows, tone entries at most 1 % of the hit entries.

Stage 3, the indirect bounce: tir_indirect_radiance's Lo is stage 2's mean with view direction -omega and S2 samples,
without tone and clamp.  tir_indirect_shade's direct part is tir_relight_shade's sum bit for bit (same header, same
order): rows without a secondary hit give tir_relight_shade's maps exactly.  Its indirect term is checked against
(1/K) sum_k T w Lo from the kernel's own T, w and Lo (R products, a chain of ceil(K/32) + 5 additions and the
division by K), and the maps through tone(direct + indirect) and the composite.

Cases: n = 4096 and 37 rays, S = 512 and 1; 16 maps in one call, mixing the 2048 x 1024 synthetic HDR map with its
400x sun, 16 x 32, 17 x 31 and 1 x 1 maps; more than 16 maps through relight_chunk_fused on the lego field with its
real visibility march; two chunks written into one [L, R, 3] output at row0 = 0 and row0 = n; rough_stride 1 and 3
and a non-uniform rescale; ray directions on the atan2 seam (y = +-0, x < 0), at both poles and on texel centres;
zero-length normals; acc exactly 0.5 and 0.9; thresholds on both sides of 0.5.

The CPU tests pin the float64 stages to oracle.tensoir_oracle.relight_chunk and its get_light run in float64, hold the
host build (tests/host_relight.cpp) to the bounds, and check that the bounds catch planted errors."""
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_shade_kernels_fp64 import EPS, LO, PI, SENTINEL, SRGB_T, R, _d, check_fin, f32, ggx_ref, tone
from helpers import build_host_lib, use_host
from oracle import tensoir_oracle as O
from tensoir_b200 import _lib, relighting
from tensoir_b200.relight import Environment_Light

DEV = "cuda:0"
ULP_ACOS, ULP_ATAN2 = 2.0, 3.0                 # CUDA Math API maximum ulp errors of acosf and atan2f
COS_MIN = np.float32(1e-6)                     # rl_cosine's test
ACC_T = f32(0.9)                               # rl_composite's threshold


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def hdr_maps(sizes, seed, big=False):
    """{name: [H, W, 3] float32}: random radiance with a block of zero texels (a CDF plateau) where the map has one,
    plus bench.synthetic_hdr() (2048 x 1024, 400x sun) first when ``big``."""
    g = np.random.default_rng(seed)
    maps = {}
    if big:
        import bench
        maps["synthetic"] = bench.synthetic_hdr()
    for k, (h, w) in enumerate(sizes):
        m = g.uniform(0.05, 3.0, (h, w, 3)).astype(np.float32)
        if h * w >= 8:
            m[h // 2, : w // 2] = 0.0                   # a plateau inside the CDF
            m[-1, -2:] = 0.0                            # and a flat tail at 1
        maps[f"m{k}_{h}x{w}"] = m
    return maps


def env_data(light, names, dev):
    """The env_tables array and, per map, the exact tensors it points into."""
    arr, keep = relighting.env_tables(light, names)
    maps = [dict(H=int(arr[k].H), W=int(arr[k].W), rgb=keep[4 * k], dir=keep[4 * k + 1], pdf=keep[4 * k + 2],
                 cdf=keep[4 * k + 3]) for k in range(len(names))]
    return arr, keep, maps


def make_chunk(n, rough_stride, seed, first_map, dev, thr=0.5):
    """fp32 rays and maps of one chunk.  Row i has class i % 12: 0/1 direction on the atan2 seam with y = +0 / -0,
    2/3 at the poles, 4 the centre of a texel of ``first_map`` (a miss: a hit whose sample direction is its own ray
    direction has a zero half vector, which no bound covers), 5 a zero-length normal, 6 acc = 0.5, 7 acc = 0.9,
    8 acc just above 0.9, 9 a miss; the rest hit with acc in (0.5, 1)."""
    g = torch.Generator().manual_seed(seed)
    d = F.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1)
    cls = torch.arange(n) % 12
    for c, sy in ((0, 1.0), (1, -1.0)):
        s = cls == c
        d[s, 0] = -d[s, 0].abs() - 0.1
        d[s, 1] = 0.0 * sy
        d[s] = F.normalize(d[s], dim=-1)
        d[s, 1] = 0.0 * sy                              # keeps the sign of zero
    d[cls == 2] = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    d[cls == 3] = torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64)
    tex = torch.randint(0, first_map["dir"].shape[0], (int((cls == 4).sum()),), generator=g)
    d = d.float()
    d[cls == 4] = first_map["dir"].cpu()[tex]
    rays = torch.cat([torch.randn(n, 3, generator=g) * 0.5, d], 1)
    normal = (F.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1)
              * (torch.rand(n, 1, generator=g, dtype=torch.float64) * 1.5 + 0.5)).float()
    normal[cls == 5] = 0.0
    acc = torch.rand(n, generator=g) * 0.5 + 0.5
    acc[cls == 6] = 0.5
    acc[cls == 7] = ACC_T
    acc[cls == 8] = float(np.nextafter(np.float32(ACC_T), np.float32(1)))
    miss = (cls == 4) | (cls == 9)
    acc[miss] = torch.rand(int(miss.sum()), generator=g) * thr
    rough = torch.rand(n, rough_stride, generator=g) * 0.9 + 0.09
    x = dict(rays=rays, depth=torch.rand(n, generator=g) * 1.5 + 0.5, normal=normal,
             albedo=torch.rand(n, 3, generator=g), rough=rough, fresnel=torch.rand(n, 3, generator=g), acc=acc)
    return {k: v.to(dev).contiguous() for k, v in x.items()}


def special_uniforms(u, maps, seed):
    """Overwrite some draws of u [L, n, S] with CDF entries, their float64 neighbours, 0 and plateau values."""
    g = torch.Generator().manual_seed(seed)
    L, n, S = u.shape
    for l, e in enumerate(maps):
        cdf = e["cdf"].cpu()
        pick = cdf[torch.randint(0, cdf.numel(), (n * S // 8,), generator=g)]
        vals = torch.cat([pick, torch.nextafter(pick, torch.zeros_like(pick)), torch.nextafter(pick, torch.ones_like(pick)),
                          torch.zeros(16, dtype=torch.float64)]).clamp(0, float(np.nextafter(1.0, 0.0)))
        flat = u[l].reshape(-1)
        where = torch.randperm(flat.numel(), generator=g)[:vals.numel()].to(u.device)
        flat[where] = vals.to(u.device)
    return u


def vis_values(m, seed, dev):
    """A visibility list: uniform values with exact 0s and 1s."""
    g = torch.Generator().manual_seed(seed)
    v = torch.rand(max(m, 1), generator=g)
    w = torch.rand(max(m, 1), generator=g)
    v[w < 0.2] = 0.0
    v[w > 0.8] = 1.0
    return v.to(dev)


# ------------------------------------------------------------------------------------------------------------------
# stage 1: the sampler, restated exactly
# ------------------------------------------------------------------------------------------------------------------
def bins_ref(cdf, u, right=True):
    return torch.searchsorted(cdf, u, right=right).clamp(max=cdf.numel() - 1)


def cosine32(L, n):
    """rl_cosine in numpy float32: (L0 n0 + L1 n1) + L2 n2, every operation rounded."""
    L, n = L.cpu().numpy(), n.cpu().numpy()
    return torch.from_numpy((L[..., 0] * n[..., 0] + L[..., 1] * n[..., 1]) + L[..., 2] * n[..., 2])


def surface32(rays, depth):
    """rl_surface in numpy float32: o + depth d."""
    r, t = rays.cpu().numpy(), depth.cpu().numpy()
    return torch.from_numpy(r[:, :3] + t[:, None] * r[:, 3:])


def check_sample(maps, x, u, thr, bins, pos, list_o, list_d, count, what, right=True):
    """Every output of one tir_relight_sample call (list rows < count written) against the exact restatement."""
    n = x["acc"].shape[0]
    hit = (x["acc"] > thr).cpu()
    surf = surface32(x["rays"], x["depth"])
    bins, pos, list_o, list_d = bins.cpu(), pos.cpu(), list_o.cpu(), list_d.cpu()
    slots = []
    for l, e in enumerate(maps):
        b, p = bins[l].long(), pos[l].long()
        want = bins_ref(e["cdf"], u[l], right).cpu()
        assert torch.equal(b[hit], want[hit]), (what, "bin", l)
        assert bool((b[~hit] == 0).all()) and bool((p[~hit] == -1).all()), (what, "non-hit rows", l)
        dirs = e["dir"].cpu()
        ok = hit[:, None] & (cosine32(dirs[b], x["normal"].cpu()[:, None]) > COS_MIN)
        assert torch.equal(p >= 0, ok), (what, "cosine set", l)
        assert torch.equal(list_d[p[ok]], dirs[b[ok]]), (what, "list_d", l)
        assert torch.equal(list_o[p[ok]], surf[:, None].expand(n, u.shape[2], 3)[ok]), (what, "list_o", l)
        slots.append(p[ok])
    slots = torch.cat(slots)
    assert int(count) == slots.numel(), (what, "count")
    assert torch.equal(slots.sort().values, torch.arange(slots.numel())), (what, "slots")


# ------------------------------------------------------------------------------------------------------------------
# stage 2: the shading, in float64 with bounds
# ------------------------------------------------------------------------------------------------------------------
def background_ref(e, d, plant=None):
    """rl_background of directions d [m,3] (fp32) under map e -> R [m,3] (module docstring)."""
    H, W = e["H"], e["W"]
    d = d.double()
    ac, th = torch.acos(d[:, 2]), torch.atan2(d[:, 1], d[:, 0])
    phi = R(ac, ULP_ACOS * EPS * ac.abs()) - LO
    theta = R(th, ULP_ATAN2 * EPS * th.abs())
    qy = (phi / PI) * 2.0 - 1.0
    qx = (-theta) / PI
    ix = ((qx + 1.0) / 2.0) * float(W if plant == "W" else W - 1)
    iy = ((qy + 1.0) / 2.0) * float(H - 1)
    assert bool((ix.e < 0.5).all() and (iy.e < 0.5).all())
    img = F.pad(e["rgb"].double().reshape(H, W, 3).permute(2, 0, 1), (3, 3, 3, 3))    # grid_sample's zero padding
    x0, y0 = ix.v.floor(), iy.v.floor()
    off = torch.arange(4, device=d.device)
    cols = (x0.long() + 2).clamp(0, W + 2)[:, None] + off                              # texels x0-1 .. x0+2
    rows = (y0.long() + 2).clamp(0, H + 2)[:, None] + off
    win = img[:, rows[:, :, None], cols[:, None, :]]                                   # [3, m, 4, 4]
    wx1, wy1 = ix.v - x0, iy.v - y0
    w = torch.stack([(1 - wy1) * (1 - wx1), (1 - wy1) * wx1, wy1 * (1 - wx1), wy1 * wx1])     # [4, m]
    t = torch.stack([win[:, :, 1, 1], win[:, :, 1, 2], win[:, :, 2, 1], win[:, :, 2, 2]], 1)  # [3, 4, m]
    val = (w[None] * t).sum(1)
    dx = (win[..., 1:] - win[..., :-1]).abs().amax((-1, -2))
    dy = (win[:, :, 1:] - win[:, :, :-1]).abs().amax((-1, -2))
    err = ix.e * dx + iy.e * dy + 8 * EPS * (w[None] * t.abs()).sum(1)
    return R(val.t(), err.t())


def linear_ref(e, P, b, q, vis, vis_kind, resc, S, sgn=None, plant=None):
    """The fp32 mean over S of rl_contrib in float64 (R [m,3]) and nov, for rows P (per-row fp32 tensors: rays,
    normal, albedo, rough, fresnel), bins b and slots q [m,S] of map e, and the visibility list."""
    N, Vr = R(P["normal"].double()), R(-P["rays"][:, 3:].double())
    r = P["rough"].double()
    r = r.expand(-1, 3) if r.shape[1] == 1 else r
    rs = resc.double().clone()
    if plant == "rescale":
        rs[1] = 1.0
    A = R(P["albedo"].double()) * R(rs)
    vq = R(vis.double()[q.clamp(min=0).long()])
    vq = 1.0 - vq if vis_kind else vq
    on = q >= 0
    v = R(torch.where(on, vq.v, 0.0), torch.where(on, vq.e, 0.0))
    bl = b.long()
    g = ggx_ref(N, Vr, R(P["fresnel"].double()), R(r), R(e["dir"].double()[bl]), sgn)
    brdf = A[:, None] / PI + g.spec
    term = brdf * (v[..., None] * R(e["rgb"].double()[bl])) * g.cosr[..., None] / R(e["pdf"].double()[bl])[..., None]
    # an exact 0 visibility makes the fp32 term an exact 0, whatever the bound of the finite fp32 brdf
    zero = ((v.v == 0) & (v.e == 0))[..., None]
    term = R(torch.where(zero, 0.0, term.v), torch.where(zero, 0.0, term.e))
    lin = term.sum(1, math.ceil(S / 32) + 5) / float(S - 1 if plant == "S-1" else S)
    return lin, g.nov


def linear_rows(e, P, b, q, vis, vis_kind, resc, S, gates, plant=None):
    """linear_ref with the sign(NoV) kink widened (module docstring)."""
    lin, nov = linear_ref(e, P, b, q, vis, vis_kind, resc, S, plant=plant)
    amb = ((nov.v.abs() <= nov.e) & (nov.e > 0)).nonzero().reshape(-1)
    gates["sign"] += int(amb.numel())
    if amb.numel():
        sub = {k: t[amb] for k, t in P.items()}
        s0 = torch.sign(nov.v[amb])
        for c in (-1.0, 0.0, 1.0):
            alt, _ = linear_ref(e, sub, b[amb], q[amb], vis, vis_kind, resc, S, torch.full_like(s0, c), plant)
            other = (s0 != c).to(alt.v.dtype)[:, None]
            lin.e[amb] += ((alt.v - lin.v[amb]).abs() + alt.e) * other
    return lin


def toned(lin, gates):
    t = lin.clamp(0.0, 1.0)
    gates["tone"] += int((((_d(t.v) - SRGB_T).abs() <= t.e) & (t.e > 0)).sum())
    return tone(lin, 1)


ROW_KEYS = ("rays", "normal", "albedo", "rough", "fresnel")


def check_shade(maps, x, thr, resc, vis_data, vis_kind, out, row0, what, gates, plant=None, block=1024):
    """The rows row0 .. row0 + n of out = (with_bg, without_bg) [L, R, 3] written by one tir_relight_shade call on the
    chunk x and vis_data = (bins, pos, vis), each map against the float64 reference, rows in blocks."""
    bins, pos, vis = vis_data
    with_bg, without_bg = out
    n, S = x["acc"].shape[0], bins.shape[2]
    acc = x["acc"]
    hit = acc > thr
    idx = hit.nonzero().reshape(-1)
    a64 = acc.double()
    acc_t = R(torch.where((a64 < ACC_T) if plant == "lt09" else (a64 <= ACC_T), 0.0, a64))[:, None]
    for l, e in enumerate(maps):
        wo_got, wb_got = without_bg[l, row0:row0 + n], with_bg[l, row0:row0 + n]
        assert bool((wo_got[~hit] == 1).all()), (what, "non-hit rows", l)
        want = R(torch.ones(n, 3, dtype=torch.float64, device=acc.device))
        for s in range(0, idx.numel(), block):
            r = idx[s:s + block]
            P = {k: x[k][r] for k in ROW_KEYS}
            t = toned(linear_rows(e, P, bins[l][r], pos[l][r], vis, vis_kind, resc, S, gates, plant), gates)
            want.v[r], want.e[r] = t.v, t.e
        check_fin(wo_got, want.v, want.e + 1e-300, f"{what}: without_bg map {l}")
        # the composite, from the kernel's own without_bg
        bg = tone(background_ref(e, x["rays"][:, 3:], plant), 1)
        wb = acc_t * R(wo_got.double()) + (1.0 - acc_t) * bg
        check_fin(wb_got, wb.v, wb.e + 1e-300, f"{what}: with_bg map {l}")
    return idx.numel()


def assert_gates(gates, n_hit, what):
    print(f"{what}: ambiguous gates {gates} of {n_hit} hit rows")
    assert gates["sign"] <= max(1, n_hit // 100), (what, gates)
    assert gates["tone"] <= max(3, 3 * n_hit // 100), (what, gates)


class FakeMarch:
    """ops.march_density on the visibility list: records the list and returns vis_values as its visibility, so the
    shading sees exact 0s, exact 1s and uniform values whatever the geometry."""

    def __init__(self, seed):
        self.seed, self.calls = seed, []

    def __call__(self, f, rays_o, rays_d, table=None, counters=None, **kw):
        v = vis_values(rays_o.shape[0], self.seed + len(self.calls), rays_o.device)
        self.calls.append((rays_o.clone(), rays_d.clone()))
        return v, v, None


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference is the oracle's computation, and its bounds hold for the host build and catch planted errors
# ------------------------------------------------------------------------------------------------------------------
def test_reference_matches_oracle_cpu(golden_rotated):
    """On the rotated_g24 fixture: the float64 stages, chained on the oracle's own float64 tables and visibility,
    give oracle.tensoir_oracle.relight_chunk run in float64, and background_ref gives its get_light."""
    fx = golden_rotated
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        d64 = lambda t: t.double() if t.is_floating_point() else t  # noqa: E731
        f = O.field_from_state_dict({k: d64(v) for k, v in fx["state_dict"].items()}, fx["aabb"], fx["grid_size"],
                                    kind=fx["kind"], light_rotation=fx["light_rotation"],
                                    alpha_volume=d64(fx["alpha_volume"]), alpha_aabb=d64(fx["alpha_aabb"]))
        f.aabb, f.alpha_volume, f.alpha_aabb = f.aabb.double(), f.alpha_volume.double(), f.alpha_aabb.double()
        oenv = O.EnvLight({"sunny": fx["env_rgb"]})
        oenv.hdr_rgbs["sunny"] = oenv.hdr_rgbs["sunny"].double()       # the fp32 radiance, exactly
        rays = fx["rays"].double()
        maps = tuple(t.double() for t in fx["relight_maps"])
        idx = fx["relight_idx"]
        S = idx.shape[1]
        ow, owo = O.relight_chunk(f, oenv, "sunny", rays, maps, 1.7, idx, S)
        depth, normal, albedo, rough, fresnel, acc = maps
        hit = acc > 0.5
        # the oracle's visibility of every sample that passes the cosine test
        surf = (rays[:, :3] + depth[:, None] * rays[:, 3:])[hit]
        dirs = oenv.hdr_dir["sunny"].reshape(-1, 3)[idx]
        cos = (dirs * normal[hit][:, None]).sum(-1)
        ok = cos > 1e-6
        nerv, _ = O.compute_transmittance(f, surf[:, None].expand(-1, S, -1)[ok], dirs[ok], 96, 0.05, 1.5)
        pos = torch.full(ok.shape, -1, dtype=torch.int64)
        pos[ok] = torch.arange(int(ok.sum()))
        H, W = fx["env_rgb"].shape[:2]
        e = dict(H=H, W=W, rgb=oenv.hdr_rgbs["sunny"].reshape(-1, 3), dir=oenv.hdr_dir["sunny"].reshape(-1, 3),
                 pdf=oenv.hdr_pdf_return["sunny"].reshape(-1))
        P = dict(rays=rays[hit], normal=normal[hit], albedo=albedo[hit], rough=rough[hit], fresnel=fresnel[hit])
        gates = dict(sign=0, tone=0)
        lin = linear_rows(e, P, idx, pos, nerv, 0, torch.full((3,), 1.7), S, gates)
        wo = tone(lin, 1)
        assert (wo.v - owo[hit]).abs().max() < 1e-6
        bg = background_ref(e, rays[:, 3:])
        # the reference's pi and 1e-6 are the kernel's fp32 constants: they move the lookup by ~1e-6 relative
        want = oenv.get_light("sunny", rays[:, 3:])
        assert bool(((bg.v - want).abs() <= 1e-6 * (1 + want.abs())).all())
        acc_t = torch.where(acc <= ACC_T, 0.0, acc)[:, None]
        full = torch.ones_like(owo)
        full[hit] = wo.v
        wb = acc_t * full + (1 - acc_t) * tone(bg, 1).v
        assert (wb - ow).abs().max() < 1e-6
        # the oracle's own sRGB and clamp in the background, and a direction set with the seam and the poles
        d = torch.cat([F.normalize(torch.randn(500, 3, generator=torch.Generator().manual_seed(3)), dim=-1),
                       torch.tensor([[-1.0, 0.0, 0.0], [-1.0, -0.0, 0.0], [0.0, 0.0, 1.0], [0.0, 0.0, -1.0]])])
        want = oenv.get_light("sunny", d)
        assert bool(((background_ref(e, d).v - want).abs() <= 1e-6 * (1 + want.abs())).all())
    finally:
        torch.set_default_dtype(old)


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_relight"), "host_relight.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


def host_case(maps_np, n, S, rough_stride, thr, vis_kind, seed, monkeypatch):
    """One chunk through the host build of tir_relight_sample / tir_relight_shade, via relight_visibility and
    relight_shade with the FakeMarch list.  -> (maps, x, u, resc, march, (bins, pos, vis), out)."""
    light = Environment_Light(maps_np, device="cpu")
    names = list(maps_np)
    arr, keep, maps = env_data(light, names, "cpu")
    x = make_chunk(n, rough_stride, seed, maps[0], "cpu", thr)
    L = len(names)
    u = special_uniforms(torch.rand(L, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(seed)),
                         maps, seed)
    march = FakeMarch(seed)
    monkeypatch.setattr(relighting.ops, "march_density", march)
    vd = relighting.relight_visibility(types.SimpleNamespace(), arr, L, x["rays"], x["depth"], x["normal"], x["acc"],
                                       u, S, thr, "nerv" if vis_kind == 0 else "nerfactor")
    resc = torch.tensor([1.3, 0.8, 1.05])
    out = (torch.full((L, n, 3), SENTINEL), torch.full((L, n, 3), SENTINEL))
    relighting.relight_shade(arr, L, x["rays"], x["normal"], x["albedo"], x["rough"], x["fresnel"], x["acc"], S, thr,
                             resc, vd, "nerv" if vis_kind == 0 else "nerfactor", out, 0)
    return maps, x, u, resc, march, vd, out


SMALL = [(16, 32), (17, 31), (1, 1), (64, 128)]


@pytest.mark.parametrize("S,rough_stride,vis_kind", [(40, 1, 0), (1, 3, 1), (70, 3, 0)])
def test_host_build_within_bounds_cpu(host_lib, monkeypatch, S, rough_stride, vis_kind):
    maps_np = hdr_maps(SMALL, 3 + S)
    maps_np["m3_64x128"][20:24, 40:46] = 400.0                      # a sun
    maps, x, u, resc, march, vd, out = host_case(maps_np, 97, S, rough_stride, 0.5, vis_kind, S, monkeypatch)
    lo, ld = march.calls[0] if march.calls else (torch.zeros(0, 3), torch.zeros(0, 3))
    check_sample(maps, x, u, 0.5, vd[0], vd[1], lo, ld, lo.shape[0], "host")
    gates = dict(sign=0, tone=0)
    n_hit = check_shade(maps, x, 0.5, resc, vd, vis_kind, out, 0, "host", gates)
    assert_gates(gates, n_hit, "host")


@pytest.mark.parametrize("plant", ["S-1", "right", "W", "rescale", "lt09"])
def test_bounds_catch_planted_errors_cpu(host_lib, monkeypatch, plant):
    """Each planted error in the reference makes the host build's outputs fail the checks: a divisor S - 1,
    searchsorted with right=False, W instead of W - 1 in the column scale, the rescale dropped on one channel, and
    acc < 0.9 instead of acc <= 0.9 in the composite."""
    maps_np = hdr_maps(SMALL, 5)
    maps, x, u, resc, march, vd, out = host_case(maps_np, 97, 40, 1, 0.5, 0, 5, monkeypatch)
    if plant == "right":
        lo, ld = march.calls[0]
        with pytest.raises(AssertionError, match="bin"):
            check_sample(maps, x, u, 0.5, vd[0], vd[1], lo, ld, lo.shape[0], "host", right=False)
        return
    stage = "without_bg" if plant in ("S-1", "rescale") else "with_bg"
    with pytest.raises(AssertionError, match=stage):
        check_shade(maps, x, 0.5, resc, vd, 0, out, 0, "host", dict(sign=0, tone=0), plant=plant)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
MIXED = [(16, 32), (17, 31), (1, 1)]


def mixed_maps(L, seed):
    """L maps: the 2048 x 1024 synthetic HDR map, 16 x 32, 17 x 31, 1 x 1, then smaller random sizes."""
    g = np.random.default_rng(seed)
    sizes = MIXED + [(int(g.integers(1, 40)), int(g.integers(1, 80))) for _ in range(L - 4)]
    return hdr_maps(sizes, seed, big=True)


def run_chunk(arr, L, x, u, S, thr, vis_kind, resc, out, row0, seed, monkeypatch):
    """relight_visibility (with FakeMarch) and relight_shade of one chunk into out at row0."""
    march = FakeMarch(seed)
    monkeypatch.setattr(relighting.ops, "march_density", march)
    eq = "nerv" if vis_kind == 0 else "nerfactor"
    vd = relighting.relight_visibility(types.SimpleNamespace(), arr, L, x["rays"], x["depth"], x["normal"], x["acc"],
                                       u, S, thr, eq)
    relighting.relight_shade(arr, L, x["rays"], x["normal"], x["albedo"], x["rough"], x["fresnel"], x["acc"], S, thr,
                             resc, vd, eq, out, row0)
    torch.cuda.synchronize()
    lo, ld = march.calls[0] if march.calls else (torch.zeros(0, 3, device=DEV),) * 2
    return vd, lo, ld


# (maps, rays, samples, rough_stride, vis_kind, thr)
CASES = [(16, 4096, 512, 1, 0, 0.5), (16, 37, 1, 3, 1, float(np.nextafter(np.float32(0.5), np.float32(0)))),
         (4, 4096, 1, 3, 0, 0.5), (4, 37, 512, 1, 1, 0.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("L,n,S,rough_stride,vis_kind,thr", CASES)
def test_relight_kernels_vs_fp64(L, n, S, rough_stride, vis_kind, thr, monkeypatch):
    """Two chunks of n rays into one [L, 2n + 3, 3] output at row0 = 0 and n, every stage checked; the last rows keep
    their sentinel."""
    _lib.load()
    seed = L * 1000 + n + S
    light = Environment_Light(mixed_maps(L, seed), device=DEV)
    names = list(light.hdr_rgbs)
    arr, keep, maps = env_data(light, names, DEV)
    resc = torch.tensor([1.25, 0.75, 1.0], device=DEV)
    out = (torch.full((L, 2 * n + 3, 3), SENTINEL, device=DEV), torch.full((L, 2 * n + 3, 3), SENTINEL, device=DEV))
    what = f"maps {L} rays {n} samples {S} stride {rough_stride} vis_kind {vis_kind} thr {thr}"
    gates = dict(sign=0, tone=0)
    n_hit = 0
    for k, row0 in enumerate((0, n)):
        x = make_chunk(n, rough_stride, seed + k, maps[0], DEV, thr)
        u = torch.rand(L, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(seed + k))
        u = special_uniforms(u, maps, seed + k).to(DEV) if k == 0 else u.to(DEV)
        vd, lo, ld = run_chunk(arr, L, x, u, S, thr, vis_kind, resc, out, row0, seed + k, monkeypatch)
        check_sample(maps, x, u, thr, vd[0], vd[1], lo, ld, lo.shape[0], f"{what} chunk {k}")
        n_hit += check_shade(maps, x, thr, resc, vd, vis_kind, out, row0, f"{what} chunk {k}", gates)
    assert bool((out[0][:, 2 * n:] == SENTINEL).all() and (out[1][:, 2 * n:] == SENTINEL).all()), what
    assert_gates(gates, n_hit * L, what)


@pytest.mark.gpu
def test_sample_capacity():
    """tir_relight_sample with a capacity below the appended total: rows at or past it get pos -1 and are not
    written, count still counts them."""
    lib = _lib.load()
    L, n, S = 4, 4096, 64
    light = Environment_Light(hdr_maps(MIXED + [(32, 64)], 9), device=DEV)
    names = list(light.hdr_rgbs)
    arr, keep, maps = env_data(light, names, DEV)
    x = make_chunk(n, 1, 9, maps[0], DEV)
    u = torch.rand(L, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(9)).to(DEV)
    total = L * n * S
    bins = torch.empty(L, n, S, dtype=torch.int32, device=DEV)
    pos = torch.empty(L, n, S, dtype=torch.int32, device=DEV)
    list_o = torch.full((total, 3), SENTINEL, device=DEV)
    list_d = torch.full((total, 3), SENTINEL, device=DEV)
    count = torch.zeros(1, dtype=torch.int64, device=DEV)
    P = _lib.dptr
    _lib.check(lib.tir_relight_sample(arr, L, P(x["rays"]), P(x["depth"]), P(x["normal"]), P(x["acc"]), n, S, 0.5,
                                      P(u, torch.float64), P(bins, torch.int32), P(pos, torch.int32), P(list_o),
                                      P(list_d), total, P(count, torch.int64), _lib.stream_ptr()), "full")
    full = int(count)
    cap = full // 3
    pos2 = torch.empty_like(pos)
    lo2, ld2 = torch.full_like(list_o, SENTINEL), torch.full_like(list_d, SENTINEL)
    count.zero_()
    _lib.check(lib.tir_relight_sample(arr, L, P(x["rays"]), P(x["depth"]), P(x["normal"]), P(x["acc"]), n, S, 0.5,
                                      P(u, torch.float64), P(bins, torch.int32), P(pos2, torch.int32), P(lo2),
                                      P(ld2), cap, P(count, torch.int64), _lib.stream_ptr()), "capped")
    torch.cuda.synchronize()
    assert int(count) == full
    kept = pos2 >= 0
    assert int(kept.sum()) == cap and bool(((pos >= 0) | ~kept).all())
    assert torch.equal(pos2[kept].sort().values.long(), torch.arange(cap, device=DEV))
    assert bool((lo2[cap:] == SENTINEL).all() and (ld2[cap:] == SENTINEL).all())
    assert not bool((lo2[:cap] == SENTINEL).any())
    # the kept rows hold their samples
    p = pos2[kept].long()
    b = bins[kept].long()
    lidx = torch.arange(L, device=DEV)[:, None, None].expand(L, n, S)[kept]
    for l, e in enumerate(maps):
        s = lidx == l
        assert torch.equal(ld2[p[s]], e["dir"][b[s]])


@pytest.fixture(scope="module")
def lego():
    from tensoir_b200.synthetic import make_lego_model
    _lib.load()
    return make_lego_model(128, DEV)


def lego_chunk(model, n=4096, seed=0):
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    ds = SyntheticViews(hemisphere_poses(1, seed=seed), 96, 96)
    rays = ds[0]["rays"].to(DEV)[:n]
    li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        _, depth, normal, albedo, rough, fresnel, acc, *_ = model(rays, li, is_train=False, white_bg=True,
                                                                  ndc_ray=False, N_samples=-1)
    return rays, (depth, normal, albedo, rough, fresnel, acc)


@pytest.mark.gpu
def test_lego_more_maps_than_one_call_vs_fp64(lego, monkeypatch):
    """relight_chunk_fused on the lego field with 18 maps (two groups) and its real visibility march: each group's
    maps against the float64 reference on the bins, slots and visibility the march gave."""
    L = _lib.RELIGHT_MAX_LIGHTS + 2
    light = Environment_Light(mixed_maps(L, 17), device=DEV)
    names = list(light.hdr_rgbs)
    arr, keep, maps = env_data(light, names, DEV)
    rays, pm = lego_chunk(lego)
    n, S = rays.shape[0], relighting.NUM_SAMPLES
    u = torch.rand(L, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(17)).to(DEV)
    seen = []
    real = relighting.relight_visibility

    def record(*a, **k):
        r = real(*a, **k)
        seen.append(r)
        return r
    monkeypatch.setattr(relighting, "relight_visibility", record)
    resc = torch.tensor([1.1, 0.9, 1.0], device=DEV)
    out = (torch.full((L, n, 3), SENTINEL, device=DEV), torch.full((L, n, 3), SENTINEL, device=DEV))
    relighting.relight_chunk_fused(lego, light, names, rays, pm, resc, u, out=out)
    torch.cuda.synchronize()
    assert len(seen) == 2
    rays_c, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(rays, pm)
    x = dict(rays=rays_c, depth=depth, normal=normal, albedo=albedo, rough=rough, fresnel=fresnel, acc=acc)
    G = _lib.RELIGHT_MAX_LIGHTS
    gates = dict(sign=0, tone=0)
    n_hit = 0
    for gi, g0 in enumerate(range(0, L, G)):
        sub = (out[0][g0:g0 + G], out[1][g0:g0 + G])
        n_hit += check_shade(maps[g0:g0 + G], x, 0.5, resc, seen[gi], 0, sub, 0, f"lego group {gi}", gates)
    assert n_hit > 500
    assert_gates(gates, n_hit * G, "lego")


# ------------------------------------------------------------------------------------------------------------------
# GPU, stage 3: the indirect bounce
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_indirect_kernels_vs_fp64(lego, monkeypatch):
    from tensoir_b200 import indirect
    lib = _lib.load()
    L, K, S, S2 = 3, 16, 512, 32
    light = Environment_Light(hdr_maps([(16, 32), (17, 31), (64, 128)], 23), device=DEV)
    names = list(light.hdr_rgbs)
    arr, keep, maps = env_data(light, names, DEV)
    rays, pm = lego_chunk(lego, seed=3)
    rays_c, (depth, normal, albedo, rough, fresnel, acc) = relighting.chunk_inputs(rays, pm)
    x = dict(rays=rays_c, depth=depth, normal=normal, albedo=albedo, rough=rough, fresnel=fresnel, acc=acc)
    n = rays_c.shape[0]
    resc = torch.tensor([1.2, 0.9, 1.0], device=DEV)
    thr = 0.5
    u_ind = torch.rand(n, K, 2, generator=torch.Generator().manual_seed(4), dtype=torch.float64).to(DEV)
    hits = indirect.secondary_hits(lego, rays_c, depth, normal, albedo, rough, fresnel, acc, resc, u_ind, thr, 'nerv')
    m_h = hits["rays"].shape[0]
    assert m_h > 500, m_h
    mats = indirect.point_materials(lego, hits["rays"][:, :3], hits["xn"])
    mats = tuple(t.detach().float().reshape(m_h, -1).contiguous() for t in mats)
    # Lo through secondary_radiance, with the bins, slots and visibility it marched
    seen = []
    real = indirect.relight_visibility

    def record(*a, **k):
        r = real(*a, **k)
        seen.append(r)
        return r
    monkeypatch.setattr(indirect, "relight_visibility", record)
    Lo = torch.full((L, m_h, 3), SENTINEL, device=DEV)
    u2 = torch.rand(L, m_h, S2, generator=torch.Generator().manual_seed(5), dtype=torch.float64).to(DEV)
    indirect.secondary_radiance(lego, arr, L, hits, mats, resc, Lo, 0, u2, 'nerv')
    torch.cuda.synchronize()
    (b2, p2, v2), = seen
    gates = dict(sign=0, tone=0)
    Ph = dict(rays=hits["rays"], normal=mats[0], albedo=mats[1], rough=mats[2], fresnel=mats[3])
    for l, e in enumerate(maps):
        for s in range(0, m_h, 2048):
            r = slice(s, s + 2048)
            lin = linear_rows(e, {k: t[r] for k, t in Ph.items()}, b2[l][r], p2[l][r], v2, 0, resc, S2, gates)
            check_fin(Lo[l, r], lin.v, lin.e + 1e-300, f"Lo map {l}")
    # the primary rays: tir_relight_shade and tir_indirect_shade on the same bins, slots and visibility
    u = torch.rand(L, n, S, generator=torch.Generator().manual_seed(6), dtype=torch.float64).to(DEV)
    vd = relighting.relight_visibility(lego, arr, L, rays_c, depth, normal, acc, u, S, thr, 'nerv', ordered=True)
    direct = (torch.full((L, n, 3), SENTINEL, device=DEV), torch.full((L, n, 3), SENTINEL, device=DEV))
    relighting.relight_shade(arr, L, rays_c, normal, albedo, rough, fresnel, acc, S, thr, resc, vd, 'nerv', direct, 0)
    P = _lib.dptr
    bins, pos, vis = vd

    def ind_shade(hit):
        wb, wo, ind = (torch.full((L, n, 3), SENTINEL, device=DEV) for _ in range(3))
        _lib.check(lib.tir_indirect_shade(arr, L, P(rays_c), P(normal), P(albedo), P(rough), int(rough.shape[1]),
                                          P(fresnel), P(acc), n, S, thr, P(resc), P(bins, torch.int32),
                                          P(pos, torch.int32), P(vis), 0, K, P(hits["T"]), P(hit, torch.int32),
                                          P(hits["w"]), P(Lo), m_h, P(wb), P(wo), P(ind), n, 0, _lib.stream_ptr()),
                   "tir_indirect_shade")
        torch.cuda.synchronize()
        return wb, wo, ind
    # no secondary hit: tir_relight_shade's maps, bit for bit
    wb0, wo0, ind0 = ind_shade(torch.full_like(hits["hit"], -1))
    assert torch.equal(wo0, direct[1]) and torch.equal(wb0, direct[0])
    assert not bool(ind0.any())
    # with the hits: the indirect term from the kernel's own T, w, Lo
    wb, wo, ind = ind_shade(hits["hit"])
    hit_rows = acc > thr
    h = hits["hit"].long()
    has = (h >= 0)
    any_row = has.any(1) & hit_rows
    assert int(any_row.sum()) > 100
    w_s = torch.where(has, hits["w"][h.clamp(min=0)], 0.0).double()
    for l in range(L):
        Lo_s = torch.where(has[..., None], Lo[l][h.clamp(min=0)], 0.0).double()
        term = R(hits["T"].double()) * R(w_s)[..., None] * R(Lo_s)
        ind_ref = term.sum(1, math.ceil(K / 32) + 5) / float(K)
        r = any_row.nonzero().reshape(-1)
        check_fin(ind[l][r], ind_ref.v[r], ind_ref.e[r] + 1e-300, f"indirect term map {l}")
        assert not bool(ind[l][~any_row].any())
        # the maps: tone(direct + indirect) with the kernel's own indirect term, then the composite
        e = maps[l]
        d_ref = torch.ones(n, 3, dtype=torch.float64, device=DEV)
        d_err = torch.zeros_like(d_ref)
        for s in range(0, r.numel(), 1024):
            rr = r[s:s + 1024]
            lin = linear_rows(e, {k: x[k][rr] for k in ROW_KEYS}, bins[l][rr], pos[l][rr], vis, 0, resc, S, gates)
            t = toned(lin + R(ind[l][rr].double()), gates)
            d_ref[rr], d_err[rr] = t.v, t.e
        check_fin(wo[l][r], d_ref[r], d_err[r] + 1e-300, f"indirect without_bg map {l}")
        assert torch.equal(wo[l][~any_row], wo0[l][~any_row]) and torch.equal(wb[l][~any_row], wb0[l][~any_row])
        a64 = acc.double()
        acc_t = R(torch.where(a64 <= ACC_T, 0.0, a64))[:, None]
        bg = tone(background_ref(e, rays_c[:, 3:]), 1)
        wbr = acc_t * R(wo[l].double()) + (1.0 - acc_t) * bg
        check_fin(wb[l], wbr.v, wbr.e + 1e-300, f"indirect with_bg map {l}")
    assert_gates(gates, int(hit_rows.sum()) * L + m_h * L, "indirect")
