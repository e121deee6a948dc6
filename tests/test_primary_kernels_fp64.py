"""The fused relight-phase primary path (csrc/tir_primary.cu, csrc/tir_epilogue_body.h) stage by stage against
float64: tir_primary_march, tir_primary_app_list, tir_primary_heads and the four-job tir_primary_backward, called
through the C ABI with the model's own job table (primary_fused._jobs), its workspace (primary_fused.Workspace) and
gradient buffers shared the way the autograd node shares them (both BRDF jobs accumulate into the same tensors).

Every stage is compared with a float64 reference built from the kernel's OWN dump of that stage's inputs, so a
failure names the stage that made the error:
  * march: counts, v_ray, v_sample, v_xn, v_z and v_dist equal vm.valid_samples (same cfg, same jitter) bit for bit;
    offsets is the exact int64 exclusive cumsum of counts; status[0] is the total and status[2] is set iff a list
    does not fit its capacity;
  * density: v_feat and v_sigma against the float64 gather (test_vm_kernels_fp64.bound of its tap sums) and
    softplus / ReLU (sigma: sigmoid(x) (|feature error| + eps32 |x|) + 4 eps32 sigma + 3e-9, the 3e-9 for the x > 20
    branch, as in test_secondary_kernels_fp64);
  * compositing: v_weight, v_trans, t_last, acc and depth against float64 raw2alpha of the kernel's own v_sigma, in
    the two regimes of test_vm_kernels_fp64.regimes with the transmittance-factor bounds of
    test_secondary_kernels_fp64 (composite_bounds); in the fp32 regime also against the fp32 scan of the same inputs
    within 1e-4 of the ray's largest value; a_counts, a_offsets and status[1] exactly from the kernel's own v_weight;
  * appearance list: rows a_offsets[r].. are ray r's selected valid rows in increasing order, and a_src / a_ray / a_w /
    a_xn are bit-exact copies; rows at and past cap_app keep the sentinel;
  * heads forward: a_xj (two roundings), x0 of both point sets (check_gather), and every job's input, h1, h2 and
    output (test_heads_kernels_fp64.Stages.forward); dn_feat / dn_dfdx against the clamped-sampler float64 gather;
  * tail forward: packed[r] is the float64 sum over the ray's rows of w x the 14 channels, computed from the kernel's
    own out rows and dn_* with the per-entry error carried through every operation (test_shade_kernels_fp64.R: one
    eps32 per IEEE op, exact product / quotient rules, Lipschitz clamps), plus sum_bound of sum|w v| over the ray's
    rows for the atomics;
  * epilogue: the 8 maps, acc_mask (exactly acc > 0.5 of the kernel's acc) and both losses from the kernel's own
    packed / acc / depth, in R arithmetic (powf 4 ulp, sqrt and quotient rules), the losses with sum_bound;
  * backward, seeded with random map gradients (fresnel and roughness None), a non-NULL g_acc_map and both loss
    gradients: g_packed / g_acc / g_depth (epilogue, R); every job's g_out, g_dn_feat / g_dn_dfdx and g_weight (tail,
    R; g_weight is exactly 0 on every valid row that is not an appearance row); every job's d z2 / d z1 / d feat / d x0
    (Stages.data_grads); the head weight gradients with the two BRDF jobs summed and basis_mat / light_line summed over
    all jobs (Stages.param_grads, whose bounds add); the appearance factors from a float64 scatter of the summed d x0 of
    each point set (check_factor_grads); g_feat from the float64 compositing backward of the kernel's own g_weight /
    g_acc + g_acc_map / g_depth times softplus' or the ReLU mask, bounded from the kernel's arithmetic on its saved
    weights and transmittance (composite_bwd_bound), wherever fp32 resolves om = 1 - alpha + 1e-10 to a relative
    error below 1/2; past that (from 1 - alpha < 2^-22 on) only finiteness; the density factors from the float64 scatter of g_feat at v_xn plus the density-grad double backward
    at a_xn (the two tap-sum magnitudes added).  Every parameter gradient is prefilled with PRE and checked for what
    was added; PRE joins the magnitude of the entry's additions.

Kinks (test_shade_kernels_fp64.Gates): where a float64 gate value lies within its own bound of the threshold, the whole
gated term joins the bound.  The gates are the epilogue's clamp01 masks and sRGB threshold, its normal's 1e-6, the
orientation dot >= 0, the rel_cost max (ties, and the 1e-6 clip), the derived normal's 1e-6 and softplus at 20.  Each
case counts its ambiguous entries per gate and asserts they are at most 1 % of the rows (plus 2).  A derivative gated by
an exact fp32 input (the ReLU of dn_feat, the softplus branch of v_feat) has no ambiguity.  Rows whose coordinate lies
within 4 eps32 (G - 1) of a texel index take a one-sided d feature / d x_hat (test_vm_kernels_fp64); they are counted,
and their dfdx is not compared.

``launch`` drives the entry points and returns a Dump; ``check_stages`` checks a Dump, whichever launch or training
step left it (tests/test_train_step_primary_fp64.py passes it the dumps and captured upstream gradients of real steps).
The radiance-only entry points tir_primary_radiance / _backward have the same pair (``launch_radiance``,
``check_radiance_stages``): march, compositing and the appearance list as above, the head through
test_heads_kernels_fp64, radiance_ray_fwd_kernel's rgb_map / depth_map and radiance_ray_bwd_kernel's g_out, g_weight
(through a_src), g_acc and g_depth in R arithmetic, then the compositing backward and the density scatter.

``test_tail_and_epilogue_backward_match_autograd_cpu`` pins the hand-written tail and epilogue backward to float64
autograd of their forward, away from kinks, to 1e-10, and ``test_chained_references_reproduce_the_oracle_cpu`` pins
the chained references to the oracle's relight-phase maps, losses and parameter gradients."""
import ctypes as C
import math

import pytest
import torch

from oracle import tensoir_oracle as O
from test_heads_kernels_fp64 import (EPS32, NF, Stages, check, check_factor_grads, check_gather, fill_sentinel,
                                     sum_bound)
from test_shade_kernels_fp64 import R, Gates, f32

DEV = "cuda:0"
PRE = 0.25                     # every parameter gradient holds this before the backward
SENT = 3.0                     # fill_sentinel
LO = f32(1e-6)
SRGB_T, SRGB_S, SRGB_A, SRGB_B = f32(0.0031308), f32(12.92), f32(1.055), f32(0.055)
SRGB_E = float(torch.tensor(1.0) / torch.tensor(2.4))                   # 1.f / 2.4f
DS_A, DS_E = float(torch.tensor(1.055) / torch.tensor(2.4)), float(torch.tensor(1.0) / torch.tensor(2.4) - 1.0)
C09, C009 = f32(0.9), f32(0.09)
F0_FP32 = True                 # fixed_fresnel as the kernel gets it (a float argument)
STATS = {}
MAP_NAMES = ("rgb", "depth", "normal", "albedo", "rough", "fresnel", "nd", "no")


# ------------------------------------------------------------------------------------------------------------------
# R helpers
# ------------------------------------------------------------------------------------------------------------------
def rc(v):
    """an exact input (the kernel's own fp32 value)"""
    return R(v)


def rconst(like, c):
    return R(torch.full_like(like.v if isinstance(like, R) else like, c))


def rmax(a, b):
    return R(torch.maximum(a.v, b.v), torch.maximum(a.e, b.e))


def rsqrt_(x):
    s = x.v.sqrt()
    e = torch.minimum(torch.where(s > 0, x.e / s.detach().clamp_min(1e-300), torch.full_like(s, math.inf)),
                      x.e.sqrt())
    return R.rnd(s, e)


def rcol(x, k):
    return R(x.v[..., k], x.e[..., k])


def rstack(xs):
    return R(torch.stack([x.v for x in xs], -1), torch.stack([x.e for x in xs], -1))


def rwhere(c, a, b):
    return R(torch.where(c, a.v, b.v), torch.where(c, a.e, b.e))


def sigmoid(x):
    """1.f / (1.f + expf(-x)): expf's 2 ulp and the argument's error move s by s (1 - s) times their relative size,
    the add and the division by s eps32 each; where expf overflows the kernel returns 0, within 2^-125 of s"""
    s = torch.sigmoid(x.v)
    sd = s.detach()
    return R(s, sd * (1 - sd) * (2 * EPS32 + torch.expm1(x.e)) + 2 * EPS32 * sd + 2.0 ** -125)


# ------------------------------------------------------------------------------------------------------------------
# the tail (tir_tail_body.h + the derived normal of tir_primary.cu) in float64 with error bounds
# ------------------------------------------------------------------------------------------------------------------
def derived_normal(ft, dfdx, softplus, shift, gates, fp32_x=False):
    """-> dict(n [R n,3], dsig [R n,1], s (sigmoid, [R n]), lin (softplus linear branch or ReLU: no second derivative
    gate), norm [R n], den [R n]).  ``fp32_x``: ft is the kernel's fp32 value, so x = ft + shift is computed exactly
    as the kernel does and the branch at 20 is the kernel's"""
    one = rconst(ft, 1.0)
    if softplus:
        x = R((ft.float() + shift).double()) if fp32_x else R.rnd(ft + shift, torch.zeros_like(ft))
        s = sigmoid(x)
        # x > 20 selects 1 instead of s: where that is ambiguous the jump is |1 - s| (2e-9 at 20), not the whole term
        amb = (((x.v - 20.0).abs() <= x.e) & (x.e > 0)).to(x.e.dtype)
        gates.n["softplus 20"] = gates.n.get("softplus 20", 0) + int(amb.sum())
        dsig = rwhere(x.v > 20.0, one, s)
        dsig = R(dsig.v, dsig.e + amb * ((1 - s.v).abs() + s.e))
    else:
        x, s = None, None
        dsig = R((ft > 0).to(ft.dtype))
    dsig = R(dsig.v[:, None], dsig.e[:, None])
    gvec = dsig * dfdx
    n2 = (gvec * gvec).sum(-1, 2.0)
    norm = rsqrt_(n2)
    den = norm.clamp(LO)
    n = -(gvec / R(den.v[:, None], den.e[:, None]))
    return dict(n=n, dsig=dsig, s=s, x=x, norm=norm, den=den, gvec=gvec)


def rel_cost(a, b):
    m = rmax(rmax(a, b), rconst(a, LO))
    q = (a - b) / m
    return q * q


def rel_cost_grad(a, b, gates, name):
    raw = rmax(a, b)
    m = raw.clamp(LO)
    d = a - b
    q = d / m
    dq_dm = -d / (m * m)
    inv = 1.0 / m
    tie = (a.v - b.v).abs() <= (a.e + b.e)
    amb = tie & ((a.e + b.e) > 0)
    gates.n[name + " tie"] = gates.n.get(name + " tie", 0) + int(amb.sum())
    out = []
    for x, y, sgn in ((a, b, 1.0), (b, a, -1.0)):
        sel = torch.where(x.v > y.v, 1.0, torch.where(x.v == y.v, 0.5, 0.0)).to(a.v.dtype)
        t = dq_dm * sel
        t = R(t.v, t.e + amb.to(t.e.dtype) * dq_dm.v.abs() + amb.to(t.e.dtype) * dq_dm.e)
        t = gates.gate(t, raw, LO, math.inf, name + " clip")
        out.append((q * 2.0) * ((inv * sgn) + t))
    return out


def tail_forward(rgb, brdf, brdfj, vn, dn, vd, both):
    """14 channels [R n,14] of one row each; rgb [n,3], brdf / brdfj [n,4], vd [n,3] exact; vn, dn R [n,3] (dn unused
    unless ``both``)."""
    ch = [rc(rgb[:, 0]), rc(rgb[:, 1]), rc(rgb[:, 2]), rcol(vn, 0), rcol(vn, 1), rcol(vn, 2),
          rc(brdf[:, 0]), rc(brdf[:, 1]), rc(brdf[:, 2])]
    rough = rc(brdf[:, 3]) * C09 + C009
    rough_j = rc(brdfj[:, 3]) * C09 + C009
    ch.append(rough)
    ch.append(rel_cost(rc(brdf[:, 0]), rc(brdfj[:, 0])) + rel_cost(rc(brdf[:, 1]), rc(brdfj[:, 1]))
              + rel_cost(rc(brdf[:, 2]), rc(brdfj[:, 2])))
    ch.append(rel_cost(rough, rough_j))
    if both:
        d = vn - dn
        ch.append((d * d).sum(-1, 2.0))
        ch.append((rc(vd) * vn).sum(-1, 2.0).clamp(0.0))
    else:
        z = rconst(rgb[:, 0], 0.0)
        ch += [z, z]
    return rstack(ch)


def tail_backward(w, rgb, brdf, brdfj, vn, dn, vd, both, G, gates):
    """-> dict(w [R n], rgb [R n,3], brdf / brdfj [R n,4], vn [R n,3], dn [R n,3]) of tail_backward_sample"""
    v = tail_forward(rgb, brdf, brdfj, vn, dn, vd, both)
    gw = (v * G).sum(-1, 14.0)
    W = R(w[:, None])
    g = {}
    g["w"] = gw
    g["rgb"] = W * G[:, 0:3]
    gvn = W * G[:, 3:6]
    gb, gbj = [], []
    for c in range(3):
        ga, gbb = rel_cost_grad(rc(brdf[:, c]), rc(brdfj[:, c]), gates, "rel_cost")
        gb.append(R(w) * G[:, 6 + c] + R(w) * G[:, 10] * ga)
        gbj.append(R(w) * G[:, 10] * gbb)
    rough = rc(brdf[:, 3]) * C09 + C009
    rough_j = rc(brdfj[:, 3]) * C09 + C009
    ga, gbb = rel_cost_grad(rough, rough_j, gates, "rel_cost")
    gb.append((R(w) * G[:, 9] + R(w) * G[:, 11] * ga) * C09)
    gbj.append((R(w) * G[:, 11] * gbb) * C09)
    g["brdf"], g["brdfj"] = rstack(gb), rstack(gbj)
    if both:
        dot = (rc(vd) * vn).sum(-1, 2.0)
        d = vn - dn
        t13 = R(w[:, None] * G[:, 13:14] * vd)
        t13 = R(t13.v, t13.e + EPS32 * t13.v.abs())           # w G13 vd: two roundings, the gate is exact
        t13 = gates.gate(t13, dot, 0.0, math.inf, "orientation")
        gvn = gvn + (W * G[:, 12:13]) * 2.0 * d + t13
        g["dn"] = -((W * G[:, 12:13]) * 2.0 * d)
    else:
        g["dn"] = R(torch.zeros_like(vd))
    g["vn"] = gvn
    return g


def derived_backward(dn, dfdx, gn, gates):
    """n = -v / max(|v|, 1e-6), v = dsig dfdx -> (g_dfdx [R n,3], g_feat [R n])"""
    n, norm, den = dn["n"], dn["norm"], dn["den"]
    dot = -((n * gn).sum(-1, 2.0))
    inv = 1.0 / den
    dot_, inv_ = R(dot.v[:, None], dot.e[:, None]), R(inv.v[:, None], inv.e[:, None])
    ga = -((gn - (-n) * dot_) * inv_)
    gb = -(gn * f32(1e6))
    nn = R(norm.v[:, None].expand_as(ga.v), norm.e[:, None].expand_as(ga.v))
    gv = gates.gate(ga, nn, LO, math.inf, "derived 1e-6", strict=True) + gates.gate(gb, nn, -math.inf, LO,
                                                                                    "derived 1e-6")
    g_dfdx = gv * dn["dsig"]
    g_dsig = (gv * dfdx).sum(-1, 3.0)
    if dn["s"] is None:
        return g_dfdx, R(torch.zeros_like(g_dsig.v))
    s = dn["s"]
    gf = g_dsig * s * (1.0 - s)
    x = dn["x"]
    if bool((x.e > 0).any()):
        gf = gates.gate(gf, x, -math.inf, 20.0, "softplus 20")
    else:                                               # the kernel's own fp32 x: the branch is exact
        dec = (x.v <= 20.0).to(gf.v.dtype)
        gf = R(gf.v * dec, gf.e * dec)
    return g_dfdx, gf


# ------------------------------------------------------------------------------------------------------------------
# the epilogue (tir_epilogue_body.h) in float64 with error bounds
# ------------------------------------------------------------------------------------------------------------------
def _f0(f0):
    return f32(f0) if F0_FP32 else f0


def _om(acc, bg):
    """1 - acc: exact for acc = 0 and (Sterbenz) for acc in [0.5, 1]"""
    if not bg:
        return R(torch.zeros_like(acc))
    om = 1.0 - rc(acc)
    exact = (_d(acc) == 0) | (_d(acc) >= 0.5)
    return R(om.v, torch.where(exact, torch.zeros_like(om.e), om.e))


def _d(x):
    return x.detach()


def radd(p, om):
    """p + om: exact where p = 0"""
    x = rc(p) + om
    return R(x.v, torch.where(_d(p) == 0, om.e, x.e))


def srgb(t, gates):
    lo = t * SRGB_S
    hi = (t + LO).pow(SRGB_E) * SRGB_A - SRGB_B
    sel = t.v <= SRGB_T
    amb = ((t.v - SRGB_T).abs() <= t.e).to(t.e.dtype)
    gates.n["srgb"] = gates.n.get("srgb", 0) + int(amb.sum())
    out = rwhere(sel, lo, hi)
    return R(out.v, out.e + amb * ((lo.v - hi.v).abs() + lo.e + hi.e))


def epilogue_forward(P, acc, depth, dz, f0, bg, gates):
    om = _om(acc, bg)
    o = {}
    o["rgb"] = rstack([srgb(radd(P[:, c], om).clamp(0.0, 1.0), gates) for c in range(3)])
    o["albedo"] = rstack([radd(P[:, 6 + c], om).clamp(0.0, 1.0) for c in range(3)])
    o["fresnel"] = rstack([(om + _f0(f0)).clamp(0.0, 1.0) for _ in range(3)])
    o["depth"] = rc(depth) + om * dz
    n = rstack([rc(P[:, 3]), rc(P[:, 4]), rc(P[:, 5]) + om])
    den = rsqrt_((n * n).sum(-1, 2.0)).clamp(LO)
    o["normal"] = n / R(den.v[:, None], den.e[:, None])
    o["rough"] = radd(P[:, 9], om).clamp(0.0, 1.0)
    o["nd"], o["no"] = rc(P[:, 12]), rc(P[:, 13])
    return o


def epilogue_backward(P, acc, dz, f0, bg, g, g_ac, g_rc, gates):
    """g: dict of map gradients ([n,3] / [n], zeros for a NULL map); g_ac / g_rc: the kernel's g_loss / n (R)
    -> (gP [R n,14], g_acc [R n], g_depth [R n])"""
    om = _om(acc, bg)
    n_ = P.shape[0]
    zero = R(torch.zeros(n_, dtype=P.dtype, device=P.device))
    gP = [None] * 14
    g_om = zero
    for c in range(3):
        x = radd(P[:, c], om)
        t = x.clamp(0.0, 1.0)
        lo = rconst(t, SRGB_S)
        hi = (t + LO).pow(DS_E) * DS_A
        amb = ((t.v - SRGB_T).abs() <= t.e).to(t.e.dtype)
        gates.n["srgb"] = gates.n.get("srgb", 0) + int(amb.sum())
        ds = rwhere(t.v <= SRGB_T, lo, hi)
        ds = R(ds.v, ds.e + amb * ((lo.v - hi.v).abs() + hi.e))
        gx = gates.gate(ds * g["rgb"][:, c], x, 0.0, 1.0, "clamp01")
        gP[c] = gx
        g_om = g_om + gx
        xa = radd(P[:, 6 + c], om)
        gP[6 + c] = gates.gate(R(g["albedo"][:, c]), xa, 0.0, 1.0, "clamp01")
        g_om = g_om + gP[6 + c]
        g_om = g_om + gates.gate(R(g["fresnel"][:, c]), om + _f0(f0), 0.0, 1.0, "clamp01")
    g_depth = R(g["depth"])
    g_om = g_om + g_depth * dz
    n = rstack([rc(P[:, 3]), rc(P[:, 4]), rc(P[:, 5]) + om])
    norm = rsqrt_((n * n).sum(-1, 2.0))
    den = norm.clamp(LO)
    y = n / R(den.v[:, None], den.e[:, None])
    gn_ = R(g["normal"])
    dot = (y * gn_).sum(-1, 2.0)
    ga = (gn_ - y * R(dot.v[:, None], dot.e[:, None])) / R(den.v[:, None], den.e[:, None])
    gb = gn_ / LO
    nn = R(norm.v[:, None].expand_as(ga.v), norm.e[:, None].expand_as(ga.v))
    gn = gates.gate(ga, nn, LO, math.inf, "epilogue normal 1e-6") + gates.gate(gb, nn, -math.inf, LO,
                                                                                "epilogue normal 1e-6", strict=False)
    for c in range(3):
        gP[3 + c] = rcol(gn, c)
    g_om = g_om + rcol(gn, 2)
    xr = radd(P[:, 9], om)
    gP[9] = gates.gate(R(g["rough"]), xr, 0.0, 1.0, "clamp01")
    g_om = g_om + gP[9]
    gP[10], gP[11] = rconst(zero, 0.0) + g_ac, rconst(zero, 0.0) + g_rc
    gP[12], gP[13] = R(g["nd"]), R(g["no"])
    g_acc = -g_om if bg else zero
    return rstack(gP), g_acc, g_depth


# ------------------------------------------------------------------------------------------------------------------
# the radiance-only tail (radiance_ray_fwd_kernel / radiance_ray_bwd_kernel) in float64 with error bounds
# ------------------------------------------------------------------------------------------------------------------
def radiance_forward(w, out, ray, acc, depth, dz, bg):
    """rgb_map [R n,3] = sum over the ray's rows of w out (+ 1 - acc) and depth_map [R n] = depth (+ (1 - acc) dz):
    w [m], out [m,3] the rows, ray [m] their ray; acc, depth, dz [n] exact.  The sequential sum carries (count) eps32 of
    sum|w out| besides its terms' own errors."""
    n = acc.shape[0]
    wo = R(w[:, None]) * R(out)
    cnt = torch.bincount(ray, minlength=n).to(acc.dtype)[:, None]
    sv = torch.zeros(n, 3, dtype=acc.dtype, device=acc.device).index_add(0, ray, wo.v)
    se = torch.zeros_like(sv).index_add(0, ray, wo.e) + EPS32 * cnt * torch.zeros_like(sv).index_add(
        0, ray, _d(wo.v).abs())
    rgb, dm = R(sv, se), rc(depth)
    if bg:
        om = 1.0 - rc(acc)
        rgb = rgb + R(om.v[:, None], om.e[:, None])
        dm = dm + om * rc(dz)
    return rgb, dm


def radiance_backward(w, out, ray, dz, g, gd, bg):
    """-> (g_out [R m,3], g_weight [R m], g_acc [R n], g_depth [R n]) of radiance_forward for the map gradients g [n,3]
    and gd [n]"""
    gr = g[ray]
    g_out = R(w[:, None]) * rc(gr)
    g_w = rc(out[:, 0]) * rc(gr[:, 0]) + rc(out[:, 1]) * rc(gr[:, 1]) + rc(out[:, 2]) * rc(gr[:, 2])
    if bg:
        g_acc = -(rc(g[:, 0]) + rc(g[:, 1]) + rc(g[:, 2])) - rc(gd) * rc(dz)
    else:
        g_acc = rc(torch.zeros_like(gd))
    return g_out, g_w, g_acc, rc(gd)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the hand-written backward equals autograd
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_tail_and_epilogue_backward_match_autograd_cpu(kind, monkeypatch):
    """tail_backward / derived_backward / epilogue_backward against float64 autograd of tail_forward /
    derived_normal / epilogue_forward on random rows away from every kink, to 1e-10.  The sRGB derivative takes the
    exact derivative's constants here; the kernel's own (1.055f / 2.4f and 1.f / 2.4f - 1.f, rounded to fp32) differ
    from them by an fp32 rounding, which the GPU comparison carries."""
    monkeypatch.setattr(__import__(__name__), "DS_A", SRGB_A * SRGB_E, raising=True)
    monkeypatch.setattr(__import__(__name__), "DS_E", SRGB_E - 1.0, raising=True)
    g = torch.Generator().manual_seed(3 + kind)
    d = torch.float64
    n = 300
    both = kind == 0
    rgb = torch.rand(n, 3, generator=g, dtype=d)
    brdf = (torch.rand(n, 4, generator=g, dtype=d) * 0.8 + 0.1).requires_grad_(True)
    brdfj = (torch.rand(n, 4, generator=g, dtype=d) * 0.8 + 0.1).requires_grad_(True)
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=d), dim=-1)
    ft = (torch.randn(n, generator=g, dtype=d) * 4 + 10).requires_grad_(True)
    dfdx = (torch.randn(n, 3, generator=g, dtype=d)).requires_grad_(True)
    vp = (torch.rand(n, 3, generator=g, dtype=d) * 2 - 1).requires_grad_(True)
    w = torch.rand(n, generator=g, dtype=d)
    G = torch.randn(n, 14, generator=g, dtype=d)
    gates = Gates()
    dn = derived_normal(ft, dfdx, True, -10.0, gates)
    vn = dn["n"] if kind == 2 else R(vp)
    v = tail_forward(rgb, brdf, brdfj, vn, dn["n"], vd, both)
    loss = (w[:, None] * v.v * G).sum()
    ins = [brdf, brdfj, ft, dfdx] + ([vp] if kind != 2 else [])
    got = torch.autograd.grad(loss, ins, allow_unused=True)
    with torch.no_grad():
        dn0 = derived_normal(ft.detach(), dfdx.detach(), True, -10.0, gates)
        vn0 = dn0["n"] if kind == 2 else R(vp.detach())
        tg = tail_backward(w, rgb, brdf.detach(), brdfj.detach(), vn0, dn0["n"], vd, both, G, gates)
        gn = tg["dn"] + (tg["vn"] if kind == 2 else R(torch.zeros(n, 3, dtype=d)))
        g_dfdx, g_ft = derived_backward(dn0, dfdx.detach(), gn, gates)
    want = [tg["brdf"].v, tg["brdfj"].v, g_ft.v, g_dfdx.v] + ([tg["vn"].v] if kind != 2 else [])
    for a, b, what in zip(got, want, ("brdf", "brdfj", "dn_feat", "dn_dfdx", "vn")):
        if kind == 1 and what in ("dn_feat", "dn_dfdx"):
            continue                                     # purely predicted: no derived normal in the loss
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-12), (kind, what, float((a - b).abs().max()))
    assert torch.allclose(tg["w"].v, (v.v.detach() * G).sum(-1), rtol=1e-10, atol=1e-12)
    # epilogue
    for bg in (0, 1):
        P = (torch.rand(n, 14, generator=g, dtype=d) * 0.8 + 0.1).requires_grad_(True)
        acc = (torch.rand(n, generator=g, dtype=d) * 0.5).requires_grad_(True)
        depth = torch.rand(n, generator=g, dtype=d).requires_grad_(True)
        dz = torch.randn(n, generator=g, dtype=d)
        o = epilogue_forward(P, acc, depth, dz, 0.04, bg, Gates())
        gm = {k: torch.randn(o[k].v.shape, generator=g, dtype=d) for k in o}
        g_ac, g_rc = 0.3 / n, -0.7 / n
        loss = sum((o[k].v * gm[k]).sum() for k in o) + g_ac * P[:, 10].sum() + g_rc * P[:, 11].sum()
        gP_a, gacc_a, gd_a = [torch.zeros_like(x) if y is None else y for x, y in zip(
            (P, acc, depth), torch.autograd.grad(loss, [P, acc, depth], allow_unused=True))]
        with torch.no_grad():
            gP, gacc, gd = epilogue_backward(P.detach(), acc.detach(), dz, 0.04, bg, gm, R(torch.full((n,), g_ac,
                                             dtype=d)), R(torch.full((n,), g_rc, dtype=d)), Gates())
        for a, b, what in ((gP_a, gP.v, "g_packed"), (gacc_a, gacc.v, "g_acc"), (gd_a, gd.v, "g_depth")):
            assert torch.allclose(a, b, rtol=1e-10, atol=1e-12), (bg, what, float((a - b).abs().max()))


@pytest.mark.parametrize("bg", [1, 0])
def test_radiance_backward_matches_autograd_cpu(bg):
    """radiance_backward against float64 autograd of radiance_forward (rows of rays with 0 to 5 rows), to 1e-10."""
    g = torch.Generator().manual_seed(21 + bg)
    d = torch.float64
    n = 40
    ray = torch.repeat_interleave(torch.arange(n), torch.randint(0, 6, (n,), generator=g))
    m_ = ray.numel()
    w = torch.rand(m_, generator=g, dtype=d).requires_grad_(True)
    out = torch.rand(m_, 3, generator=g, dtype=d).requires_grad_(True)
    acc = torch.rand(n, generator=g, dtype=d).requires_grad_(True)
    depth = (torch.rand(n, generator=g, dtype=d) * 4).requires_grad_(True)
    dz = torch.randn(n, generator=g, dtype=d)
    gm, gd = torch.randn(n, 3, generator=g, dtype=d), torch.randn(n, generator=g, dtype=d)
    rgb, dm = radiance_forward(w, out, ray, acc, depth, dz, bg)
    got = torch.autograd.grad((rgb.v * gm).sum() + (dm.v * gd).sum(), [out, w, acc, depth], allow_unused=True)
    got = [torch.zeros_like(x) if y is None else y for x, y in zip((out, w, acc, depth), got)]
    want = radiance_backward(w.detach(), out.detach(), ray, dz, gm, gd, bg)
    for a, b, what in zip(got, want, ("g_out", "g_weight", "g_acc", "g_depth")):
        assert torch.allclose(a, b.v, rtol=1e-10, atol=1e-12), (bg, what, float((a - b.v).abs().max()))


def test_chained_references_reproduce_the_oracle_cpu(monkeypatch):
    """derived_normal, tail_forward and epilogue_forward, chained in float64 on rotated_g24's per-sample head outputs
    (the oracle's own functions, its xyz noise passed in), reproduce O.primary_forward's relight-phase maps and losses,
    and the float64 autograd gradients of a loss of those maps with respect to every oracle parameter.  The constants
    take the oracle's float64 values here (the kernel's are their fp32 roundings)."""
    mod = __import__(__name__)
    for k, v in dict(SRGB_T=0.0031308, SRGB_S=12.92, SRGB_A=1.055, SRGB_B=0.055, SRGB_E=1 / 2.4, C09=0.9, C009=0.09,
                     LO=1e-6, F0_FP32=False).items():
        monkeypatch.setattr(mod, k, v)
    from gpu_helpers import load_fixture
    from helpers import oracle_field
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        fx = load_fixture("rotated_g24.pt")
        f = oracle_field(fx, requires_grad=True).to("cpu", torch.float64)
        params = [p.requires_grad_(True) for p in f.parameters()]
        rays, li = fx["rays"][:24].double(), fx["light_idx"][:24]
        n = rays.shape[0]
        aux = O.primary_forward(f, rays, li, is_train=False, xyz_noise=torch.zeros(1, 3), return_aux=True)[-1]
        app = aux["app_mask"]
        noise = torch.randn(int(app.sum()), 3, generator=torch.Generator().manual_seed(9))
        want = O.primary_forward(f, rays, li, is_train=False, xyz_noise=noise, return_aux=True)
        g = torch.Generator().manual_seed(10)
        gm = [torch.randn(x.shape, generator=g) for x in want[:9]]
        loss_o = sum((x * y).sum() for x, y in zip(want[:9], gm)) + 0.3 * want[10] - 0.7 * want[11]
        go = torch.autograd.grad(loss_o, params, allow_unused=True)
        # the per-sample inputs of the tail, from the oracle's own functions
        xyz, _, _ = O.sample_ray(f, rays[:, :3], rays[:, 3:6], False, -1)
        xyz = O.normalize_coord(f, xyz)[app]
        ray = app.nonzero()[:, 0]
        w = aux["weight"][app]
        rad, intr = O.both_feature(f, xyz, li.view(-1)[ray].view(-1, 1))
        vd = rays[ray, 3:6]
        rgb = O.mlp_render_fea(f, f.mlp_rgb, vd, rad)
        brdf = O.mlp_pe_and_feature(f, f.mlp_brdf, xyz, intr, torch.sigmoid)
        xj = xyz + noise * 0.01
        brdfj = O.mlp_pe_and_feature(f, f.mlp_brdf, xj, O.intrin_feature(f, xj), torch.sigmoid)
        vn = O.mlp_pe_and_feature(f, f.mlp_normal, xyz, intr, torch.tanh)
        xs = xyz.detach().requires_grad_(True) if not xyz.requires_grad else xyz
        ft = O.density_feature_with_xyz_grad(f, xs)
        (dfdx,) = torch.autograd.grad(ft.sum(), xs, create_graph=True)
        gates = Gates()
        dn = derived_normal(ft, dfdx, True, float(f.density_shift), gates)
        assert torch.allclose(dn["n"].v, O.derived_normals(f, xyz.detach().clone()), rtol=1e-10, atol=1e-12)
        v = tail_forward(rgb, brdf, brdfj, R(vn), dn["n"], vd, True)
        P = torch.zeros(n, 14).index_add(0, ray, w[:, None] * v.v)
        acc, depth = aux["weight"].sum(1), (aux["weight"] * aux["z"]).sum(1)
        eo = epilogue_forward(P, acc, depth, rays[:, 5], f.fixed_fresnel, 1, gates)
        got = [eo["rgb"].v, eo["depth"].v, eo["normal"].v, eo["albedo"].v, eo["rough"].v[:, None],
               eo["fresnel"].v, acc, eo["nd"].v[:, None], eo["no"].v[:, None]]
        for k, (x, y) in enumerate(zip(got, want[:9])):
            assert torch.allclose(x, y.reshape(x.shape), rtol=1e-10, atol=1e-12), (k, float((x - y.reshape(x.shape))
                                                                                             .abs().max()))
        assert torch.allclose(P[:, 10].mean(), want[10]) and torch.allclose(P[:, 11].mean(), want[11])
        loss = sum((x * y.reshape(x.shape)).sum() for x, y in zip(got, gm)) + 0.3 * P[:, 10].mean() - \
            0.7 * P[:, 11].mean()
        gg = torch.autograd.grad(loss, params, allow_unused=True)
        for k, (a, b) in enumerate(zip(gg, go)):
            if a is None or b is None:
                assert (a is None or float(a.abs().max()) == 0) and (b is None or float(b.abs().max()) == 0), k
                continue
            assert torch.allclose(a, b, rtol=1e-9, atol=1e-12), (k, float((a - b).abs().max()))
    finally:
        torch.set_default_dtype(old)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def chk(got, want, bnd, what, key):
    """test_heads_kernels_fp64.check, with a finite bound, at least one entry, and the largest err/bound recorded"""
    bnd = torch.as_tensor(bnd, dtype=torch.float64, device=want.device).expand(want.shape)
    assert want.numel() > 0, what
    bad = ~torch.isfinite(bnd)
    assert not bool(bad.any()), (what, bad.nonzero()[:5].tolist(), want[bad][:5].tolist(), bnd[bad][:5].tolist())
    err = (got.detach().double().reshape(want.shape) - want.detach().double()).abs()
    r = float((err / bnd.clamp_min(1e-30)).max())
    STATS[key] = max(STATS.get(key, 0.0), r)
    check(got, want, bnd, what)


def chk_r(got, ref, what, key):
    chk(got, ref.v, ref.e + 1e-30, what, key)


def grad_bufs(m, dev):
    """channel-last VM gradient buffers prefilled with PRE, in the order dplane, dline, aplane, aline"""
    out = []
    for name in ("density_plane", "density_line", "app_plane", "app_line"):
        out.append([torch.full((p.shape[2], p.shape[3], p.shape[1]), PRE, device=dev) for p in getattr(m, name)])
    return out


class Case:
    def __init__(self, m, rays, li, n_samples, seed, table=None):
        self.m, self.rays, self.li, self.n_samples = m, rays.to(DEV).float().contiguous(), li.to(DEV), n_samples
        self.table = table                                # z table of TIR_SAMPLE_TABLE (then no jitter)
        g = torch.Generator().manual_seed(seed)
        self.g = g
        self.jitter = torch.rand(self.rays.shape[0], 1, generator=g).to(DEV)
        self.grid = [int(x) for x in m.gridSize]


def _oracle_density(m):
    """the model's density factors as an OracleField in float64 (for the gathers)"""
    ps = [p.detach().double() for p in m.density_plane]
    ls = [p.detach().double() for p in m.density_line]
    return ps, ls


class Dump:
    """What check_stages reads: the workspace ``ws`` a forward/backward left its dumps in, the inputs of that launch
    (model, rays, light ids, jitter or z table, noise, background flag) and the upstream gradients of its backward
    (``gm``: map gradients by name, None for a map that got none; ``g_acc_map``, ``g_la``, ``g_lr``: None or tensors),
    and the parameter gradients it produced: ``vmg`` (channel-last density planes, density lines, app planes, app
    lines), ``g_basis``, ``g_ll``, ``mod`` (head module -> its six tensors), each prefilled with ``pre``."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def run_case(cs, ws=None, n_rays=None, cap_valid=None, cap_app=None, bg=1, stats_key=""):
    """Drive the four entry points once on ``cs`` and check every stage.  -> dict with the totals.  With ``ws``
    given, its integer arrays keep what the launch before left in them."""
    return check_stages(launch(cs, ws, n_rays, cap_valid, cap_app, bg), stats_key)


def launch(cs, ws=None, n_rays=None, cap_valid=None, cap_app=None, bg=1):
    """tir_primary_march / _app_list / _heads / _backward once on ``cs``, seeded with random map gradients (fresnel
    and roughness None), a non-NULL g_acc_map and both loss gradients, every parameter gradient prefilled with PRE
    -> Dump"""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.primary_fused import Workspace, _jobs
    lib = _lib.load()
    m = cs.m
    n_rays = n_rays or cs.rays.shape[0]
    rays, li = cs.rays[:n_rays].contiguous(), cs.li.reshape(-1)[:n_rays].to(torch.int32).contiguous()
    jitter = cs.jitter[:n_rays].contiguous()
    g = cs.g
    f = ops.device_field(m).refresh(m, force=True)
    keep = []
    jobs, n_jobs, heads, kind = _jobs(m, keep)
    if cs.table is not None:
        jitter = None
    cfg = ops.march_cfg(m, table=cs.table, n_samples=cs.n_samples, jitter=jitter, keep=keep)
    total = int(march_reference(m, rays, cs.n_samples, jitter, cs.table)["offsets"][-1])
    cv = cap_valid if cap_valid is not None else total
    ca = cap_app if cap_app is not None else total
    fresh = ws is None
    if fresh:
        ws = Workspace(DEV)
        ws.ensure(n_rays, cv + 257, ca + 257, n_jobs, True)
        fill_sentinel(ws)
    else:
        for x in ws.t.values():
            if x.is_floating_point():
                x.fill_(SENT)
    assert ws.cap_valid >= cv + 1 and ws.cap_app >= ca + 1           # guard rows behind both capacities
    noise = torch.full((ws.cap_app, 3), SENT, device=DEV)
    noise[:ca] = torch.randn(ca, 3, generator=g).to(DEV)
    w = ws.work_struct(noise, n_jobs, True)
    w.cap_valid, w.cap_app = cv, ca
    stream = _lib.stream_ptr()
    _lib.check(lib.tir_primary_march(C.byref(f), _lib.dptr(rays), n_rays, C.byref(cfg), C.byref(w), None, stream),
               "tir_primary_march")
    _lib.check(lib.tir_primary_app_list(C.byref(f), n_rays, C.byref(w), stream), "tir_primary_app_list")
    maps_t = [torch.full((n_rays, c), SENT, device=DEV) for c in (3, 1, 3, 3, 1, 3, 1, 1)]
    maps = _lib.TirRayMaps()
    for k, x in zip(MAP_NAMES, maps_t):
        setattr(maps, k, x.data_ptr())
    mask = torch.empty(n_rays, dtype=torch.bool, device=DEV)
    losses = torch.full((2,), SENT, device=DEV)
    f0 = float(m.fixed_fresnel)
    _lib.check(lib.tir_primary_heads(C.byref(f), jobs, n_jobs, kind, _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                     n_rays, C.byref(w), f0, bg, C.byref(maps), _lib.dptr(mask, torch.bool),
                                     _lib.dptr(losses), None, stream), "tir_primary_heads")
    # --- backward
    gm = {}
    for k, x in zip(MAP_NAMES, maps_t):
        gm[k] = None if k in ("fresnel", "rough") else torch.randn(x.shape, generator=g).to(DEV)
    gmaps = _lib.TirRayMaps()
    for k in MAP_NAMES:
        setattr(gmaps, k, None if gm[k] is None else gm[k].data_ptr())
    g_acc_map = torch.randn(n_rays, generator=g).to(DEV)
    g_la, g_lr = torch.randn(1, generator=g).to(DEV), torch.randn(1, generator=g).to(DEV)
    b = ws.bwd_struct(n_jobs)
    gr = _lib.TirPrimaryGrads()
    vmg = grad_bufs(m, DEV)
    for k in range(3):
        gr.dplane[k], gr.dline[k] = vmg[0][k].data_ptr(), vmg[1][k].data_ptr()
        gr.aplane[k], gr.aline[k] = vmg[2][k].data_ptr(), vmg[3][k].data_ptr()
    g_basis = torch.full_like(m.basis_mat.weight, PRE)
    gr.basis = g_basis.data_ptr()
    ll = getattr(m, "light_line", None)
    g_ll = torch.full_like(ll.weight, PRE) if ll is not None else None
    gr.light_line = None if ll is None else g_ll.data_ptr()
    mod = {}
    for j, head in enumerate(heads):
        if head not in mod:
            mlp = getattr(m, head).mlp
            mod[head] = [torch.full_like(x, PRE) for x in (mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias,
                                                           mlp[4].weight, mlp[4].bias)]
        gr.w0[j], gr.b0[j], gr.w1[j], gr.b1[j], gr.w2[j], gr.b2[j] = [x.data_ptr() for x in mod[head]]
    _lib.check(lib.tir_primary_backward(C.byref(f), jobs, n_jobs, kind, _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                        n_rays, C.byref(w), C.byref(b), f0, bg, C.byref(gmaps), _lib.dptr(g_acc_map),
                                        _lib.dptr(g_la), _lib.dptr(g_lr), C.byref(gr), stream), "tir_primary_backward")
    torch.cuda.synchronize()
    return Dump(m=m, ws=ws, rays=rays, li=li, jitter=jitter, table=cs.table, n_samples=cs.n_samples, cv=cv, ca=ca,
                noise=noise, bg=bg, maps=maps_t, mask=mask, losses=losses, gm=gm, g_acc_map=g_acc_map, g_la=g_la,
                g_lr=g_lr, vmg=vmg, g_basis=g_basis, g_ll=g_ll, mod=mod, pre=PRE, guards=True, fresh=fresh)


def _scalar(g):
    return 0.0 if g is None else float(g.reshape(-1)[0])


def march_reference(m, rays, n_samples, jitter, table):
    """the modular valid-sample list (pinned to the oracle elsewhere) of the same march"""
    from tensoir_b200 import vm_autograd as vm
    return vm.valid_samples(m, rays[:, :3], rays[:, 3:6], n_samples=n_samples, jitter=jitter, table=table)


def front(d, what0):
    """march, density, compositing and the appearance list of the launch in ``d`` against their references (the
    module docstring's first three items) -> dict of what the later stages need"""
    import test_vm_kernels_fp64 as V
    m, ws, rays, t = d.m, d.ws, d.rays, d.ws.t
    n_rays = rays.shape[0]
    grid = [int(x) for x in m.gridSize]
    cv, ca = d.cv, d.ca
    ref = march_reference(m, rays, d.n_samples, d.jitter, d.table)
    total = int(ref["offsets"][-1])
    # ================= 1. march
    status = t["status"].tolist()
    nv = min(total, cv)
    assert status[0] == total, what0
    assert torch.equal(t["counts"][:n_rays], ref["counts"]), what0
    want_off = torch.cat([torch.zeros(1, dtype=torch.int64, device=DEV), t["counts"][:n_rays].long().cumsum(0)])
    assert torch.equal(t["offsets"][:n_rays + 1], want_off), what0
    for k, kr in (("v_ray", "ray"), ("v_sample", "sample"), ("v_xn", "xn"), ("v_z", "z"), ("v_dist", "dist")):
        assert torch.equal(t[k][:nv], ref[kr][:nv]), (what0, k)
        if d.guards and (d.fresh or t[k].is_floating_point()):
            assert bool((t[k][nv:] == (SENT if t[k].is_floating_point() else 0)).all()), (what0, k, "guard")
    # ================= 2. density and compositing
    softplus = m.fea2denseAct == "softplus"
    shift = float(m.density_shift)
    dps, dls = _oracle_density(m)
    xv = t["v_xn"][:nv].double()
    with V.f64():
        fo = O.OracleField(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), grid_size=grid, density_plane=dps,
                           density_line=dls, app_plane=dps, app_line=dls, basis_w=None, mlp_rgb=None)
        feat64 = O.density_feature(fo, xv)
    ts = V.tap_sums(dps, dls, xv, False, False, grid)
    tu = V.tap_sums(dps, dls, xv, False, True, grid)
    efeat = V.bound(sum((q["AP"] * q["AL"]).sum(1) for q in ts), sum((q["AP"] * q["AL"]).sum(1) for q in tu),
                    grid=grid)
    chk(t["v_feat"][:nv], feat64, efeat, f"{what0}: v_feat", "v_feat")
    featk = t["v_feat"][:nv].double()
    if softplus:
        x = featk + shift
        sig64 = torch.nn.functional.softplus(x)
        esig = torch.sigmoid(x) * EPS32 * x.abs() + 4 * EPS32 * sig64 + 3e-9
    else:
        sig64 = featk.clamp_min(0)
        esig = torch.zeros_like(sig64) + 1e-30
    chk(t["v_sigma"][:nv], sig64, esig, f"{what0}: v_sigma", "v_sigma")
    # compositing from the kernel's own sigma
    ray_v = t["v_ray"][:nv].long()
    pos = torch.arange(nv, device=DEV) - t["offsets"][ray_v]
    S = int(pos.max()) + 1 if nv else 1
    valid = torch.zeros(n_rays, S, dtype=torch.bool, device=DEV)
    valid[ray_v, pos] = True

    def pad(x, dtype=torch.float64):
        out = torch.zeros(n_rays, S, dtype=dtype, device=DEV)
        out[ray_v, pos] = x[:nv].to(dtype)
        return out
    scale = float(m.distance_scale)
    d32 = t["v_dist"][:nv] * scale                                   # the kernel's fp32 product
    r = {}
    for dt in (torch.float64, torch.float32):
        sig = pad(t["v_sigma"], dt).requires_grad_(True)
        dd = pad(d32, dt)
        alpha, wgt, T_last = O.raw2alpha(sig, dd) if dt == torch.float64 else _raw2alpha32(sig, dd)
        T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1. - alpha + 1e-10], -1), -1)[:, :-1]
        r[dt] = dict(sig=sig, alpha=alpha, w=wgt, T=T.detach(), T_last=T_last.reshape(-1), valid=valid, d=dd)
    r64, r32 = r[torch.float64], r[torch.float32]
    fp64_ok, fp32_reg, has_opaque = V.regimes(r64)
    z = pad(t["v_z"])
    bw, bT, bTl = composite_bounds(r64, fp64_ok, fp32_reg, has_opaque)
    for k, kk, b_ in (("v_weight", "w", bw), ("v_trans", "T", bT)):
        got = pad(t[k])
        for reg, name in ((fp64_ok, "fp64 regime"), (fp32_reg, "fp32 regime")):
            if bool(reg.any()):
                chk(got[reg], r64[kk].detach()[reg], b_[reg], f"{what0}: {k} {name}", f"{k} ({name})")
        if bool(fp32_reg.any()):
            w32 = r32[kk].detach().double()
            sc = w32.abs().amax(1, keepdim=True).expand_as(w32)
            chk(got[fp32_reg], w32[fp32_reg], 1e-4 * sc[fp32_reg] + 1e-30, f"{what0}: {k} vs the fp32 scan",
                f"{k} (vs the fp32 scan)")
    Sr = valid.sum(1).double()
    acc64, depth64 = r64["w"].detach().sum(1), (r64["w"].detach() * z).sum(1)
    for k, want, extra in (("acc", acc64, bw.sum(1)), ("depth", depth64, (bw * z).sum(1)),
                           ("t_last", r64["T_last"].detach(), bTl)):
        bnd = extra + EPS32 * (Sr + 1) * want.abs() + 2.0 ** -126
        chk(t[k][:n_rays], want, bnd, f"{what0}: {k}", k)
    for k, want in (("acc", r32["w"].detach().sum(1)), ("depth", (r32["w"].detach() * z.float()).sum(1)),
                    ("t_last", r32["T_last"].detach())):
        o_ = has_opaque
        if bool(o_.any()):
            chk(t[k][:n_rays][o_], want.double()[o_], 1e-4 * (1 + want.double().abs()[o_]),
                f"{what0}: {k} vs the fp32 scan", f"{k} (vs the fp32 scan)")
    thres = float(torch.tensor(float(m.rayMarch_weight_thres), dtype=torch.float32))
    sel = torch.zeros(max(ws.cap_valid, 1), dtype=torch.bool, device=DEV)
    sel[:nv] = t["v_weight"][:nv] > thres
    want_ac = torch.zeros(n_rays, dtype=torch.int64, device=DEV).index_add_(0, ray_v, sel[:nv].long())
    assert torch.equal(t["a_counts"][:n_rays].long(), want_ac), what0
    want_aoff = torch.cat([torch.zeros(1, dtype=torch.int64, device=DEV), want_ac.cumsum(0)])
    assert torch.equal(t["a_offsets"][:n_rays + 1], want_aoff), what0
    total_app = int(want_aoff[-1])
    assert status[1] == total_app, what0
    assert status[2] == int(total > cv or total_app > ca), (what0, status, cv, ca)
    # ================= 3. appearance list
    na = min(total_app, ca)
    src = torch.nonzero(sel[:nv]).reshape(-1)[:na]
    assert torch.equal(t["a_src"][:na], src), what0
    assert torch.equal(t["a_ray"][:na], t["v_ray"][src]), what0
    assert torch.equal(t["a_w"][:na], t["v_weight"][src]), what0
    assert torch.equal(t["a_xn"][:na], t["v_xn"][src]), what0
    return dict(gates=Gates(), total=total, total_app=total_app, nv=nv, na=na, src=src, sel=sel, cv=cv, ca=ca, grid=grid,
                softplus=softplus, shift=shift, dps=dps, dls=dls, xv=xv, fo=fo, ts=ts, tu=tu, ray_v=ray_v, pos=pos, S=S,
                valid=valid, pad=pad, r64=r64, fp64_ok=fp64_ok, z=z, bw=bw, bT=bT)


def check_stages(d, stats_key=""):
    """Every stage of a relight-phase forward/backward against float64, from the dumps and inputs in ``d`` (Dump).
    With ``d.guards`` the rows past the lists' capacities must hold the sentinel (a launch of ``launch``).
    -> dict with the totals"""
    from tensoir_b200.primary_fused import _jobs
    import test_vm_kernels_fp64 as V
    m, ws, rays, li, bg, noise, PRE = d.m, d.ws, d.rays, d.li, d.bg, d.noise, d.pre
    fresh = d.fresh
    t = ws.t
    n_rays = rays.shape[0]
    jobs, n_jobs, heads, kind = _jobs(m, [])
    ll = getattr(m, "light_line", None)
    f0 = float(m.fixed_fresnel)
    maps_t, mask, losses, gm = d.maps, d.mask, d.losses, d.gm
    names = MAP_NAMES
    vmg, g_basis, g_ll, mod = d.vmg, d.g_basis, d.g_ll, d.mod
    what0 = f"{stats_key} n_rays {n_rays}"
    c = front(d, what0)
    gates = c["gates"]
    total, total_app, nv, na, src, sel = c["total"], c["total_app"], c["nv"], c["na"], c["src"], c["sel"]
    softplus, shift, grid, fo, dps, dls = c["softplus"], c["shift"], c["grid"], c["fo"], c["dps"], c["dls"]
    # ================= 3. appearance list (guard rows)
    if d.guards:
        for k in ("a_w", "a_xn", "a_xj", "dn_feat", "dn_dfdx", "g_dn_feat", "g_dn_dfdx") + tuple(
                f"{p}{j}" for j in range(n_jobs) for p in ("out", "g_out", "inp", "h2_", "gx0_")):
            assert bool((t[k][na:] == SENT).all()), (what0, k, "guard")
        if fresh:
            assert bool((t["a_src"][na:] == 0).all()), (what0, "a_src guard")
    if na == 0:
        return dict(total=total, total_app=total_app, ws=ws, gates=gates)
    # ================= 4. heads forward
    T = {k: v[:na].double() for k, v in t.items() if v.shape[0] == ws.cap_app and v.is_floating_point()}
    ray = t["a_ray"][:na].long()
    nz = noise[:na].double()
    chk(T["a_xj"], T["a_xn"] + nz * 0.01, 2 * EPS32 * (T["a_xn"].abs() + 0.01 * nz.abs()), f"{what0}: a_xj", "a_xj")
    pts = [T["a_xn"], T["a_xj"]]
    aps, als = [p.detach() for p in m.app_plane], [p.detach() for p in m.app_line]
    for ps in (0, 1):
        check_gather(aps, als, grid, pts[ps], T[f"x0_{ps}"], f"{what0}: x0 of point set {ps}")
    basis = m.basis_mat.weight.detach().double()
    ll64 = ll.weight.detach().double() if ll is not None else None
    L = ll64.shape[0] if ll is not None else 1
    li_row = li.long()[ray]
    stages = []
    for j in range(n_jobs):
        mlp = getattr(m, heads[j]).mlp
        W = [mlp[i].weight.detach().double() for i in (0, 2, 4)]
        B = [mlp[i].bias.detach().double() for i in (0, 2, 4)]
        lm = jobs[j].light_mode if ll is not None else 0
        ps = jobs[j].point_set
        vec = rays[ray, 3:6].double() if jobs[j].x_in == 0 else pts[ps]
        st = Stages(na, lm, jobs[j].act, L, W, B, basis, ll64, li_row, vec, T[f"x0_{ps}"], T[f"inp{j}"],
                    T[f"h1_{j}"], T[f"h2_{j}"], T[f"out{j}"][:, :W[2].shape[0]])
        st.forward(f"{what0}: job {j}")
        stages.append(st)
    has_dn = kind != 1
    if has_dn:
        xa = T["a_xn"]
        with V.f64():
            xs = xa.clone().requires_grad_(True)
            ftc = O.density_feature_with_xyz_grad(fo, xs)
            (dfd,) = torch.autograd.grad(ftc.sum(), xs)
        tsc = V.tap_sums(dps, dls, xa, True, False, grid)
        tuc = V.tap_sums(dps, dls, xa, True, True, grid)
        mf, md = V._grad_mags(tsc, xa)
        uf, ud = V._grad_mags(tuc, xa)
        chk(T["dn_feat"], ftc.detach(), V.bound(mf, uf, grid=grid), f"{what0}: dn_feat", "dn_feat")
        gi = torch.stack([(xa[:, a] + 1) / 2 * (grid[a] - 1) for a in range(3)], 1)
        near = ((gi - gi.round()).abs() <= 4 * EPS32 * (max(grid) - 1)).any(1)
        STATS["texel-centre rows"] = STATS.get("texel-centre rows", 0) + int(near.sum())
        assert int(near.sum()) <= 0.01 * na + 2, (what0, int(near.sum()))
        chk(T["dn_dfdx"][~near], dfd[~near], V.bound(md, ud, grid=grid)[~near], f"{what0}: dn_dfdx", "dn_dfdx")
    # ================= 5. tail forward
    j_of = {jobs[j].role: j for j in range(n_jobs)}
    o_rgb, o_b, o_bj = T[f"out{j_of[0]}"], T[f"out{j_of[1]}"], T[f"out{j_of[2]}"]
    vd = rays[ray, 3:6].double()
    dn = derived_normal(T["dn_feat"], T["dn_dfdx"], softplus, shift, gates, fp32_x=True) if has_dn else None
    vn = dn["n"] if kind == 2 else R(T[f"out{j_of[3]}"][:, :3])
    dnn = dn["n"] if has_dn else R(torch.zeros_like(vd))
    both = kind == 0
    v = tail_forward(o_rgb[:, :3], o_b, o_bj, vn, dnn, vd, both)
    wv = R(T["a_w"][:, None]) * v
    P = torch.zeros(n_rays, 14, dtype=torch.float64, device=DEV).index_add_(0, ray, wv.v)
    Pe = torch.zeros_like(P).index_add_(0, ray, wv.e)
    Pm = torch.zeros_like(P).index_add_(0, ray, wv.v.abs())
    cnt = torch.bincount(ray, minlength=n_rays).double()[:, None]
    chk(t["packed"][:n_rays], P, Pe + Pm * EPS32 * (16 + 4 * cnt.sqrt()) + 1e-30, f"{what0}: packed", "packed")
    # ================= 6. epilogue forward (from the kernel's own packed / acc / depth)
    Pk = t["packed"][:n_rays].double()
    acck, depthk = t["acc"][:n_rays].double(), t["depth"][:n_rays].double()
    dz = rays[:, 5].double()
    eo = epilogue_forward(Pk, acck, depthk, dz, f0, bg, gates)
    for k, x in zip(names, maps_t):
        if k == "fresnel":
            continue
        chk_r(x.reshape(eo[k].v.shape), eo[k], f"{what0}: map {k}", f"map {k}")
    chk_r(maps_t[5], eo["fresnel"], f"{what0}: map fresnel", "map fresnel")
    assert torch.equal(mask, t["acc"][:n_rays] > 0.5), what0
    for i, col in enumerate((10, 11)):
        want = Pk[:, col].sum() / n_rays
        bnd = sum_bound(Pk[:, col].abs().sum(), n_rays) / n_rays + 2 * EPS32 * Pk[:, col].abs().sum() / n_rays
        chk(losses[i:i + 1], want.reshape(1), bnd.reshape(1) + 1e-30, f"{what0}: loss {i}", "losses")
    # ================= 7. backward: epilogue
    gz = {k: (gm[k].double() if gm[k] is not None else torch.zeros(x.shape, dtype=torch.float64, device=DEV))
          for k, x in zip(names, maps_t)}
    gz = {k: (v_.reshape(-1) if v_.shape[1] == 1 else v_) for k, v_ in gz.items()}
    g_ac = R(torch.full((n_rays,), _scalar(d.g_la), dtype=torch.float64, device=DEV)) / float(n_rays)
    g_rc = R(torch.full((n_rays,), _scalar(d.g_lr), dtype=torch.float64, device=DEV)) / float(n_rays)
    gP, gacc, gdep = epilogue_backward(Pk, acck, dz, f0, bg, gz, g_ac, g_rc, gates)
    chk_r(t["g_packed"][:n_rays], gP, f"{what0}: g_packed", "g_packed")
    chk_r(t["g_acc"][:n_rays], gacc, f"{what0}: g_acc", "g_acc")
    chk_r(t["g_depth"][:n_rays], gdep, f"{what0}: g_depth", "g_depth")
    # ================= tail backward (from the kernel's own g_packed)
    Gk = t["g_packed"][:n_rays].double()[ray]
    tg = tail_backward(T["a_w"], o_rgb[:, :3], o_b, o_bj, vn, dnn, vd, both, Gk, gates)
    chk_r(T[f"g_out{j_of[0]}"][:, :3], tg["rgb"], f"{what0}: g_out rgb", "g_out")
    assert bool((t[f"g_out{j_of[0]}"][:na, 3] == 0).all()), what0
    chk_r(T[f"g_out{j_of[1]}"], tg["brdf"], f"{what0}: g_out brdf", "g_out")
    chk_r(T[f"g_out{j_of[2]}"], tg["brdfj"], f"{what0}: g_out brdf jitter", "g_out")
    if kind != 2:
        chk_r(T[f"g_out{j_of[3]}"][:, :3], tg["vn"], f"{what0}: g_out normal", "g_out")
    gw_full = t["g_weight"][:nv].double()
    chk_r(gw_full[src], tg["w"], f"{what0}: g_weight", "g_weight")
    other = torch.ones(nv, dtype=torch.bool, device=DEV)
    other[src] = False
    assert bool((t["g_weight"][:nv][other] == 0).all()), what0
    if has_dn:
        gn = tg["dn"] + (tg["vn"] if kind == 2 else R(torch.zeros_like(vd)))
        g_dfdx, g_ft = derived_backward(dn, T["dn_dfdx"], gn, gates)
        chk_r(T["g_dn_dfdx"], g_dfdx, f"{what0}: g_dn_dfdx", "g_dn_dfdx")
        chk_r(T["g_dn_feat"], g_ft, f"{what0}: g_dn_feat", "g_dn_feat")
    # ================= heads backward
    a_ps = [torch.zeros(na, 144, dtype=torch.float64, device=DEV) for _ in range(2)]
    wsum, bsum = {}, {}
    for j, st in enumerate(stages):
        a = st.data_grads(f"{what0}: job {j}", T[f"g_out{j}"], T[f"gz2_{j}"], T[f"gz1_{j}"], T[f"gfeat{j}"][:, :NF],
                          T[f"gx0_{j}"])
        a_ps[jobs[j].point_set] += T[f"gx0_{j}"]
        want, bnds = st.param_grads(T[f"g_out{j}"], T[f"gz2_{j}"], T[f"gz1_{j}"], T[f"gfeat{j}"][:, :NF], a,
                                    n_add_w=14 * n_jobs)
        for k in ("w0", "b0", "w1", "b1", "w2", "b2"):
            key = (heads[j], k)
            wsum[key] = wsum.get(key, 0) + want[k]
            bsum[key] = bsum.get(key, 0) + bnds[k]
        for k in ("basis", "light"):
            if k in want:
                wsum[k] = wsum.get(k, 0) + want[k]
                bsum[k] = bsum.get(k, 0) + bnds[k]
    names6 = ("w0", "b0", "w1", "b1", "w2", "b2")
    for head, bufs in mod.items():
        for k, buf in zip(names6, bufs):
            want = wsum[(head, k)]
            bnd = bsum[(head, k)] + sum_bound(PRE, 14 * n_jobs)
            chk(buf - PRE, want, bnd, f"{what0}: d {head}.{k}", "head weights")
    chk(g_basis - PRE, wsum["basis"], bsum["basis"] + sum_bound(PRE, 14 * n_jobs), f"{what0}: d basis_mat",
        "basis_mat")
    if ll is not None:
        chk(g_ll - PRE, wsum["light"], bsum["light"] + sum_bound(PRE, na * n_jobs), f"{what0}: d light_line",
            "light_line")
    # the appearance factors: both point sets through one float64 scatter of the summed d x0
    check_factor_grads(aps, als, grid, torch.cat(pts), torch.cat(a_ps), vmg[2], vmg[3],
                       f"{what0}: appearance factors", prefill=PRE)
    back(d, c, what0, (T["a_xn"], T["g_dn_feat"], T["g_dn_dfdx"], tsc, tuc) if has_dn else None)
    return dict(total=total, total_app=total_app, ws=ws, gates=gates, lengths=t["counts"][:n_rays].clone(),
                flat_rows=int((dn["norm"].v <= LO).sum()) if has_dn else 0, weights=t["v_weight"][:nv].clone(),
                t_zero=int((t["v_trans"][:nv] == 0).sum()), t_last_zero=int((t["t_last"][:n_rays] == 0).sum()))


def back(d, c, what0, dgrad):
    """compositing backward and density scatter of the launch in ``d`` (``c``: front's dict), from the kernel's own
    g_weight, g_acc (+ the caller's g_acc_map) and g_depth; ``dgrad``: None, or (a_xn, g_dn_feat, g_dn_dfdx, tap sums
    of the gradient gather, their unit sums) of the derived normals' double backward"""
    import test_vm_kernels_fp64 as V
    t, PRE, vmg = d.ws.t, d.pre, d.vmg
    n_rays = d.rays.shape[0]
    nv, cv, grid, pad, r64, z = c["nv"], c["cv"], c["grid"], c["pad"], c["r64"], c["z"]
    bw, bT, fp64_ok, valid, softplus, shift = c["bw"], c["bT"], c["fp64_ok"], c["valid"], c["softplus"], c["shift"]
    dps, dls, xv, ts, tu = c["dps"], c["dls"], c["xv"], c["ts"], c["tu"]
    if dgrad is not None:
        xa, g_dn_feat, g_dn_dfdx, tsc, tuc = dgrad
    g_ext = d.g_acc_map.double() if d.g_acc_map is not None else torch.zeros(n_rays, dtype=torch.float64, device=DEV)
    # ================= compositing backward (from the kernel's own g_weight, g_acc + g_acc_map, g_depth)
    ga_tot = t["g_acc"][:n_rays].double() + g_ext
    gdk = t["g_depth"][:n_rays].double()
    gw_pad = pad(t["g_weight"])
    loss = (r64["w"] * gw_pad).sum() + (r64["w"].sum(1) * ga_tot).sum() + ((r64["w"] * z).sum(1) * gdk).sum()
    (gsig64,) = torch.autograd.grad(loss, r64["sig"])
    featp = pad(t["v_feat"])
    if softplus:
        xk = pad((t["v_feat"][:nv] + shift).float(), torch.float64)          # the kernel's fp32 feat + shift
        ds = torch.where(xk > 20, torch.ones_like(xk), torch.sigmoid(xk))
    else:
        ds = (featp > 0).double()
    gfeat64 = gsig64 * ds
    bnd, bwd_ok = composite_bwd_bound(r64, bw, bT, gw_pad, ga_tot, gdk, z, g_ext, t["g_acc"][:n_rays].double(),
                              gsig64, ds, gfeat64)
    gf = pad(t["g_feat"])
    assert bool(torch.isfinite(t["g_feat"][:nv]).all()), what0
    bwd_ok = bwd_ok & fp64_ok
    bwd_32 = valid & ~bwd_ok
    if bool(bwd_ok.any()):
        chk(gf[bwd_ok], gfeat64[bwd_ok], bnd[bwd_ok], f"{what0}: g_feat fp64 regime", "g_feat")
    # the rest (om not resolved by fp32, from 1 - alpha < 2^-22 on): g_alpha = gw T - suffix / om divides by an om
    # that fp32 knows to no relative precision, so neither float64 nor the fp32 autograd of the reference's
    # expression (which differentiates cumprod, not the kernel's suffix sum) bounds it; only finiteness is checked
    STATS["g_feat rows with om unresolved"] = STATS.get("g_feat rows with om unresolved", 0) + int(bwd_32.sum())
    if d.guards:
        assert bool((t["g_feat"][cv:] == SENT).all()) and bool((t["g_weight"][cv:] == SENT).all()), (what0, "guard")
    # ================= density factors: g_feat at v_xn (zero padding) + the double backward at a_xn (clamped)
    gfk = t["g_feat"][:nv].double()
    with V.f64():
        dps_ = [p.clone().requires_grad_(True) for p in dps]
        dls_ = [p.clone().requires_grad_(True) for p in dls]
        fg = O.OracleField(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), grid_size=grid, density_plane=dps_,
                           density_line=dls_, app_plane=dps_, app_line=dls_, basis_w=None, mlp_rgb=None)
        loss = (O.density_feature(fg, xv) * gfk).sum()
        if dgrad is not None:
            xs = xa.clone().requires_grad_(True)
            ftc = O.density_feature_with_xyz_grad(fg, xs)
            (dfd,) = torch.autograd.grad(ftc.sum(), xs, create_graph=True)
            loss = loss + (ftc * g_dn_feat).sum() + (dfd * g_dn_dfdx).sum()
        loss.backward()
    agf = gfk.abs()[:, None]
    mv = V.scatter(ts, lambda k, q, j: agf * q["ptaps"][j][1][:, None] * q["AL"],
                   lambda k, q, j: agf * q["ltaps"][j][1][:, None] * q["AP"], 16)
    uv = V.scatter(tu, lambda k, q, j: agf * q["ptaps"][j][1][:, None] * q["AL"],
                   lambda k, q, j: agf * q["ltaps"][j][1][:, None] * q["AP"], 16)
    if dgrad is not None:
        mc, uc = _dgrad_scatter(tsc, tuc, g_dn_feat.abs(), g_dn_dfdx.abs())
        mv = [tuple(a + b_ for a, b_ in zip(x, y)) for x, y in zip(mv, mc)]
        uv = [tuple(a + b_ for a, b_ in zip(x, y)) for x, y in zip(uv, uc)]
    mv = [(mp + PRE, ml + PRE, cp, cl) for mp, ml, cp, cl in mv]
    V.check_scatter([x - PRE for x in vmg[0]], [x - PRE for x in vmg[1]], [p.grad for p in dps_],
                    [p.grad for p in dls_], mv, uv, f"{what0}: density factors", grid)


def launch_radiance(cs, bg=1):
    """tir_primary_march / _app_list / _radiance / _radiance_backward once on ``cs`` with random rgb, depth and acc map
    gradients, every parameter gradient prefilled with PRE -> Dump"""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.primary_fused import Workspace, _radiance_job
    lib = _lib.load()
    m, g = cs.m, cs.g
    n_rays = cs.rays.shape[0]
    rays, li = cs.rays, cs.li.reshape(-1).to(torch.int32).contiguous()
    jitter = None if cs.table is not None else cs.jitter
    f = ops.device_field(m).refresh(m, force=True)
    keep = []
    job = _radiance_job(m, keep)
    cfg = ops.march_cfg(m, table=cs.table, n_samples=cs.n_samples, jitter=jitter, keep=keep)
    total = int(march_reference(m, rays, cs.n_samples, jitter, cs.table)["offsets"][-1])
    ws = Workspace(DEV, point_sets=1)
    ws.ensure(n_rays, total + 257, total + 257, 1, True)
    fill_sentinel(ws)
    w = ws.work_struct(None, 1, True)
    w.cap_valid, w.cap_app = total, total
    stream = _lib.stream_ptr()
    _lib.check(lib.tir_primary_march(C.byref(f), _lib.dptr(rays), n_rays, C.byref(cfg), C.byref(w), None, stream),
               "tir_primary_march")
    _lib.check(lib.tir_primary_app_list(C.byref(f), n_rays, C.byref(w), stream), "tir_primary_app_list")
    rgb, depth = torch.full((n_rays, 3), SENT, device=DEV), torch.full((n_rays, 1), SENT, device=DEV)
    _lib.check(lib.tir_primary_radiance(C.byref(f), C.byref(job), _lib.dptr(rays), _lib.dptr(li, torch.int32), n_rays,
                                        C.byref(w), bg, _lib.dptr(rgb), _lib.dptr(depth), stream),
               "tir_primary_radiance")
    gm = dict(rgb=torch.randn(n_rays, 3, generator=g).to(DEV), depth=torch.randn(n_rays, 1, generator=g).to(DEV))
    g_acc_map = torch.randn(n_rays, generator=g).to(DEV)
    b = ws.bwd_struct(1)
    gr = _lib.TirPrimaryGrads()
    vmg = grad_bufs(m, DEV)
    for k in range(3):
        gr.dplane[k], gr.dline[k] = vmg[0][k].data_ptr(), vmg[1][k].data_ptr()
        gr.aplane[k], gr.aline[k] = vmg[2][k].data_ptr(), vmg[3][k].data_ptr()
    g_basis = torch.full_like(m.basis_mat.weight, PRE)
    gr.basis = g_basis.data_ptr()
    ll = getattr(m, "light_line", None)
    g_ll = torch.full_like(ll.weight, PRE) if ll is not None else None
    gr.light_line = None if ll is None else g_ll.data_ptr()
    mlp = m.renderModule.mlp
    mod = {"renderModule": [torch.full_like(x, PRE) for x in (mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias,
                                                               mlp[4].weight, mlp[4].bias)]}
    gr.w0[0], gr.b0[0], gr.w1[0], gr.b1[0], gr.w2[0], gr.b2[0] = [x.data_ptr() for x in mod["renderModule"]]
    _lib.check(lib.tir_primary_radiance_backward(C.byref(f), C.byref(job), _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                                 n_rays, C.byref(w), C.byref(b), bg, _lib.dptr(gm["rgb"]),
                                                 _lib.dptr(gm["depth"]), _lib.dptr(g_acc_map), C.byref(gr), stream),
               "tir_primary_radiance_backward")
    torch.cuda.synchronize()
    return Dump(m=m, ws=ws, rays=rays, li=li, jitter=jitter, table=cs.table, n_samples=cs.n_samples, cv=total,
                ca=total, noise=None, bg=bg, maps=[rgb, depth], mask=None, losses=None, gm=gm, g_acc_map=g_acc_map,
                g_la=None, g_lr=None, vmg=vmg, g_basis=g_basis, g_ll=g_ll, mod=mod, pre=PRE, guards=True, fresh=True)


def check_radiance_stages(d, stats_key=""):
    """Every stage of a radiance-only forward/backward (tir_primary_radiance / _backward) against float64, from the
    dumps and inputs in ``d`` (Dump; ``d.maps`` = [rgb_map, depth_map], ``d.gm`` holds "rgb" and "depth"):
      * march, density, compositing and the appearance list as in check_stages;
      * the head (test_heads_kernels_fp64: gather, Stages.forward, data_grads, param_grads, check_factor_grads);
      * radiance_ray_fwd_kernel: rgb_map = sum_rows w out (+ 1 - acc) and depth_map = depth (+ (1 - acc) rays[..., 5])
        from the kernel's own rows, acc and depth, in R arithmetic with (count) eps32 of sum|w out| for the sum;
      * radiance_ray_bwd_kernel: g_out = w g_rgb (4th column 0), g_weight[a_src] = out . g_rgb (0 on every other
        valid row), g_acc = -(sum g_rgb) - g_depth rays[..., 5] under a background (else 0), g_depth = g_depth_map;
      * compositing backward and the density scatter (back), with no double backward.
    -> dict with the totals"""
    from tensoir_b200.primary_fused import _radiance_job
    from test_heads_kernels_fp64 import P_W
    m, ws, rays, li, bg, PRE = d.m, d.ws, d.rays, d.li, d.bg, d.pre
    t = ws.t
    n_rays = rays.shape[0]
    what0 = f"{stats_key} radiance n_rays {n_rays}"
    c = front(d, what0)
    grid, nv, na, src = c["grid"], c["nv"], c["na"], c["src"]
    if d.guards:
        for k in ("a_w", "a_xn", "out0", "g_out0", "inp0", "h2_0", "gx0_0"):
            assert bool((t[k][na:] == SENT).all()), (what0, k, "guard")
    if na == 0:
        return dict(total=c["total"], total_app=c["total_app"], ws=ws, gates=c["gates"])
    T = {k: v[:na].double() for k, v in t.items() if v.shape[0] == ws.cap_app and v.is_floating_point()}
    ray = t["a_ray"][:na].long()
    aps, als = [p.detach() for p in m.app_plane], [p.detach() for p in m.app_line]
    check_gather(aps, als, grid, T["a_xn"], T["x0_0"], f"{what0}: x0")
    job = _radiance_job(m, [])
    ll = getattr(m, "light_line", None)
    ll64 = ll.weight.detach().double() if ll is not None else None
    mlp = m.renderModule.mlp
    W = [mlp[i].weight.detach().double() for i in (0, 2, 4)]
    B = [mlp[i].bias.detach().double() for i in (0, 2, 4)]
    vd = rays[ray, 3:6].double()
    st = Stages(na, job.light_mode if ll is not None else 0, 0, ll64.shape[0] if ll is not None else 1, W, B,
                m.basis_mat.weight.detach().double(), ll64, li.long()[ray], vd, T["x0_0"], T["inp0"], T["h1_0"],
                T["h2_0"], T["out0"][:, :3])
    st.forward(f"{what0}: head")
    # ================= radiance_ray_fwd_kernel, from the kernel's own rows, acc and depth
    o, aw = T["out0"][:, :3], T["a_w"]
    dz = rays[:, 5].double()
    rgb, depth = radiance_forward(aw, o, ray, t["acc"][:n_rays].double(), t["depth"][:n_rays].double(), dz, bg)
    chk_r(d.maps[0], rgb, f"{what0}: rgb_map", "radiance rgb_map")
    chk_r(d.maps[1].reshape(-1), depth, f"{what0}: depth_map", "radiance depth_map")
    # ================= radiance_ray_bwd_kernel
    zero3 = torch.zeros(n_rays, 3, dtype=torch.float64, device=DEV)
    g = d.gm["rgb"].double().reshape(n_rays, 3) if d.gm.get("rgb") is not None else zero3
    gd = d.gm["depth"].double().reshape(-1) if d.gm.get("depth") is not None else zero3[:, 0]
    g_out, gw, g_acc, g_depth = radiance_backward(aw, o, ray, dz, g, gd, bg)
    chk_r(t["g_acc"][:n_rays], g_acc, f"{what0}: g_acc", "radiance g_acc")
    chk_r(t["g_depth"][:n_rays], g_depth, f"{what0}: g_depth", "radiance g_depth")
    chk_r(T["g_out0"][:, :3], g_out, f"{what0}: g_out", "radiance g_out")
    assert bool((t["g_out0"][:na, 3] == 0).all()), what0
    chk_r(t["g_weight"][:nv].double()[src], gw, f"{what0}: g_weight", "radiance g_weight")
    other = torch.ones(nv, dtype=torch.bool, device=DEV)
    other[src] = False
    assert bool((t["g_weight"][:nv][other] == 0).all()), what0
    # ================= head backward and the appearance factors
    a = st.data_grads(f"{what0}: head", T["g_out0"], T["gz2_0"], T["gz1_0"], T["gfeat0"][:, :NF], T["gx0_0"])
    want, bnds = st.param_grads(T["g_out0"], T["gz2_0"], T["gz1_0"], T["gfeat0"][:, :NF], a)
    for k, buf in zip(("w0", "b0", "w1", "b1", "w2", "b2"), d.mod["renderModule"]):
        chk(buf - PRE, want[k], bnds[k] + sum_bound(PRE, P_W) + 1e-30, f"{what0}: d renderModule.{k}", "head weights")
    chk(d.g_basis - PRE, want["basis"], bnds["basis"] + sum_bound(PRE, P_W) + 1e-30, f"{what0}: d basis_mat",
        "basis_mat")
    if "light" in want:
        chk(d.g_ll - PRE, want["light"], bnds["light"] + sum_bound(PRE, na) + 1e-30, f"{what0}: d light_line",
            "light_line")
    check_factor_grads(aps, als, grid, T["a_xn"], T["gx0_0"], d.vmg[2], d.vmg[3], f"{what0}: appearance factors",
                       prefill=PRE)
    back(d, c, what0, None)
    return dict(total=c["total"], total_app=c["total_app"], ws=ws, gates=c["gates"],
                lengths=t["counts"][:n_rays].clone())


def composite_bwd_bound(r64, bw, bT, gw_pad, ga_tot, gdk, z, g_ext, g_acc_k, gsig64, ds, gfeat64):
    """Bound of primary_composite_bwd_kernel's g_feat in the fp64 regime, from the kernel's arithmetic on the forward's
    saved weight and trans (bounds bw, bT of composite_bounds):
      gw_i = g_weight_i + (g_acc + g_acc_ext) + g_depth z_i: 4 eps32 of its |terms|;
      suffix_i = sum_{j>i} gw_j w_j: the terms' errors |gw_j| bw_j + e_gw_j w_j + eps32 |gw_j w_j|, plus
        eps32 (7 + ceil(S / 32)) (sum|terms| + |gw_i w_i|) for the warp scan (5 levels), the carry over 32-sample
        chunks and the exclusive difference incl - t_i, whose inclusive sum holds t_i as well;
      g_alpha = gw_i T_i - suffix_i / om_i: e_gw T + |gw| bT + (e_suffix + |suffix| rel_om) / (om (1 - rel_om)) plus
        eps32 for the product, the quotient and the difference, with om's relative error rel_om = eps32 (4 + 2 sigma d
        + 1 / om) (composite_bounds);
      g_sigma = g_alpha d expf(-sigma d): eps32 (4 + sigma d) |g_alpha| more (expf's 2 ulp, its argument, 2 products);
      g_feat = g_sigma ds: ds (sigmoid, 4 eps32) times that, plus 5 eps32 |g_feat|.
    -> (bound, the samples it covers: om resolved to a relative error below 1/2)"""
    valid = r64["valid"]
    sig, dd = r64["sig"].detach(), r64["d"]
    alpha, T, w = r64["alpha"].detach(), r64["T"], r64["w"].detach()
    om = torch.where(valid, 1. - alpha + 1e-10, torch.ones_like(alpha))
    e = torch.exp(-sig * dd)
    S = valid.sum(1, keepdim=True).double()
    ga_abs = (g_ext.abs() + g_acc_k.abs())[:, None]
    gw = (gw_pad + ga_tot[:, None] + gdk[:, None] * z) * valid
    e_gw = 4 * EPS32 * (gw_pad.abs() + ga_abs + (gdk[:, None] * z).abs()) * valid
    t_abs = gw.abs() * w
    t_err = gw.abs() * bw + e_gw * w + EPS32 * t_abs

    def after(x):                                                   # sum over j > i
        return x.flip(1).cumsum(1).flip(1) - x
    suf_abs = after(t_abs)
    e_suf = after(t_err) + EPS32 * (7 + torch.ceil(S / 32)) * (suf_abs + t_abs)
    rel_om = EPS32 * (4 + 2 * sig * dd + 1 / om)
    q_abs = suf_abs / om
    e_ga = e_gw * T + gw.abs() * bT + (e_suf + suf_abs * rel_om) / (om * (1 - rel_om)) + \
        3 * EPS32 * (gw.abs() * T + q_abs)
    ga_mag = gw.abs() * T + q_abs
    e_gs = dd * e * (e_ga + EPS32 * (4 + sig * dd) * ga_mag)
    # where om's relative error reaches 1/2 (1 - alpha within 2^-23 of 0) fp32 does not resolve om: those samples
    # join the fp32 regime
    ok = valid & (rel_om < 0.5)
    return torch.where(ok, ds * e_gs + 5 * EPS32 * gfeat64.abs(), torch.zeros_like(e_gs)) + 1e-300, ok


def composite_bounds(r64, fp64_ok, fp32_reg, opaque):
    """Bounds of the fp32 scan on exact sigma (test_secondary_kernels_fp64.reference_march with no sigma error): every
    factor om = 1 - alpha + 1e-10 is off by eps32 (4 + 2 sigma d + 1 / om) relative, T_i by forward_bounds plus
    T_i expm1(sum of those in front of it), w_i by alpha_i times that plus T_i eps32 ((2 + sigma d) e + 2 alpha); in
    the fp32 regime everything is within the bound of T at the ray's first opaque sample plus 2^-21 T there.
    -> (bound of w, bound of T, bound of t_last)"""
    import test_vm_kernels_fp64 as V
    valid, alpha, T = r64["valid"], r64["alpha"].detach(), r64["T"]
    sig, dd = r64["sig"].detach(), r64["d"]
    om = torch.where(valid, 1. - alpha + 1e-10, torch.ones_like(alpha))
    e = torch.exp(-sig * dd)
    rel = torch.where(valid, EPS32 * (4 + 2 * sig * dd + 1 / om), torch.zeros_like(om))
    R_excl = torch.cumsum(rel, 1) - rel
    fb = V.forward_bounds(r64, fp64_ok)
    bT = fb + T * torch.expm1(R_excl)
    bw = alpha * bT + T * (EPS32 * ((2 + sig * dd) * e + 2 * alpha)) + 2.0 ** -126
    S = valid.sum(1).double()
    T_last = r64["T_last"].detach()
    bTl = EPS32 * 8 * (S + 2) * T_last + T_last * torch.expm1(rel.sum(1)) + 2.0 ** -126
    first = fp32_reg.float().argmax(1)
    rows = torch.arange(valid.shape[0], device=DEV)
    Tf = T[rows, first]
    pos_f = valid.cumsum(1)[rows, first].double()
    b32 = Tf * (EPS32 * 8 * (pos_f + 1) + torch.expm1(R_excl[rows, first]) + 2.0 ** -21) + 2.0 ** -125
    bw = torch.where(fp64_ok, bw, torch.where(fp32_reg, b32[:, None], torch.zeros_like(bw)))
    bT = torch.where(fp64_ok, bT, torch.where(fp32_reg, b32[:, None], torch.zeros_like(bT)))
    bTl = torch.where(opaque, b32, bTl)
    return bw, bT, bTl


def _raw2alpha32(sig, dist):
    alpha = 1. - torch.exp(-sig * dist)
    T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1. - alpha + 1e-10], -1), -1)
    return alpha, alpha * T[:, :-1], T[:, -1:]


def _dgrad_scatter(ts, tu, agf, agx):
    """magnitudes of the density-grad double backward's scatter (test_vm_kernels_fp64.test_density_grad_fwd_bwd)"""
    import test_vm_kernels_fp64 as V
    MAT, VEC = V.MAT, V.VEC

    def coef_p(k, q, j):
        sx, sy, sl = q["s"]
        _, w_, dwx, dwy = q["ptaps"][j]
        g0, g1, gv = agx[:, MAT[k][0]] * sx, agx[:, MAT[k][1]] * sy, agx[:, VEC[k]] * sl
        return (agf * w_ + g0 * dwx + g1 * dwy)[:, None] * q["AL"] + (gv * w_)[:, None] * q["AZ"]

    def coef_l(k, q, j):
        sx, sy, sl = q["s"]
        _, w_, kz = q["ltaps"][j]
        g0, g1, gv = agx[:, MAT[k][0]] * sx, agx[:, MAT[k][1]] * sy, agx[:, VEC[k]] * sl
        return q["AP"] * (agf * w_ + gv * kz)[:, None] + w_[:, None] * (g0[:, None] * q["AX"] + g1[:, None] * q["AY"])
    return V.scatter(ts, coef_p, coef_l, 16), V.scatter(tu, coef_p, coef_l, 16)


def assert_gates(gates, rows, what):
    for name, n in gates.n.items():
        STATS[f"ambiguous {name}"] = STATS.get(f"ambiguous {name}", 0) + n
        assert n <= 0.01 * rows + 2, (what, name, n, rows)


def report(what):
    print(f"\n[{what}] " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(STATS.items())))


# ---- cases ------------------------------------------------------------------------------------------------------------
def rotated(kind):
    from gpu_helpers import load_fixture, model_from_fixture
    fx = load_fixture("rotated_g24.pt")
    m = model_from_fixture(fx, DEV)
    m.normals_kind = kind
    return m, fx["rays"], fx["light_idx"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["derived_plus_predicted", "purely_predicted", "purely_derived"])
def test_rotated_g24_stages(kind):
    m, rays, li = rotated(kind)
    res = run_case(Case(m, rays, li, -1, 1), stats_key=f"rotated {kind}")
    assert res["total_app"] > 100
    assert_gates(res["gates"], res["total_app"], kind)
    report(f"rotated {kind}")


@pytest.mark.gpu
def test_lego_bench_batch_stages():
    """The benchmark's field and batch: 4096 rays (four 1024-ray chunks of the offsets scan) and n_samples_for(128)
    samples, so rays longer than two 32-sample chunks of the compositing backward, and the chunk boundaries 31 / 32 /
    33 / 64 / 65 all occur."""
    from tensoir_b200.synthetic import hemisphere_poses, make_lego_model, n_samples_for, training_batch
    m = make_lego_model(128, DEV)
    rays, li = training_batch(hemisphere_poses(100), 4096, 0)
    res = run_case(Case(m, rays, li, n_samples_for(128), 3), stats_key="lego 128")
    lens = set(res["lengths"].tolist())
    print("\nvalid samples per ray present:", sorted(lens & {0, 1, 31, 32, 33, 64, 65}), "max", max(lens))
    assert max(lens) > 64 and 0 in lens, max(lens)
    assert_gates(res["gates"], res["total_app"], "lego")
    report("lego 128")


@pytest.mark.gpu
@pytest.mark.parametrize("bg", [1, 0], ids=["bg", "no_bg"])
def test_radiance_stages(bg):
    """tir_primary_radiance / _backward on rotated_g24 (a light_line model: the head reads each ray's own light) with
    random rgb, depth and acc map gradients, with and without the background term."""
    m, rays, li = rotated("derived_plus_predicted")
    res = check_radiance_stages(launch_radiance(Case(m, rays, li, -1, 8), bg=bg), stats_key=f"rotated bg {bg}")
    assert res["total_app"] > 100
    report(f"radiance bg {bg}")


@pytest.mark.gpu
def test_shrunk_state_b_stages():
    from gpu_helpers import load_shrunk_state, model_from_fixture
    fx = load_shrunk_state("B")
    m = model_from_fixture(fx, DEV, with_mask=True)
    res = run_case(Case(m, fx["rays"], fx["light_idx"], -1, 2), bg=0, stats_key="shrunk B")
    assert res["total_app"] > 100
    assert_gates(res["gates"], res["total_app"], "shrunk B")
    report("shrunk B")


LENGTHS = [0, 1, 31, 32, 33, 64, 65, 2, 17, 47, 70, 0, 1, 96]
H_TABLE = 0.01


def constant_field(feature):
    """rotated_g24 without its alpha mask, the density factors set to one constant (feature = 48 p l everywhere, so
    d feature / d x is exactly 0: every derived normal takes the |v| <= 1e-6 branch), and axis-parallel rays over a z
    table of spacing H_TABLE that start LENGTHS[r] samples in front of the aabb's far x face: ray r has exactly
    LENGTHS[r] valid samples."""
    from gpu_helpers import load_fixture, model_from_fixture
    fx = load_fixture("rotated_g24.pt")
    m = model_from_fixture(fx, DEV, with_mask=False)
    c = math.sqrt(feature / 48.0)
    with torch.no_grad():
        for p in list(m.density_plane) + list(m.density_line):
            p.fill_(c)
    lo, hi = m.aabb[0].cpu().double(), m.aabb[1].cpu().double()
    n = len(LENGTHS)
    rays = torch.zeros(n, 6, dtype=torch.float64)
    for r, L in enumerate(LENGTHS):
        f = (r + 0.5) / n
        rays[r, 0] = hi[0] - L * H_TABLE if L else hi[0] + 0.5 * H_TABLE
        rays[r, 1] = lo[1] + (0.1 + 0.8 * f) * (hi[1] - lo[1])
        rays[r, 2] = lo[2] + (0.9 - 0.8 * f) * (hi[2] - lo[2])
        rays[r, 3] = 1.0
    table = ((torch.arange(128, dtype=torch.float64) + 0.5) * H_TABLE).float().to(DEV)
    li = fx["light_idx"].reshape(-1)[:n]
    return m, rays.float(), li, table


@pytest.mark.gpu
def test_ray_lengths_flat_density_and_a_weight_threshold_tie():
    """Rays of exactly 0, 1, 31, 32, 33, 64, 65 (and 96) valid samples, the compositing backward's chunk edges, in a
    field of constant density (the derived normal's 1e-6 branch on every appearance row); then the same launch with
    rayMarch_weight_thres set to one of the kernel's own weights, so one valid row lies exactly on the threshold."""
    m, rays, li, table = constant_field(10.5)
    cs = Case(m, rays, li, -1, 6, table=table)
    res = run_case(cs, stats_key="lengths")
    assert res["lengths"].tolist() == LENGTHS
    assert res["flat_rows"] == res["total_app"] > 0
    w = res["weights"]
    w_tie = float(w[(w > 1e-3) & (w < 0.2)][3])
    m.rayMarch_weight_thres = w_tie
    res = run_case(cs, stats_key="threshold tie")
    assert int((res["weights"] == torch.tensor(w_tie)).sum()) >= 1
    for r in (res,):
        assert_gates(r["gates"], r["total_app"], "lengths")
    report("lengths")


@pytest.mark.gpu
def test_transmittance_reaches_zero():
    """A constant density with sigma d about 20: fp32 alpha rounds to 1 on every sample, T falls by 1e-10 per sample
    and is exactly 0 from the sixth sample of a ray on."""
    m, rays, li, table = constant_field(90.0)
    cs = Case(m, rays, li, -1, 7, table=table)
    res = run_case(cs, stats_key="T = 0")
    assert res["t_zero"] > 0 and res["t_last_zero"] > 0
    assert_gates(res["gates"], max(res["total_app"], 1), "T = 0")
    report("T = 0")


@pytest.mark.gpu
def test_capacities_below_the_totals():
    """cap_valid and cap_app below the real totals, a guard of sentinel rows behind each: both overflow flags are set,
    nothing is written past either capacity, and forward and backward equal the references of the cut lists."""
    m, rays, li = rotated("derived_plus_predicted")
    cs = Case(m, rays, li, -1, 4)
    probe = run_case(cs, stats_key="probe")
    assert int(probe["ws"].t["status"][2]) == 0
    cv = probe["total"] * 2 // 3
    # the appearance list alone overflows, then both lists
    for kw in (dict(cap_app=probe["total_app"] // 2), dict(cap_valid=cv, cap_app=probe["total_app"] // 3)):
        res = run_case(cs, stats_key="capacity", **kw)
        assert int(res["ws"].t["status"][2]) == 1, kw
        assert_gates(res["gates"], res["total_app"], "capacity")
    report("capacity")


@pytest.mark.gpu
def test_consecutive_launches_on_one_workspace():
    """Three forward/backward launches of different ray counts on one workspace: offsets past n_rays hold stale values
    of the launch before."""
    from tensoir_b200.primary_fused import Workspace
    m, rays, li = rotated("purely_derived")
    cs = Case(m, rays, li, -1, 5)
    n = cs.rays.shape[0]
    ws = Workspace(DEV)
    ws.ensure(n, 96 * n + 1024, 96 * n + 1024, 3, True)
    for k in (n, n // 3, (2 * n) // 3):
        res = run_case(cs, ws=ws, n_rays=k, stats_key="consecutive")
        assert_gates(res["gates"], res["total_app"], "consecutive")
    report("consecutive")
