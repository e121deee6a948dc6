"""The shading kernels against float64: tir_shade_fwd / _bwd (the list form that render_with_BRDF uses) and
tir_shade_hits_fwd / _bwd (the hits form that render_hits runs on every relight-phase training step), csrc/tir_shade.cu
with the GGX terms of csrc/tir_ggx.h, forward and backward, called through the C ABI.

The reference restates the kernel's own expression in float64: the raw-normal cosine, normalisation with eps 1e-12,
sign(NoV), the [1e-6, 1] clamps, the [1e-6, 4 pi] clamp of nom, the quadrature and (hits form) tone; and the backward is
the kernel's analytic formulas written out, not autograd.  Its constants are the kernel's fp32 constants (pi, 1e-6,
the Fresnel and sRGB coefficients, including the compile-time folded 1.055f / 2.4f and 1.f / 2.4f - 1.f of tone_grad),
so the reference is the kernel's expression in exact arithmetic.  ``test_reference_backward_matches_autograd_cpu`` pins
the explicit backward to float64 autograd of the forward away from kinks, to 1e-10 relative.

Bounds, per entry.  Every intermediate x of the reference is carried as a pair (value, e) where e bounds |x32 - x|, the
distance of the kernel's fp32 value from the float64 one (class ``R``).  With u = eps32 = 2^-23 (twice the unit
roundoff, so one correctly rounded op is covered with a factor 2 to spare) the rules are:
  * a + b:  e_a + e_b + u (|a + b| + e_a + e_b)              (the fp32 result is rounded once)
  * a * b:  |a| e_b + |b| e_a + e_a e_b + u (|ab| + that)     (exact in the inputs' errors, not first order)
  * a / b:  (e_a + |a/b| e_b) / (|b| - e_b) + u (...)           (infinite when e_b >= |b|)
  * sqrt:   min(e / sqrt(x), sqrt(e)) + u (...);  exp2f: 2^x (2^e - 1) + 2u 2^x (the CUDA Math API's 2 ulp);
    powf(x, y): |y| max((x - e)^(y - 1), (x + e)^(y - 1)) e + 4u x^y (its 4 ulp); mean-value bounds at the worst
    end of [x - e, x + e], so not first order
  * clamp / fmaxf: 1-Lipschitz, so e passes through; where the value is clamped by more than e, the result is exact
  * a contraction: the errors of its terms plus c u (sum |terms| + sum e) with c the longest chain of fp32 additions
    any term goes through, independent of the order: 2 for a 3-vector dot product or the 3 channels of a direction;
    ceil(nl / 32) + 5 for the quadrature and every per-row backward sum (lane-strided partial sums, then the 5-level
    warp butterfly); 3 ceil(nl / 32) + 5 for d NoV, whose lanes accumulate the three channels of every direction
  * g_direct (shared-memory atomics per CTA, then global atomics onto whatever the buffer held): the terms' errors
    plus ``sum_bound`` (test_heads_kernels_fp64.py) of sum |terms| + |initial value| over the rows of each light.
An FMA contraction by the device compiler rounds once where these rules round twice, so it stays inside them.

Kinks.  A gate takes a branch from a value; when the float64 value lies within its own bound e of the threshold, fp32
may take the other branch.  The clamps of NoL, NoH, NoV and nom, ``cosr > 0`` and the [0, 1] tone clamp are continuous
in the forward, so the Lipschitz rule above covers them.  In the backward each of them switches a term on or off: where
it is ambiguous, the whole term (value and its e) is added to its bound (``gate``), which is the jump between the two
branches.  sign(NoV) flips the whole row: an ambiguous row is evaluated again with the other signs, and the largest
difference plus that evaluation's bound goes into every entry of the row.  The tone gates (clamp, sRGB threshold)
read the kernel's own saved ``lin``, so the reference takes the kernel's branch there and no kink arises.  Every case
counts its ambiguous entries and asserts they are a small fraction: ambiguous sign and NoV-clamp rows are the views
placed 1e-7 off grazing on purpose (one row in ten) plus at most 1 % of the rows; ambiguous NoL, NoH and cos gates stay
below 1 % of the (row, direction) pairs and nom below 1 % of the (row, direction, channel) entries.  Every bound handed
to the comparison must be finite, so none can go vacuous by a divisor within its own error of 0.

Cases cover both forms; 1, 37, 2 num_sms 8 + 5 (the first row of the backward grid's second grid-stride pass, plus 4)
and 4096 rows; 512, 128 and 60 directions with area weights and equal 4 pi / nl weights; 1, 3, 8 (a 48 KB table), 9
(the shared-memory opt-in) and 33 lights (the largest table at 512 directions); roughness uniform over [0.09, 0.99] with
blocks at exactly 0.09 and 0.99; back-facing, grazing (|NoV| ~ 1e-7 and 1e-5) and mirror views (NoH ~ 1, so at
roughness 0.09 the nom clamp is active and gates g_nom off); vis with exact 0s and 1s; and per-row light scales that put
the hits form's lin at 0, below 0.0031308, in the nonlinear branch and above 1."""
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import tensoir_oracle as O
from test_heads_kernels_fp64 import check, sum_bound

DEV = "cuda:0"
EPS = 2.0 ** -23
ULP_EXP2, ULP_POW = 2.0, 4.0                     # CUDA Math API maximum ulp errors of exp2f and powf
SENTINEL = 7.0


def f32(x):
    return float(np.float32(x))


PI = f32(math.pi)                                # kPi
FOUR_PI = 4.0 * PI                               # 4.f * kPi (exact)
LO = f32(1e-6)
TINY = f32(1e-12)
FM_A, FM_B = f32(-5.55473), f32(6.98316)
SRGB_T, SRGB_S, SRGB_A, SRGB_B = f32(0.0031308), f32(12.92), f32(1.055), f32(0.055)
SRGB_E = float(np.float32(1.0) / np.float32(2.4))                       # 1.f / 2.4f
TG_A = float(np.float32(1.055) / np.float32(2.4))                       # 1.055f / 2.4f
TG_E = float(np.float32(SRGB_E) - np.float32(1.0))                      # 1.f / 2.4f - 1.f


# ------------------------------------------------------------------------------------------------------------------
# float64 value with an fp32 error bound
# ------------------------------------------------------------------------------------------------------------------
def _abs(x):
    return x.abs() if torch.is_tensor(x) else abs(x)


def _d(x):
    return x.detach() if torch.is_tensor(x) else x


class R:
    """A float64 value ``v`` of the kernel's expression and ``e``, a bound on |fp32 value - v| (module docstring)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(_d(v)) if e is None else e

    @staticmethod
    def rnd(v, e, c=1.0):
        return R(v, e + c * EPS * (_d(v).abs() + e))

    def __getitem__(self, i):
        return R(self.v[i], self.e[i])

    def __neg__(self):
        return R(-self.v, self.e)

    def __add__(self, b):
        if isinstance(b, R):
            return R.rnd(self.v + b.v, self.e + b.e)
        return R.rnd(self.v + b, self.e)

    __radd__ = __add__

    def __sub__(self, b):
        return self + (-b)

    def __rsub__(self, b):
        return (-self) + b

    def __mul__(self, b):
        if isinstance(b, R):
            return R.rnd(self.v * b.v, self.e * _d(b.v).abs() + b.e * _d(self.v).abs() + self.e * b.e)
        return R.rnd(self.v * b, self.e * _abs(_d(b)))

    __rmul__ = __mul__

    def __truediv__(self, b):
        if isinstance(b, R):
            q = self.v / b.v
            den = (_d(b.v).abs() - b.e).clamp_min(0.0)
            return R.rnd(q, (self.e + _d(q).abs() * b.e) / den)
        return R.rnd(self.v / b, self.e / _abs(b))

    def __rtruediv__(self, a):                  # a constant over self
        q = a / self.v
        den = (_d(self.v).abs() - self.e).clamp_min(0.0)
        return R.rnd(q, _d(q).abs() * self.e / den)

    def sqrt(self):
        s = self.v.sqrt()
        # |sqrt(x + e) - sqrt(x)| <= min(e / sqrt(x), sqrt(e)); an exact input adds only the rounding
        return R.rnd(s, torch.where(self.e > 0, torch.minimum(self.e / _d(s), self.e.sqrt()), 0.0))

    def exp2(self):
        p = torch.exp2(self.v)
        return R.rnd(p, _d(p) * torch.expm1(self.e * math.log(2.0)), ULP_EXP2)

    def pow(self, y):
        p = self.v ** y
        lo, hi = (_d(self.v) - self.e).clamp_min(0.0), _d(self.v) + self.e
        slope = torch.maximum(lo ** (y - 1.0), hi ** (y - 1.0))           # y < 1: lo is the worst end, y > 1: hi
        return R.rnd(p, abs(y) * slope * self.e, ULP_POW)

    def clamp(self, lo=-math.inf, hi=math.inf):
        v = _d(self.v)
        exact = (v < lo - self.e) | (v > hi + self.e)
        return R(self.v.clamp(lo, hi), torch.where(exact, torch.zeros_like(self.e), self.e))

    def sum(self, dim, c):
        return R(self.v.sum(dim), self.e.sum(dim) + c * EPS * (_d(self.v).abs().sum(dim) + self.e.sum(dim)))


def dot3(a, b):
    return (a * b).sum(-1, 2.0)


class Gates:
    """Counts the ambiguous entries of every gate (module docstring, kinks)."""

    def __init__(self):
        self.n = {}

    def gate(self, term, x, lo, hi, name, strict=False):
        """term where lo <= x <= hi (0 < x when ``strict``), else 0; an ambiguous gate adds the whole term."""
        v = _d(x.v)
        dec = (v > lo) if strict else ((v >= lo) & (v <= hi))
        amb = (v - lo).abs() <= x.e
        if hi != math.inf:
            amb |= (v - hi).abs() <= x.e
        amb &= x.e > 0                          # an exact value takes the kernel's branch
        self.n[name] = self.n.get(name, 0) + int(amb.sum())
        while dec.dim() < _d(term.v).dim():
            dec, amb = dec[..., None], amb[..., None]
        dec, amb = dec.to(term.e.dtype), amb.to(term.e.dtype)
        return R(term.v * dec, term.e * torch.maximum(dec, amb) + _d(term.v).abs() * amb)


# ------------------------------------------------------------------------------------------------------------------
# the kernel's shading, forward and explicit backward, in float64
# ------------------------------------------------------------------------------------------------------------------
def tone(lin, srgb):
    """tone() of tir_ggx.h on a value (the kernel's saved lin) or on an R; returns R.  Where an R lies within its
    bound of the sRGB threshold, the jump between the two branches is added to the bound."""
    t = (lin if isinstance(lin, R) else R(lin)).clamp(0.0, 1.0)
    if not srgb:
        return t
    lo = t * SRGB_S
    hi = (t + LO).pow(SRGB_E) * SRGB_A - SRGB_B
    sel = _d(t.v) <= SRGB_T
    amb = ((_d(t.v) - SRGB_T).abs() <= t.e) & (t.e > 0)
    jump = torch.where(amb, (lo.v - hi.v).abs() + torch.maximum(lo.e, hi.e), torch.zeros_like(t.e))
    return R(torch.where(sel, lo.v, hi.v), torch.where(sel, lo.e, hi.e) + jump)


def tone_grad(lin, srgb):
    """tone_grad() of tir_shade.cu on the kernel's saved lin; returns R."""
    inside = ((lin >= 0) & (lin <= 1)).to(lin.dtype)
    if not srgb:
        return R(inside)
    hi = (R(lin).clamp(0.0, 1.0) + LO).pow(TG_E) * TG_A
    v = torch.where(lin <= SRGB_T, torch.full_like(lin, SRGB_S), hi.v) * inside
    e = torch.where(lin <= SRGB_T, torch.zeros_like(lin), hi.e) * inside
    return R(v, e)


def ggx_ref(N, Vr, F0r, Rr, L, sgn=None):
    """ggx_point, ggx_dir and ggx_terms of tir_ggx.h in float64 (R): N, Vr, F0r, Rr [m,3] as the kernel loads them,
    L [nl,3] directions shared by every row or [m,nl,3] per row, both as stored; sgn [m] replaces sign(nov).  Returns
    a namespace of the intermediates the shading forward and backward read; spec is GGX_specular [m,nl,3]."""
    # ggx_point
    inv_nn = 1.0 / dot3(N, N).sqrt().clamp(TINY)
    inv_vn = 1.0 / dot3(Vr, Vr).sqrt().clamp(TINY)
    Vn = Vr * inv_vn[:, None]
    nov = (Vn * N * inv_nn[:, None]).sum(-1, 2.0)
    s = torch.sign(_d(nov.v)) if sgn is None else sgn
    Np = N * inv_nn[:, None] * s[:, None]
    nov2 = dot3(Np, Vn)
    NoV = nov2.clamp(LO, 1.0)
    al = Rr * Rr
    alpha2 = al * al
    k = (al + Rr * 2.0 + 1.0) / 8.0
    nom1 = NoV[:, None] * (1.0 - k) + k
    # ggx_dir, [m|1,nl]
    L = L if L.v.dim() == 3 else L[None]
    cosr = dot3(L, N[:, None])                                          # [m,nl] raw L . n
    cosv = cosr.clamp(0.0)
    inv_ln = 1.0 / dot3(L, L).sqrt().clamp(TINY)
    Ln = L * inv_ln[..., None]
    H = (Ln + Vn[:, None]) * 0.5
    Hn = H * (1.0 / dot3(H, H).sqrt().clamp(TINY))[..., None]
    NoL_raw, NoH_raw, VoH_raw = dot3(Np[:, None], Ln), dot3(Np[:, None], Hn), dot3(Vn[:, None], Hn)
    NoL, NoH, VoH = NoL_raw.clamp(LO, 1.0), NoH_raw.clamp(LO, 1.0), VoH_raw.clamp(LO, 1.0)
    p2 = ((VoH * FM_A - FM_B) * VoH).exp2()
    # ggx_terms, [m,nl,3]
    F0c, al2, kc, n1 = F0r[:, None], alpha2[:, None], k[:, None], nom1[:, None]
    NoHc, NoLc, p2c = NoH[..., None], NoL[..., None], p2[..., None]
    frac0 = F0c + (1.0 - F0c) * p2c
    frac = frac0 * al2
    nom0 = NoHc * NoHc * (al2 - 1.0) + 1.0
    nom2 = NoLc * (1.0 - kc) + kc
    nomr = FOUR_PI * nom0 * nom0 * n1 * nom2
    nom = nomr.clamp(LO, FOUR_PI)
    spec = frac / nom
    return types.SimpleNamespace(inv_nn=inv_nn, Vn=Vn, nov=nov, s=s, Np=Np, nov2=nov2, NoV=NoV, k=k, cosr=cosr,
                                 cosv=cosv, Ln=Ln, Hn=Hn, NoL_raw=NoL_raw, NoH_raw=NoH_raw, F0c=F0c, al2=al2, kc=kc,
                                 n1=n1, NoHc=NoHc, NoLc=NoLc, p2c=p2c, frac0=frac0, nom0=nom0, nom2=nom2, nomr=nomr,
                                 nom=nom, spec=spec)


def shade_ref(n, V, a, F0, r, dirs, w, D, vis, ind, go=None, sgn=None, gates=None):
    """One row block: n, V, a, F0, r [m,3] (V as loaded: the list form's view or minus the ray direction; r broadcast
    over the channels in the hits form), dirs [nl,3], w [nl], D = direct[light] [m,nl,3], vis [m,nl], ind [m,nl,3],
    go [m,3] (R) the gradient reaching the linear value.  Returns a dict of R: lin [m,3]; with go also g_normal,
    g_albedo, g_fresnel, g_rough [m,3] (per channel, before any channel sum) and gd [m,nl,3], each row's term of the
    direct-light gradient; plus nov, the value whose sign picks the normal's side."""
    gates = gates if gates is not None else Gates()
    nl = dirs.shape[0]
    c_lane = math.ceil(nl / 32) + 5
    N, Vr, A, F0r, Rr = R(n), R(V), R(a), R(F0), R(r)
    g = ggx_ref(N, Vr, F0r, Rr, R(dirs), sgn)
    inv_nn, Vn, nov, s, Np, nov2, NoV, k = g.inv_nn, g.Vn, g.nov, g.s, g.Np, g.nov2, g.NoV, g.k
    cosr, cosv, Ln, Hn, NoL_raw, NoH_raw = g.cosr, g.cosv, g.Ln, g.Hn, g.NoL_raw, g.NoH_raw
    F0c, al2, kc, n1, NoHc, NoLc, p2c = g.F0c, g.al2, g.kc, g.n1, g.NoHc, g.NoLc, g.p2c
    frac0, nom0, nom2, nomr, nom, spec = g.frac0, g.nom0, g.nom2, g.nomr, g.nom, g.spec
    brdf = A[:, None] / PI + spec
    light = R(vis)[..., None] * R(D) + R(ind)
    cw = cosv * R(w)[None]
    lin = (brdf * light * cw[..., None]).sum(1, c_lane)
    out = dict(lin=lin, nov=nov)
    if go is None:
        return out
    # shade_bwd_kernel
    gc = go[:, None, :] * R(w)[None, :, None]
    g_brdf = gc * light * cosv[..., None]
    g_cos = (gc * brdf * light).sum(-1, 2.0)
    out["gd"] = gc * brdf * cosv[..., None] * R(vis)[..., None]
    ga_t = g_brdf / PI
    g_frac = g_brdf / nom
    g_nom = gates.gate(-g_brdf * spec / nom, nomr, LO, FOUR_PI, "nom")
    base = g_nom * FOUR_PI
    g_nom0 = base * 2.0 * nom0 * n1 * nom2
    g_nom1 = base * nom0 * nom0 * nom2
    g_nom2 = base * nom0 * nom0 * n1
    gal2_t = g_frac * frac0 + g_nom0 * NoHc * NoHc
    gF0_t = g_frac * al2 * (1.0 - p2c)
    g_NoH = (g_nom0 * 2.0 * NoHc * (al2 - 1.0)).sum(-1, 2.0)
    g_NoL = (g_nom2 * (1.0 - kc)).sum(-1, 2.0)
    gk_t = g_nom2 * (1.0 - NoLc) + g_nom1 * (1.0 - NoV[:, None, None])
    gNoV_t = g_nom1 * (1.0 - kc)
    g_NoL = gates.gate(g_NoL, NoL_raw, LO, 1.0, "NoL")
    g_NoH = gates.gate(g_NoH, NoH_raw, LO, 1.0, "NoH")
    gNp_t = g_NoL[..., None] * Ln + g_NoH[..., None] * Hn
    gn_t = gates.gate(g_cos[..., None] * R(dirs)[None], cosr, 0.0, math.inf, "cos", strict=True)
    gNp, gn, ga, gF0, gal2, gk = (t.sum(1, c_lane) for t in (gNp_t, gn_t, ga_t, gF0_t, gal2_t, gk_t))
    m = n.shape[0]
    gNoV = R(gNoV_t.v.reshape(m, -1), gNoV_t.e.reshape(m, -1)).sum(1, 3 * math.ceil(nl / 32) + 5)
    gNoV = gates.gate(gNoV, nov2, LO, 1.0, "NoV")
    # lane 0
    gNn = (gNp + gNoV[:, None] * Vn) * s[:, None]
    Nn = N * inv_nn[:, None]
    dot = dot3(Nn, gNn)
    out["g_normal"] = gn + (gNn - Nn * dot[:, None]) * inv_nn[:, None]
    out["g_albedo"], out["g_fresnel"] = ga, gF0
    out["g_rough"] = gal2 * 4.0 * Rr * Rr * Rr + gk * (Rr * 2.0 + 2.0) / 8.0
    return out


OUT_KEYS = ("lin", "g_normal", "g_albedo", "g_fresnel", "g_rough", "gd")


def shade_ref_rows(args, go, gates):
    """shade_ref with the sign(NoV) kink: rows whose nov is within its bound of 0 are evaluated again with the other
    signs of {-1, 0, 1}, and each difference plus that evaluation's bound is added to every entry of the row."""
    out = shade_ref(*args, go=go, gates=gates)
    nov = out["nov"]
    amb = (nov.v.abs() <= nov.e).nonzero().reshape(-1)
    gates.n["sign"] = gates.n.get("sign", 0) + int(amb.numel())
    if amb.numel():
        sub = [t if i in (5, 6) else t[amb] for i, t in enumerate(args)]          # dirs and weights are shared
        s0 = torch.sign(nov.v[amb])
        for c in (-1.0, 0.0, 1.0):
            other = s0 != c
            if not bool(other.any()):
                continue
            alt = shade_ref(*sub, go=go[amb] if go is not None else None, sgn=torch.full_like(s0, c), gates=Gates())
            for key in OUT_KEYS:
                if key not in out:
                    continue
                d = (alt[key].v - out[key].v[amb]).abs() + alt[key].e
                d = d * other.reshape(-1, *[1] * (d.dim() - 1)).to(d.dtype)
                out[key].e[amb] = out[key].e[amb] + d
    return out


# ------------------------------------------------------------------------------------------------------------------
# CPU: the explicit backward equals autograd of the forward
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("srgb", [None, 0, 1])
def test_reference_backward_matches_autograd_cpu(srgb):
    """shade_ref's explicit backward (and tone_grad) equal float64 autograd of shade_ref's forward (and tone), on rows
    away from every kink, to 1e-10 relative to each gradient's largest entry."""
    g = torch.Generator().manual_seed(5 + (srgb or 0) + (srgb is None))
    d = torch.float64
    m = 23
    w, dirs = O.generate_envir_map_dir(6, 10)
    dirs, w = dirs.to(d), w.to(d)
    nl = dirs.shape[0]
    n = F.normalize(torch.randn(m, 3, generator=g, dtype=d), dim=-1) * (torch.rand(m, 1, generator=g, dtype=d) + 0.5)
    V = F.normalize(torch.randn(m, 3, generator=g, dtype=d), dim=-1)
    a = torch.rand(m, 3, generator=g, dtype=d)
    F0 = torch.rand(m, 3, generator=g, dtype=d)
    r = torch.rand(m, 3, generator=g, dtype=d) * 0.6 + 0.3
    if srgb is not None:
        r = r[:, :1].expand(m, 3)
    L = 3
    direct = torch.rand(L, nl, 3, generator=g, dtype=d) * 2
    li = torch.arange(m) % L
    vis = torch.rand(m, nl, generator=g, dtype=d)
    ind = torch.rand(m, nl, 3, generator=g, dtype=d) * (0.3 if srgb is None else 0.05)
    g_rgb = torch.randn(m, 3, generator=g, dtype=d)
    leaves = [t.clone().requires_grad_(True) for t in (n, a, F0, r, direct)]
    nL, aL, FL, rL, dL = leaves
    gates = Gates()
    lin = shade_ref(nL, V, aL, FL, rL, dirs, w, dL[li], vis, ind, gates=gates)["lin"].v
    if srgb is None:
        y, go = lin, R(g_rgb)
    else:
        t = lin.clamp(0, 1)
        y = torch.where(t <= SRGB_T, t * SRGB_S, SRGB_A * (t + LO) ** SRGB_E - SRGB_B) if srgb else t
        tg = tone_grad(lin.detach(), srgb)
        # the kernel's folded constants differ from the exact derivative of tone's by a known factor
        fix = torch.where(lin.detach() <= SRGB_T, torch.ones_like(lin.detach()),
                          (TG_A / (SRGB_A * SRGB_E)) * (lin.detach().clamp(0, 1) + LO) ** (TG_E - (SRGB_E - 1)))
        if not srgb:
            fix = torch.ones_like(fix)
        (want_tg,) = torch.autograd.grad(y.sum(), lin, retain_graph=True)
        assert torch.allclose(tg.v, want_tg * fix, rtol=1e-12, atol=0), "tone_grad"
        go = R(g_rgb * want_tg)
    (y * g_rgb).sum().backward()
    got = shade_ref(n, V, a, F0, r, dirs, w, direct[li], vis, ind, go=go, gates=gates)
    # away from kinks: no gate ambiguous, and no value at a threshold
    assert all(v == 0 for v in gates.n.values()), gates.n
    gd = torch.zeros(L, nl, 3, dtype=d).index_add_(0, li, got["gd"].v)
    gr = got["g_rough"].v
    if srgb is not None:
        gr = gr.sum(1, keepdim=True)
        rL_grad = rL.grad[:, :1] + rL.grad[:, 1:2] + rL.grad[:, 2:]   # rough1.repeat(1, 3) sums the channels
    else:
        rL_grad = rL.grad
    for what, x, y_ in (("normal", got["g_normal"].v, nL.grad), ("albedo", got["g_albedo"].v, aL.grad),
                        ("fresnel", got["g_fresnel"].v, FL.grad), ("rough", gr, rL_grad), ("direct", gd, dL.grad)):
        err = float((x - y_).abs().max()) / float(y_.abs().max())
        assert err < 1e-10, (what, err)


def test_bounds_are_exact_for_exact_inputs_cpu():
    """R's rules on a few fp32 computations done in fp32: the fp32 result is within the bound of the float64 value."""
    g = torch.Generator().manual_seed(2)
    x32 = torch.rand(10000, generator=g) + 0.01
    y32 = torch.rand(10000, generator=g) - 0.5
    X, Y = R(x32.double()), R(y32.double())
    for got, want in ((x32 * y32 + x32, X * Y + X), (x32 / (y32 + 2), X / (Y + 2.0)),
                      (torch.sqrt(x32 * x32 + y32 * y32), (X * X + Y * Y).sqrt()),
                      (1.0 / (x32 - y32 * y32), 1.0 / (X - Y * Y))):
        assert bool(((got.double() - want.v).abs() <= want.e).all())


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernels on constructed cases
# ------------------------------------------------------------------------------------------------------------------
def directions(h, w_, equal, g):
    """(dirs [nl,3], weight [nl]) fp32: the fixed environment grid with its area weights, or the equal-area
    stratified sample with 4 pi / nl each."""
    if not equal:
        wt, dirs = O.generate_envir_map_dir(h, w_)
        return dirs.float().contiguous(), wt.float().contiguous()
    jit = (torch.rand(h, w_, generator=g), torch.rand(h, w_, generator=g))
    dirs = O.gen_light_incident_dirs(types.SimpleNamespace(envmap_h=h, envmap_w=w_), 'stratifed_sample_equal_areas',
                                     jit).float().contiguous()
    return dirs, torch.full((dirs.shape[0],), 4 * math.pi / dirs.shape[0])


def make_case(form, m, h, w_, equal, L, seed):
    """Inputs of one case (fp32, CPU).  Row i has geometry class i % 10 and light scale class (i // 3 + 2) % 5."""
    g = torch.Generator().manual_seed(seed)
    dirs, wt = directions(h, w_, equal, g)
    nl = dirs.shape[0]
    nh = F.normalize(torch.randn(m, 3, generator=g, dtype=torch.float64), dim=-1)
    view = F.normalize(torch.randn(m, 3, generator=g, dtype=torch.float64), dim=-1)
    cls = torch.arange(m) % 10
    # grazing views: |NoV| about 1e-7 (class 4) and 1e-5 (class 5)
    tang = F.normalize(view - (view * nh).sum(-1, keepdim=True) * nh, dim=-1)
    sgn = torch.where(torch.rand(m, 1, generator=g) < 0.5, -1.0, 1.0).double()
    for c, eps in ((4, 1e-7), (5, 1e-5)):
        view[cls == c] = F.normalize(tang + sgn * eps * nh, dim=-1)[cls == c]
    # mirror views (classes 6, 7): the reflection of a direction with L . n > 0.3 about the normal
    cosd = nh @ F.normalize(dirs.double(), dim=-1).t()
    pick = torch.multinomial((cosd > 0.3).double() + 1e-12, 1, generator=g).reshape(-1)
    Lk = F.normalize(dirs.double()[pick], dim=-1)
    mirror = 2 * (nh * Lk).sum(-1, keepdim=True) * nh - Lk
    mm = (cls == 6) | (cls == 7)
    view[mm] = mirror[mm]
    normal = (nh * (torch.rand(m, 1, generator=g) * 1.5 + 0.5)).float()
    if form == "list":
        rough = torch.rand(m, 3, generator=g) * 0.9 + 0.09
    else:
        rough = torch.rand(m, 1, generator=g) * 0.9 + 0.09
    rough[(cls == 6) | (cls == 8)] = f32(0.09)
    rough[cls == 9] = f32(0.99)
    fres = torch.rand(m, 3, generator=g)
    fres[(cls == 3) | (cls == 6) | (cls == 8)] = f32(0.04)
    albedo = torch.rand(m, 3, generator=g)
    vis = torch.rand(m, nl, generator=g)
    u = torch.rand(m, nl, generator=g)
    vis[u < 0.2] = 0.0
    vis[u > 0.8] = 1.0
    ind = torch.rand(m, nl, 3, generator=g) * 0.3
    tone_cls = (torch.arange(m) // 3 + 2) % 5
    vis[tone_cls == 0] = 0.0                                     # lin = 0
    ind[tone_cls == 0] = 0.0
    vis[tone_cls == 1] *= 1e-4                                   # lin <= 0.0031308
    ind[tone_cls == 1] *= 1e-4
    ind[tone_cls == 4] *= 30                                     # lin > 1
    direct = torch.rand(L, nl, 3, generator=g) * 2
    li = (torch.arange(m) % L)[torch.randperm(m, generator=g)].to(torch.int32)
    mask = torch.rand(m, generator=g) > 0.3 if form == "hits" else torch.ones(m, dtype=torch.bool)
    if m == 1:
        mask[:] = True
    for j in range(L):                                           # every light id, the last included, is shaded
        mask[(li == j).nonzero()[0]] = True
    g_rgb = torch.randn(m, 3, generator=g)
    view32 = view.float()
    rays = torch.cat([torch.randn(m, 3, generator=g), -view32], 1)
    return dict(normal=normal, albedo=albedo, rough=rough, fresnel=fres, view=view32, rays=rays, mask=mask, light=li,
                dirs=dirs, weight=wt, direct=direct, vis=vis, ind=ind, g_rgb=g_rgb, grazing=int((cls == 4).sum()))


def run_kernels(form, x, srgb):
    """Forward twice and backward once through the C ABI; every output starts as a finite sentinel, g_direct as a
    non-zero buffer.  Returns (rgb, lin or None, grads dict, g_direct start)."""
    from tensoir_b200 import _lib
    lib = _lib.load()
    d = {k: (v.to(DEV).contiguous() if torch.is_tensor(v) else v) for k, v in x.items()}
    m, nl, L = d["normal"].shape[0], d["dirs"].shape[0], d["direct"].shape[0]
    P = _lib.dptr
    st = _lib.stream_ptr()
    common = (P(d["dirs"]), P(d["weight"]), nl, P(d["direct"]), L, P(d["vis"]), P(d["ind"]))
    outs = []
    for _ in range(2):
        rgb = torch.full((m, 3), SENTINEL, device=DEV)
        lin = torch.full((m, 3), SENTINEL, device=DEV)
        if form == "list":
            _lib.check(lib.tir_shade_fwd(P(d["normal"]), P(d["albedo"]), P(d["rough"]), P(d["fresnel"]), P(d["view"]),
                                         P(d["light"], torch.int32), m, *common, P(rgb), st), "tir_shade_fwd")
        else:
            _lib.check(lib.tir_shade_hits_fwd(P(d["rays"]), P(d["mask"], torch.bool), P(d["normal"]), P(d["albedo"]),
                                              P(d["rough"]), P(d["fresnel"]), P(d["light"], torch.int32), m, *common,
                                              srgb, P(rgb), P(lin), st), "tir_shade_hits_fwd")
        outs.append((rgb, lin))
    (rgb, lin), (rgb2, lin2) = outs
    torch.cuda.synchronize()
    assert torch.equal(rgb, rgb2) and torch.equal(lin, lin2), "two launches differ"
    gr = {k: torch.full_like(d[s], SENTINEL) for k, s in (("g_normal", "normal"), ("g_albedo", "albedo"),
                                                          ("g_rough", "rough"), ("g_fresnel", "fresnel"))}
    gd0 = (torch.rand(L, nl, 3, generator=torch.Generator().manual_seed(m)) - 0.5).to(DEV)
    gd = gd0.clone()
    tail = (P(gr["g_normal"]), P(gr["g_albedo"]), P(gr["g_rough"]), P(gr["g_fresnel"]), P(gd), st)
    if form == "list":
        rc = lib.tir_shade_bwd(P(d["normal"]), P(d["albedo"]), P(d["rough"]), P(d["fresnel"]), P(d["view"]),
                               P(d["light"], torch.int32), m, *common, P(d["g_rgb"]), *tail)
    else:
        rc = lib.tir_shade_hits_bwd(P(d["rays"]), P(d["mask"], torch.bool), P(d["normal"]), P(d["albedo"]),
                                    P(d["rough"]), P(d["fresnel"]), P(d["light"], torch.int32), m, *common, srgb,
                                    P(lin), P(d["g_rgb"]), *tail)
    _lib.check(rc, f"tir_shade{'_hits' if form == 'hits' else ''}_bwd")
    torch.cuda.synchronize()
    gr["g_direct"] = gd
    return rgb, (lin if form == "hits" else None), gr, gd0


def check_fin(got, want, bnd, what):
    """check() with a finite bound: a bound that went infinite (a divisor within its own error of 0) would pass
    anything."""
    assert bool(torch.isfinite(torch.as_tensor(bnd)).all()), (what, "non-finite bound")
    check(got, want, bnd, what)


def assert_gates(n_gates, n_rows, nl, grazing, what):
    """Ambiguous entries stay few, each gate against its own entry count: sign and NoV rows at most the rows placed
    1e-7 off grazing plus 1 % of the rows; NoL, NoH and cos at most 1 % of the (row, direction) pairs; nom at most 1 %
    of the (row, direction, channel) entries."""
    for k in ("sign", "NoV"):
        assert n_gates.get(k, 0) <= grazing + max(1, n_rows // 100), (what, n_gates)
    for k in ("NoL", "NoH", "cos"):
        assert n_gates.get(k, 0) <= max(3, n_rows * nl // 100), (what, n_gates)
    assert n_gates.get("nom", 0) <= max(3, n_rows * nl * 3 // 100), (what, n_gates)


def check_shading(form, x, srgb, rgb, lin, grads, gd0, what, chunk=512):
    """Every output of one kernel run against shade_ref, chunked over rows.  Returns the gate counts, the number of
    shaded rows and the shaded rows per light."""
    d64 = {k: (v.to(DEV).double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in x.items()}
    mask = x["mask"].to(DEV)
    li = x["light"].to(DEV).long()
    m, nl, L = d64["normal"].shape[0], d64["dirs"].shape[0], d64["direct"].shape[0]
    # nothing keeps its sentinel; masked rows shade to 1 (lin 2) with exact zero gradients
    for k, t in list(grads.items())[:4] + [("rgb", rgb)] + ([("lin", lin)] if lin is not None else []):
        assert not bool((t == SENTINEL).any()), (what, k)
    if form == "hits":
        off = ~mask
        assert bool((rgb[off] == 1).all()) and bool((lin[off] == 2).all()), what
        for k in ("g_normal", "g_albedo", "g_rough", "g_fresnel"):
            assert bool((grads[k][off] == 0).all()), (what, k)
    rows = mask.nonzero().reshape(-1)
    gates = Gates()
    gd_want = gd0.double().clone()
    gd_err = torch.zeros_like(gd_want)
    gd_mag = gd0.double().abs()
    cnt = torch.zeros(L, device=DEV, dtype=torch.float64)
    V64 = d64["view"] if form == "list" else -d64["rays"][:, 3:6]
    for s in range(0, rows.numel(), chunk):
        idx = rows[s:s + chunk]
        r = d64["rough"][idx].expand(-1, 3)
        args = (d64["normal"][idx], V64[idx], d64["albedo"][idx], d64["fresnel"][idx], r, d64["dirs"],
                d64["weight"], d64["direct"][li[idx]], d64["vis"][idx], d64["ind"][idx])
        g_rgb = R(d64["g_rgb"][idx])
        if form == "hits":
            linb = lin[idx].double()
            rgb_want = tone(linb, srgb)
            check_fin(rgb[idx], rgb_want.v, rgb_want.e + 1e-300, f"{what}: rgb from lin")
            go = g_rgb * tone_grad(linb, srgb)
        else:
            go = g_rgb
        out = shade_ref_rows(args, go, gates)
        got_lin = lin[idx] if form == "hits" else rgb[idx]
        check_fin(got_lin, out["lin"].v, out["lin"].e + 1e-300, f"{what}: lin")
        for k in ("g_normal", "g_albedo", "g_fresnel"):
            check_fin(grads[k][idx], out[k].v, out[k].e + 1e-300, f"{what}: {k}")
        grough = out["g_rough"]
        if form == "hits":                                # backward of .repeat(1, 3): the channel sum
            grough = grough.sum(1, 2.0)[:, None]
        check_fin(grads["g_rough"][idx], grough.v, grough.e + 1e-300, f"{what}: g_rough")
        gdt = out["gd"]
        gd_want.index_add_(0, li[idx], gdt.v)
        gd_err.index_add_(0, li[idx], gdt.e)
        gd_mag.index_add_(0, li[idx], gdt.v.abs() + gdt.e)
        cnt.index_add_(0, li[idx], torch.ones(idx.numel(), device=DEV, dtype=torch.float64))
    bnd = gd_err + torch.stack([sum_bound(gd_mag[j], float(cnt[j]) + 1) for j in range(L)])
    check_fin(grads["g_direct"], gd_want, bnd + 1e-300, f"{what}: g_direct")
    # the gradient was added onto the buffer's contents, for every light
    hit = (gd_want - gd0.double()).abs().sum((1, 2)) > 0
    assert bool(((grads["g_direct"] - gd0).abs().sum((1, 2)) > 0)[hit].all()) and bool(hit.any()), what
    return gates.n, rows.numel(), cnt


def sm_rows():
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 8 + 5


# (form, rows, (H, W), equal-area weights, lights, srgb); rows None = 2 num_sms 8 + 5
CASES = [("list", 1, (16, 32), False, 1, 0), ("list", 37, (16, 32), False, 8, 0), ("list", 37, (6, 10), True, 3, 0),
         ("list", None, (16, 32), True, 9, 0), ("list", 4096, (8, 16), False, 3, 0),
         ("hits", 1, (8, 16), False, 1, 1), ("hits", 37, (6, 10), False, 3, 0), ("hits", 37, (16, 32), True, 33, 1),
         ("hits", None, (16, 32), False, 33, 1), ("hits", None, (6, 10), True, 8, 0),
         ("hits", 4096, (16, 32), False, 9, 1), ("hits", 4096, (8, 16), True, 3, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("form,m,hw,equal,L,srgb", CASES)
def test_shading_kernels_vs_fp64(form, m, hw, equal, L, srgb):
    from tensoir_b200 import _lib
    _lib.load()
    m = sm_rows() if m is None else m
    x = make_case(form, m, hw[0], hw[1], equal, L, seed=1000 * L + m + 7 * hw[0] + int(equal))
    what = f"{form} rows {m} dirs {hw} equal {equal} lights {L} srgb {srgb}"
    rgb, lin, grads, gd0 = run_kernels(form, x, srgb)
    if form == "hits":
        lv = lin[x["mask"].to(DEV)]
        if m >= 37:                                                # every tone region is reached
            assert bool((lv == 0).any()) and bool(((lv > 0) & (lv <= SRGB_T)).any()), what
            assert bool(((lv > SRGB_T) & (lv <= 1)).any()) and bool((lv > 1).any()), what
    n_gates, n_rows, per_light = check_shading(form, x, srgb, rgb, lin, grads, gd0, what)
    assert bool((per_light > 0).all()), (what, "a light id has no shaded row")
    assert_gates(n_gates, n_rows, x["dirs"].shape[0], x["grazing"], what)


@pytest.mark.gpu
def test_training_step_shading_vs_fp64(golden_rotated, monkeypatch):
    """The shading checks on the inputs of a real relight-phase step (the step of test_boundary_train_step_grads):
    the model's own normals, albedo, roughness and fresnel, its SG light table, vis and indirect from the secondary
    march, and the gradient the step's loss sends into rgb_with_brdf."""
    from gpu_helpers import model_from_fixture, renderer_args
    from tensoir_b200 import Renderer_TensoIR_train
    from tensoir_b200 import shade as S
    fx = golden_rotated
    m = model_from_fixture(fx, DEV)
    m.__dict__["_tir_randn_like"] = lambda t: torch.randn(t.shape).to(t.device)
    seen = {}
    shade_hits = S.shade_hits

    def capture(normal, albedo, rough1, fresnel, direct, rays, mask, light_idx, dirs, weight, vis, indirect,
                srgb=True):
        nl = dirs.shape[0]
        seen.update(normal=normal, albedo=albedo, rough=rough1, fresnel=fresnel, direct=direct, rays=rays,
                    mask=mask.bool(), light=light_idx.reshape(-1).to(torch.int32), dirs=dirs, weight=weight,
                    vis=vis.reshape(-1, nl), ind=indirect.reshape(-1, nl, 3))
        seen.update({k: v.detach().float().clone() for k, v in seen.items() if v.is_floating_point()})
        seen["srgb"] = int(bool(srgb))
        out = shade_hits(normal, albedo, rough1, fresnel, direct, rays, mask, light_idx, dirs, weight, vis, indirect,
                         srgb)
        out.register_hook(lambda g: seen.__setitem__("g_rgb", g.detach().float().clone()))
        return out
    monkeypatch.setattr(S, "shade_hits", capture)
    torch.manual_seed(fx["train_seed"])
    got = Renderer_TensoIR_train(fx["rays"], None, fx["light_idx"], m, N_samples=60, white_bg=True, is_train=True,
                                 is_relight=True, sample_method='stratified_sampling', chunk_size=160000,
                                 device=DEV, args=renderer_args(24))
    target = torch.full_like(got["rgb_map"], 0.5)
    loss = (((got["rgb_map"] - target) ** 2).mean() + 0.2 * ((got["rgb_with_brdf_map"] - target) ** 2).mean()
            + 0.0005 * got["normals_diff_map"].mean() + 0.001 * got["normals_orientation_loss_map"].mean()
            + 0.001 * got["albedo_smoothness_loss"] + 0.001 * got["roughness_smoothness_loss"])
    loss.backward()
    assert "g_rgb" in seen and int(seen["mask"].sum()) > 0
    srgb = seen.pop("srgb")
    x = dict(seen, view=None, grazing=0)
    rgb, lin, grads, gd0 = run_kernels("hits", x, srgb)
    assert torch.equal(rgb, got["rgb_with_brdf_map"].detach().reshape(rgb.shape))
    n_gates, n_rows, _ = check_shading("hits", x, srgb, rgb, lin, grads, gd0, "training step")
    assert_gates(n_gates, n_rows, x["dirs"].shape[0], 0, "training step")


@pytest.mark.gpu
def test_shared_memory_opt_in_in_a_fresh_process():
    """cudaFuncSetAttribute persists for the whole process: once any call has raised shade_bwd_kernel's dynamic
    shared-memory limit, a later table between 48 KB and that limit launches whether or not its own call opts in.  So
    a 9-light table at 512 directions (55 KB) is also run as the first shading backward of a new process."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_shade_kernels_fp64 as T; "
            "T.test_shading_kernels_vs_fp64('hits', 37, (16, 32), False, 9, 1)") % (here, os.path.dirname(here))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
