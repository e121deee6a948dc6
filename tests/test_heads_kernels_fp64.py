"""The appearance-head kernels stage by stage against float64: the split-BF16 forward with its activation dumps
(csrc/tir_mlp.cu) and the backward's heads_dgrad_kernel / heads_wgrad_kernel (csrc/tir_mlp_bwd.cu), driven through
tir_primary_radiance / tir_primary_radiance_backward and tir_primary_heads on appearance lists written by hand.

The valid list is left empty (offsets all zero), so compositing, the density gather and the density scatter do nothing
and every gradient comes from the head path.  The appearance list (a_offsets, a_ray, a_w, a_xn, a_src) is written
directly; its capacity is well above the real row count and every workspace row past that count holds a finite
sentinel, so a kernel that walks the capacity instead of the device-side count a_offsets[n_rays] reads it.

Every stage is compared with a float64 reference built from the kernel's OWN dumped input, so an error is pinned to the
stage that makes it: x0 from the gather; the MLP input from x0, the light row, basis_mat and the positional encoding; h1
from the input, h2 from h1, out from h2; g_out from the ray gradient; d z2, d z1, d feat and d x0; the weight, bias,
basis_mat and light_line gradients; the appearance-factor gradients from a float64 scatter of the kernel's own d x0.

Tolerances follow from the arithmetic, per entry, in float64:
  * a split-BF16 product (x = hi + lo, hi = bf16(x), lo = bf16(x - hi), so |x - hi - lo| <= 2^-16 |x|) summed as
    hi*hi + hi*lo + lo*hi misses at most 3 * 2^-16 |a||b| per term (the two representation errors and the dropped
    lo*lo); a contraction of length K adds the fp32 accumulation eps32 (16 + 4 sqrt(3K + n_add)) per |term| (three mma
    per k step, n_add atomics into the entry; an fp32 sum of n terms makes ~sqrt(n) roundings, as in
    test_vm_kernels_fp64.py);
  * the dumps store hi + lo of the fp32 value: 2^-16 + eps32 of the value.  A stage that reads a dump as its tile reads
    exactly the hi / lo the kernel multiplied, so the dump rounding enters only the stage that writes it;
  * ReLU is 1-Lipschitz, so a forward entry whose pre-activation is within its bound of 0 may take either branch and
    still stays within that bound; the backward masks come from the dumped h1 / h2, which the kernel reads as well;
  * fp32 CUDA-core steps (light scaling, the PE backward, sigmoid / tanh and their derivatives) add a few eps32 of the
    magnitudes they combine.
The reference functions themselves are pinned by ``test_stage_references_match_autograd_cpu``: chained, they equal
torch autograd of the same head as an nn.Sequential in float64.

The four-job backward, whose g_out comes from the tail kernels, is checked by test_primary_kernels_fp64.py with
Stages.data_grads and Stages.param_grads."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import tensoir_oracle as O

DEV = "cuda:0"
EPS32 = 2.0 ** -23
SPLIT = 3 * 2.0 ** -16            # one split-BF16 product
DUMP = 2.0 ** -16 + EPS32         # hi + lo of an fp32 value
K0, NF, IN, HID = 144, 27, 150, 128
P_W = 14                          # wgrad row slices per big weight gradient (tir_mlp_bwd.cu)


# ------------------------------------------------------------------------------------------------------------------
# float64 stage references
# ------------------------------------------------------------------------------------------------------------------
def light_row(mode, ll, light):
    """[n, 144] light factor of every row: 1, light_line[light] or the mean light_line row."""
    if mode == 0:
        return torch.ones(light.shape[0], K0, dtype=ll.dtype if ll is not None else torch.float64,
                          device=light.device)
    if mode == 1:
        return ll[light.long()]
    return ll.mean(0, keepdim=True).expand(light.shape[0], K0)


def pe(x):
    return O.positional_encoding(x, 2)


def head_input(x0, lrow, basis, vec):
    """[feat 27 | vec 3 | sin, cos PE(feat) | sin, cos PE(vec)]"""
    feat = (x0 * lrow) @ basis.t()
    return torch.cat([feat, vec, pe(feat), pe(vec)], 1)


def hidden(x, w, b):
    return torch.relu(x @ w.t() + b)


def head_out(h2, w2, b2, act):
    z = h2 @ w2.t() + b2
    return torch.sigmoid(z) if act == 0 else torch.tanh(z)


def act_grad(out, act):
    return out * (1 - out) if act == 0 else 1 - out * out


def g_z3(g_out, out, act):
    return g_out * act_grad(out, act)


def g_z2(gz3, w2, h2):
    return (gz3 @ w2) * (h2 > 0)


def g_z1(gz2, w1, h1):
    return (gz2 @ w1) * (h1 > 0)


def g_feat(gin, inp):
    """positional-encoding backward: d feat_f = d in_f + sum_p 2^p (d sin_fp cos_fp - d cos_fp sin_fp)"""
    s1, s2, c1, c2 = inp[:, 30:84:2], inp[:, 31:84:2], inp[:, 84:138:2], inp[:, 85:138:2]
    return (gin[:, :NF] + gin[:, 30:84:2] * c1 - gin[:, 84:138:2] * s1
            + 2 * (gin[:, 31:84:2] * c2 - gin[:, 85:138:2] * s2))


def g_feat_abs(gin, inp):
    """the same sum over |terms|"""
    gin, inp = gin.abs(), inp.abs()
    return (gin[:, :NF] + gin[:, 30:84:2] * inp[:, 84:138:2] + gin[:, 84:138:2] * inp[:, 30:84:2]
            + 2 * (gin[:, 31:84:2] * inp[:, 85:138:2] + gin[:, 85:138:2] * inp[:, 31:84:2]))


def g_products(gfeat, basis):
    """d (x0 * light row) = d feat @ basis_mat"""
    return gfeat @ basis


def g_light(a, x0, mode, light, n_lights):
    t = a * x0
    if mode == 1:
        return torch.zeros(n_lights, K0, dtype=t.dtype, device=t.device).index_add_(0, light.long(), t)
    return (t.sum(0, keepdim=True) / n_lights).expand(n_lights, K0)


def weight_grads(gz1, gz2, gz3, inp, h1, h2, gfeat, xl):
    return dict(w0=gz1.t() @ inp, b0=gz1.sum(0), w1=gz2.t() @ h1, b1=gz2.sum(0), w2=gz3.t() @ h2, b2=gz3.sum(0),
                basis=gfeat.t() @ xl)


# ------------------------------------------------------------------------------------------------------------------
# bounds
# ------------------------------------------------------------------------------------------------------------------
def gemm_bound(mag, k, n_add=1, split=True):
    """per-entry error of a contraction whose sum|a_k||b_k| is ``mag`` (see the module docstring)"""
    return mag * ((SPLIT if split else 0.0) + EPS32 * (16.0 + 4.0 * math.sqrt(3 * k + n_add)))


def sum_bound(mag, n):
    """an fp32 sum (threads, shuffles, atomics) of n terms whose sum|terms| is ``mag``"""
    return mag * EPS32 * (16.0 + 4.0 * math.sqrt(n))


def check(got, want, bnd, what):
    got, want = got.detach().double().reshape(want.shape), want.detach().double()
    assert bool(torch.isfinite(got).all()), what
    err = (got - want).abs()
    bnd = torch.as_tensor(bnd, dtype=torch.float64, device=want.device).expand(want.shape)
    ratio = err / bnd.clamp_min(1e-30)
    worst = int(ratio.reshape(-1).argmax())
    assert float(ratio.max()) <= 1.0, (what, float(ratio.max()), float(err.reshape(-1)[worst]),
                                       float(want.reshape(-1)[worst]), float(bnd.reshape(-1)[worst]))


# ------------------------------------------------------------------------------------------------------------------
# CPU: the references equal autograd
# ------------------------------------------------------------------------------------------------------------------
def _linear_init(fan_in, fan_out, g, dtype=torch.float32):
    """nn.Linear's initial scale: weight and bias uniform in +-1 / sqrt(fan_in)."""
    s = 1.0 / math.sqrt(fan_in)
    return ((torch.rand(fan_out, fan_in, generator=g) * 2 - 1) * s).to(dtype), \
        ((torch.rand(fan_out, generator=g) * 2 - 1) * s).to(dtype)


@pytest.mark.parametrize("mode,act", [(0, 0), (1, 0), (2, 1), (1, 1)])
def test_stage_references_match_autograd_cpu(mode, act):
    """The float64 stage functions, chained, equal torch autograd of an nn.Sequential head in float64 (forward,
    every parameter gradient, d x0, d basis_mat, d light_line)."""
    g = torch.Generator().manual_seed(11 + mode + 3 * act)
    n, L, od = 97, 5, 3 + act
    d = torch.float64
    x0 = torch.randn(n, K0, generator=g, dtype=d).requires_grad_(True)
    ll = torch.randn(L, K0, generator=g, dtype=d).requires_grad_(True)
    basis = (torch.randn(NF, K0, generator=g, dtype=d) / 12).requires_grad_(True)
    vec = F.normalize(torch.randn(n, 3, generator=g, dtype=d), dim=-1)
    light = torch.randint(0, L, (n,), generator=g)
    seq = torch.nn.Sequential(torch.nn.Linear(IN, HID), torch.nn.ReLU(), torch.nn.Linear(HID, HID), torch.nn.ReLU(),
                              torch.nn.Linear(HID, od)).to(d)
    with torch.no_grad():
        for i, (fi, fo) in zip((0, 2, 4), ((IN, HID), (HID, HID), (HID, od))):
            w, b = _linear_init(fi, fo, g, d)
            seq[i].weight.copy_(w)
            seq[i].bias.copy_(b)
    g_out = torch.randn(n, od, generator=g, dtype=d)
    lr = [torch.ones(n, K0, dtype=d), F.embedding(light, ll), ll.mean(0, keepdim=True).expand(n, K0)][mode]
    feat = F.linear(x0 * lr, basis)
    inp_t = torch.cat([feat, vec, O.positional_encoding(feat, 2), O.positional_encoding(vec, 2)], -1)
    out_t = seq(inp_t)
    out_t = torch.sigmoid(out_t) if act == 0 else torch.tanh(out_t)
    (out_t * g_out).sum().backward()

    W = [seq[i].weight.detach() for i in (0, 2, 4)]
    B = [seq[i].bias.detach() for i in (0, 2, 4)]
    x0d, lld, bd = x0.detach(), ll.detach(), basis.detach()
    lrow = light_row(mode, lld, light)
    inp = head_input(x0d, lrow, bd, vec)
    h1 = hidden(inp, W[0], B[0])
    h2 = hidden(h1, W[1], B[1])
    out = head_out(h2, W[2], B[2], act)
    gz3 = g_z3(g_out, out, act)
    gz2 = g_z2(gz3, W[2], h2)
    gz1 = g_z1(gz2, W[1], h1)
    gf = g_feat(gz1 @ W[0], inp)
    a = g_products(gf, bd)
    wg = weight_grads(gz1, gz2, gz3, inp, h1, h2, gf, x0d * lrow)

    def same(x, y, what):
        assert torch.allclose(x, y, rtol=1e-10, atol=1e-12), (what, float((x - y).abs().max()))
    same(inp, inp_t.detach(), "input")
    same(out, out_t.detach(), "out")
    same(a * lrow, x0.grad, "d x0")
    same(wg["basis"], basis.grad, "d basis_mat")
    for k, i in (("0", 0), ("1", 2), ("2", 4)):
        same(wg["w" + k], seq[i].weight.grad, "d W" + k)
        same(wg["b" + k], seq[i].bias.grad, "d b" + k)
    if mode:
        same(g_light(a, x0d, mode, light, L), ll.grad, "d light_line")
    else:
        assert ll.grad is None


# ------------------------------------------------------------------------------------------------------------------
# GPU: hand-written appearance lists
# ------------------------------------------------------------------------------------------------------------------
def ray_counts(n, g):
    """samples per ray: one ray with one sample, an empty ray, one with 300 (when n allows), the rest 1..40, and an
    empty last ray"""
    counts = [min(1, n), 0]
    left = n - counts[0]
    if left:
        counts.append(min(300, left))
        left -= counts[-1]
    while left:
        counts.append(min(left, int(torch.randint(1, 41, (1,), generator=g))))
        left -= counts[-1]
    counts.append(0)
    return torch.tensor(counts)


class Head:
    """Random weights of one head (nn.Linear's initial scale) and the TirMlp pointing at them."""

    def __init__(self, g, od, basis, ll, mode):
        from tensoir_b200 import _lib
        self.w, self.b = [], []
        for fi, fo in ((IN, HID), (HID, HID), (HID, od)):
            w, b = _linear_init(fi, fo, g)
            self.w.append(w.to(DEV))
            self.b.append(b.to(DEV))
        m = _lib.TirMlp()
        m.w0, m.w1, m.w2 = [t.data_ptr() for t in self.w]
        m.b0, m.b1, m.b2 = [t.data_ptr() for t in self.b]
        m.basis = basis.data_ptr()
        m.light_line = ll.data_ptr() if (mode and ll is not None) else None
        m.n_lights = ll.shape[0] if (mode and ll is not None) else 0
        m.feat_dim, m.hidden, m.out_dim, m.pe_feat, m.pe_x = NF, HID, od, 2, 2
        self.od, self.mlp = od, m

    def w64(self):
        return [t.double() for t in self.w], [t.double() for t in self.b]


def fill_sentinel(ws):
    """Every float row of the workspace holds 3.0 (finite, outside the field's box) until a kernel writes it."""
    for t in ws.t.values():
        if t.is_floating_point():
            t.fill_(3.0)
        else:
            t.zero_()


def build_list(ws, n, n_rays_counts, g):
    """Write the appearance list of ``n`` rows by hand; the valid list stays empty."""
    counts = n_rays_counts
    n_rays = counts.numel()
    t = ws.t
    t["offsets"].zero_()
    t["a_offsets"].copy_(torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)]).to(DEV))
    ray = torch.repeat_interleave(torch.arange(n_rays), counts)
    t["a_ray"][:n] = ray.to(DEV, torch.int32)
    t["a_src"][:n] = torch.arange(n, device=DEV)
    t["a_w"][:n] = (torch.rand(n, generator=g) * 0.9 + 0.1).to(DEV)
    t["a_xn"][:n] = (torch.rand(n, 3, generator=g) * 2 - 1).to(DEV)
    t["acc"].copy_(torch.rand(n_rays, generator=g).to(DEV))
    t["depth"].copy_(torch.rand(n_rays, generator=g).to(DEV) * 4)
    o = torch.randn(n_rays, 3, generator=g)
    d = F.normalize(torch.randn(n_rays, 3, generator=g), dim=-1)
    return torch.cat([o, d], 1).to(DEV).contiguous(), ray.to(DEV)


# ---- stage checks shared by the hand-written lists and the training step --------------------------------------------
class Stages:
    """Float64 references and bounds of one head on the kernel's dumps of ``n`` rows."""

    def __init__(self, n, mode, act, n_lights, W, B, basis, ll, light, vec, x0, inp, h1, h2, out):
        self.n, self.mode, self.act, self.L = n, mode, act, n_lights
        self.W, self.B, self.basis, self.ll, self.light = W, B, basis, ll, light
        self.vec = vec
        self.x0, self.inp, self.h1, self.h2, self.out = x0, inp, h1, h2, out
        self.lrow = light_row(mode, ll, light) if mode else torch.ones(n, K0, dtype=torch.float64, device=DEV)
        if mode == 2:
            self.lrow_abs = ll.abs().mean(0, keepdim=True).expand(n, K0)
            self.c_l = n_lights + 2.0             # fp32 mean of L rows, then the product
        else:
            self.lrow_abs = self.lrow.abs()
            self.c_l = 1.0

    def forward(self, what):
        W, B = self.W, self.B
        x0, inp, h1, h2 = self.x0, self.inp, self.h1, self.h2
        xl_mag = x0.abs() * self.lrow_abs
        # MLP input: features from the dumped products; the 3-vector and its encoding from the fp32 inputs
        feat = (x0 * self.lrow) @ self.basis.t()
        fb = (gemm_bound(xl_mag @ self.basis.abs().t(), K0) + EPS32 * self.c_l * (xl_mag @ self.basis.abs().t())
              + DUMP * feat.abs())
        check(inp[:, :NF], feat, fb, f"{what}: features")
        check(inp[:, NF:NF + 3], self.vec, DUMP * self.vec.abs() + 1e-30, f"{what}: 3-vector")
        featd = inp[:, :NF]
        # sincosf of the fp32 feature, which the dump holds to DUMP: the argument moves by p * DUMP |feat|
        pf = pe(featd)
        arg = torch.cat([featd.abs().repeat_interleave(2, 1) * torch.tensor([1.0, 2.0], device=DEV, dtype=torch.float64)
                         .repeat(NF)] * 2, 1)
        check(inp[:, 30:138], pf, DUMP * arg + DUMP + 4 * EPS32, f"{what}: PE(features)")
        check(inp[:, 138:150], pe(self.vec), 2 * DUMP * 2 + DUMP + 4 * EPS32, f"{what}: PE(3-vector)")
        # hidden layers from the dumped tiles
        for k, (a, h) in enumerate(((inp, h1), (h1, h2))):
            z = a @ W[k].t() + B[k]
            mag = a.abs() @ W[k].abs().t()
            bnd = gemm_bound(mag, a.shape[1]) + EPS32 * (z.abs() + B[k].abs()) + DUMP * torch.relu(z)
            check(h, torch.relu(z), bnd, f"{what}: h{k + 1}")
        z = h2 @ W[2].t() + B[2]
        ez = gemm_bound(h2.abs() @ W[2].abs().t(), HID) + EPS32 * (z.abs() + B[2].abs())
        y = head_out(h2, W[2], B[2], self.act)
        check(self.out, y, ez * (act_grad(y, self.act).abs() + ez) + 4 * EPS32 * y.abs() + 1e-30, f"{what}: out")

    def backward(self, what, g_outd, gz2, gz1, gfeat, gx0, grads, g_light_got=None, n_add_w=P_W):
        """grads: dict w0, b0, w1, b1, w2, b2, basis of the kernel (only this head's contributions)."""
        a = self.data_grads(what, g_outd, gz2, gz1, gfeat, gx0)
        want, bnds = self.param_grads(g_outd, gz2, gz1, gfeat, a, n_add_w)
        if self.mode:
            check(g_light_got, want["light"], bnds["light"] + 1e-30, f"{what}: d light_line")
        for k in ("w0", "b0", "w1", "b1", "w2", "b2", "basis"):
            check(grads[k], want[k], bnds[k] + 1e-30, f"{what}: d {k}")
        return a

    def data_grads(self, what, g_outd, gz2, gz1, gfeat, gx0):
        """d z2, d z1, d feat and d x0 of the kernel against float64 from its own upstream dumps -> d (x0 * light)"""
        act, W = self.act, self.W
        od = W[2].shape[0]
        inp, h1, h2, out = self.inp, self.h1, self.h2, self.out[:, :od]
        gz3 = g_z3(g_outd[:, :od], out, act)
        gz3_mag = g_outd[:, :od].abs() * act_grad(out, act).abs()
        check(gz2, g_z2(gz3, W[2], h2), 8 * EPS32 * (gz3_mag @ W[2].abs()) * (h2 > 0) + 1e-30, f"{what}: d z2")
        check(gz1, g_z1(gz2, W[1], h1), gemm_bound(gz2.abs() @ W[1].abs(), HID) * (h1 > 0) + 1e-30, f"{what}: d z1")
        gin = gz1 @ W[0]
        e_gin = gemm_bound(gz1.abs() @ W[0].abs(), HID)
        fb = g_feat_abs(e_gin, inp) + 8 * EPS32 * g_feat_abs(gin, inp)
        check(gfeat, g_feat(gin, inp), fb + 1e-30, f"{what}: d feat")
        a = g_products(gfeat, self.basis)
        a_mag = gfeat.abs() @ self.basis.abs()
        e_a = gemm_bound(a_mag, 32)
        check(gx0, a * self.lrow, e_a * self.lrow_abs + EPS32 * (self.c_l + 1) * a_mag * self.lrow_abs + 1e-30,
              f"{what}: d x0")
        return a

    def param_grads(self, g_outd, gz2, gz1, gfeat, a, n_add_w=P_W):
        """float64 weight, bias, basis_mat and (light modes 1, 2) light_line gradients of this head and their bounds:
        (want, bounds), two dicts, so the contributions of heads that share a parameter can be summed."""
        n, act, W = self.n, self.act, self.W
        od = W[2].shape[0]
        inp, h1, h2, x0, out = self.inp, self.h1, self.h2, self.x0, self.out[:, :od]
        gz3 = g_z3(g_outd[:, :od], out, act)
        gz3_mag = g_outd[:, :od].abs() * act_grad(out, act).abs()
        xl = x0 * self.lrow
        xl_mag = x0.abs() * self.lrow_abs
        want = weight_grads(gz1, gz2, gz3, inp, h1, h2, gfeat, xl)
        sl = lambda v: v.sum(0)                    # noqa: E731
        bnds = dict(w0=gemm_bound(gz1.abs().t() @ inp.abs(), n, n_add_w),
                    b0=sum_bound(sl(gz1.abs()), n + n_add_w),
                    w1=gemm_bound(gz2.abs().t() @ h1.abs(), n, n_add_w),
                    b1=sum_bound(sl(gz2.abs()), n + n_add_w),
                    w2=gemm_bound(gz3_mag.t() @ h2.abs(), n, n_add_w) + 4 * EPS32 * (gz3_mag.t() @ h2.abs()),
                    b2=sum_bound(sl(gz3_mag), n + n_add_w) + 4 * EPS32 * sl(gz3_mag),
                    basis=gemm_bound(gfeat.abs().t() @ xl_mag, n, n_add_w)
                    + EPS32 * self.c_l * (gfeat.abs().t() @ xl_mag))
        if self.mode:
            a_mag = gfeat.abs() @ self.basis.abs()
            e_a = gemm_bound(a_mag, 32)
            t_mag = a_mag * x0.abs()
            want["light"] = g_light(a, x0, self.mode, self.light, self.L)
            if self.mode == 1:
                cnt = torch.bincount(self.light.long(), minlength=self.L).double()[:, None]
                mag = torch.zeros(self.L, K0, dtype=torch.float64, device=DEV).index_add_(0, self.light.long(), t_mag)
                emag = torch.zeros_like(mag).index_add_(0, self.light.long(), e_a * x0.abs())
            else:
                cnt = torch.full((self.L, 1), float(n), dtype=torch.float64, device=DEV)
                mag = (t_mag.sum(0, keepdim=True) / self.L).expand(self.L, K0)
                emag = ((e_a * x0.abs()).sum(0, keepdim=True) / self.L).expand(self.L, K0)
            bnds["light"] = emag + mag * EPS32 * (18.0 + 4.0 * cnt.sqrt())
        return want, bnds


def check_factor_grads(planes, lines, grid, xn, gx0, gp, gl, what, prefill=0.0):
    """Appearance-factor gradients (channel-last, from the kernel) against a float64 scatter of the kernel's d x0.
    ``prefill``: the value every gradient entry held before the kernel accumulated into it; its modulus joins the
    magnitude of every entry, for the roundings of adding to it."""
    import test_vm_kernels_fp64 as V
    with V.f64():
        ps_ = [p.detach().double().clone().requires_grad_(True) for p in planes]
        ls_ = [p.detach().double().clone().requires_grad_(True) for p in lines]
        f = O.OracleField(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), grid_size=list(grid), density_plane=ps_,
                          density_line=ls_, app_plane=ps_, app_line=ls_, basis_w=None, mlp_rgb=None)
        ps, ls = O._app_products(f, xn)
        (ps * ls).t().backward(gx0)
        ts = V.tap_sums(ps_, ls_, xn, False, False, grid)
        tu = V.tap_sums(ps_, ls_, xn, False, True, grid)
        ga = gx0.abs().view(-1, 3, 48)
        m = V.scatter(ts, lambda k, t, j: ga[:, k] * t["ptaps"][j][1][:, None] * t["AL"],
                      lambda k, t, j: ga[:, k] * t["ltaps"][j][1][:, None] * t["AP"], 48)
        u = V.scatter(tu, lambda k, t, j: ga[:, k] * t["ptaps"][j][1][:, None] * t["AL"],
                      lambda k, t, j: ga[:, k] * t["ltaps"][j][1][:, None] * t["AP"], 48)
        m = [(mp + abs(prefill), ml + abs(prefill), cp, cl) for mp, ml, cp, cl in m]
        V.check_scatter([g - prefill for g in gp], [g - prefill for g in gl], [p.grad for p in ps_],
                        [p.grad for p in ls_], m, u, what, grid)


def check_gather(planes, lines, grid, xn, x0, what):
    """x0 (the raw products the forward dumps) against the float64 gather."""
    import test_vm_kernels_fp64 as V
    with V.f64():
        ps_ = [p.detach().double() for p in planes]
        ls_ = [p.detach().double() for p in lines]
        f = O.OracleField(aabb=torch.tensor([[-1.0] * 3, [1.0] * 3]), grid_size=list(grid), density_plane=ps_,
                          density_line=ls_, app_plane=ps_, app_line=ls_, basis_w=None, mlp_rgb=None)
        ps, ls = O._app_products(f, xn)
        ts = V.tap_sums(ps_, ls_, xn, False, False, grid)
        tu = V.tap_sums(ps_, ls_, xn, False, True, grid)
        mag = torch.cat([t["AP"] * t["AL"] for t in ts], 1)
        unit = torch.cat([t["AP"] * t["AL"] for t in tu], 1)
        V.check(x0, (ps * ls).t(), V.bound(mag, unit, grid=grid), what)


@pytest.fixture(scope="module")
def field():
    from tensoir_b200 import _lib
    import test_vm_kernels_fp64 as V
    _lib.load()
    return V.Field(0)


# (light_mode, lights, act, real rows): every light mode, light rows on both sides of the 8 kept in shared memory,
# both activations, partial tiles, lists shorter than the wgrad row slices (14 x 64) and one above them
RADIANCE_CASES = [(0, 0, 0, 1), (0, 0, 1, 63), (1, 1, 0, 64), (1, 3, 1, 65), (1, 8, 0, 1000), (1, 9, 1, 1000),
                  (1, 13, 0, 3 * P_W * 64 + 37), (1, 13, 1, 1), (2, 1, 0, 63), (2, 3, 1, 1000), (2, 9, 0, 65),
                  (2, 13, 1, 3 * P_W * 64 + 37)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,n_lights,act,n", RADIANCE_CASES)
def test_radiance_head_stages(field, mode, n_lights, act, n):
    from tensoir_b200 import _lib
    from tensoir_b200.primary_fused import Workspace
    import test_vm_kernels_fp64 as V
    lib = _lib.load()
    g = torch.Generator().manual_seed(1000 * mode + 100 * n_lights + 10 * act + n)
    counts = ray_counts(n, g)
    n_rays = counts.numel()
    ws = Workspace(DEV, point_sets=1)
    ws.ensure(n_rays, max(n, 1), n + 1500, 1, True)
    fill_sentinel(ws)
    rays, ray = build_list(ws, n, counts, g)
    ll = torch.randn(max(n_lights, 1), K0, generator=g).to(DEV)
    basis = (torch.randn(NF, K0, generator=g) / 12).to(DEV)
    head = Head(g, 3, basis, ll if mode else None, mode)
    li = torch.randint(0, max(n_lights, 1), (n_rays,), generator=g, dtype=torch.int32)
    li[0] = max(n_lights, 1) - 1                         # the last light row is used, past the 8 in shared memory
    li = li.to(DEV)
    job = _lib.TirHeadJob()
    job.mlp, job.point_set, job.x_in, job.light_mode, job.act, job.role = head.mlp, 0, 0, mode, act, 0
    bg = int(n % 2)
    rgb, depth = torch.empty(n_rays, 3, device=DEV), torch.empty(n_rays, device=DEV)
    w = ws.work_struct(None, 1, True)
    _lib.check(lib.tir_primary_radiance(C.byref(field.struct), C.byref(job), _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                        n_rays, C.byref(w), bg, _lib.dptr(rgb), _lib.dptr(depth), _lib.stream_ptr()),
               "tir_primary_radiance")
    g_rgb = torch.randn(n_rays, 3, generator=g).to(DEV)
    g_depth = torch.randn(n_rays, generator=g).to(DEV)
    b = ws.bwd_struct(1)
    gr = _lib.TirPrimaryGrads()
    gp, gl, ap, al = V.grad_shadows(field, "app")
    dgp, dgl, dp, dl = V.grad_shadows(field, "density")
    for k in range(3):
        gr.aplane[k], gr.aline[k], gr.dplane[k], gr.dline[k] = ap[k], al[k], dp[k], dl[k]
    gb = torch.zeros(NF, K0, device=DEV)
    gll = torch.zeros_like(ll)
    gr.basis = gb.data_ptr()
    gr.light_line = gll.data_ptr() if mode else None
    gw = [torch.zeros_like(t) for t in head.w]
    gbias = [torch.zeros_like(t) for t in head.b]
    gr.w0[0], gr.w1[0], gr.w2[0] = [t.data_ptr() for t in gw]
    gr.b0[0], gr.b1[0], gr.b2[0] = [t.data_ptr() for t in gbias]
    _lib.check(lib.tir_primary_radiance_backward(C.byref(field.struct), C.byref(job), _lib.dptr(rays),
                                                 _lib.dptr(li, torch.int32), n_rays, C.byref(w), C.byref(b), bg,
                                                 _lib.dptr(g_rgb), _lib.dptr(g_depth), None, C.byref(gr),
                                                 _lib.stream_ptr()), "tir_primary_radiance_backward")
    torch.cuda.synchronize()
    t = {k: v[:n].double() for k, v in ws.t.items() if v.shape[0] == ws.cap_app and v.is_floating_point()}
    what = f"mode {mode} L {n_lights} act {act} n {n}"
    # nothing past the device-side count was written, and nothing reached the density factors
    for k in ("out0", "inp0", "h1_0", "h2_0", "x0_0", "g_out0", "gz1_0", "gz2_0", "gfeat0", "gx0_0"):
        assert bool((ws.t[k][n:] == 3.0).all()), (what, k)
    assert all(float(x.abs().max()) == 0.0 for x in dgp + dgl), what
    # forward stages
    xn = t["a_xn"]
    check_gather([p.to(DEV) for p in field.aplane], [p.to(DEV) for p in field.aline], V.GRID, xn, t["x0_0"],
                 f"{what}: x0")
    W, B = head.w64()
    st = Stages(n, mode, act, max(n_lights, 1), W, B, basis.double(), ll.double(), li[ray], rays[ray, 3:6].double(),
                t["x0_0"], t["inp0"], t["h1_0"], t["h2_0"], t["out0"][:, :3])
    st.forward(what)
    # the ray gradient reaches every row as a_w * d rgb; column 3 of the padded output carries none
    aw = t["a_w"][:, None]
    want_gout = aw * g_rgb.double()[ray]
    check(t["g_out0"][:, :3], want_gout, EPS32 * want_gout.abs() + 1e-30, f"{what}: g_out")
    assert bool((ws.t["g_out0"][:n, 3] == 0).all()), what
    grads = dict(w0=gw[0], b0=gbias[0], w1=gw[1], b1=gbias[1], w2=gw[2], b2=gbias[2], basis=gb)
    st.backward(what, t["g_out0"], t["gz2_0"], t["gz1_0"], t["gfeat0"][:, :NF], t["gx0_0"], grads,
                gll if mode else None)
    if not mode:
        assert float(gll.abs().max()) == 0.0
    # the appearance factors from a float64 scatter of the kernel's own d x0
    check_factor_grads([p.to(DEV) for p in field.aplane], [p.to(DEV) for p in field.aline], V.GRID, xn, t["gx0_0"],
                       gp, gl, f"{what}: factor gradients")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [65, 2 * P_W * 64 + 5])
def test_four_head_forward_stages(field, n):
    """tir_primary_heads with four jobs (both point sets, an indexed and a mean light, sigmoid and tanh, out_dim 3
    and 4) and TIR_NORMALS_PREDICTED: each job's x0, input, h1, h2 and output against its float64 stage reference.
    The tail and the maps are not checked here."""
    from tensoir_b200 import _lib
    from tensoir_b200.primary_fused import Workspace
    import test_vm_kernels_fp64 as V
    lib = _lib.load()
    g = torch.Generator().manual_seed(77 + n)
    counts = ray_counts(n, g)
    n_rays = counts.numel()
    ws = Workspace(DEV, point_sets=2)
    ws.ensure(n_rays, n, n + 700, 4, True)
    fill_sentinel(ws)
    rays, ray = build_list(ws, n, counts, g)
    L = 3
    ll = torch.randn(L, K0, generator=g).to(DEV)
    basis = (torch.randn(NF, K0, generator=g) / 12).to(DEV)
    li = torch.randint(0, L, (n_rays,), generator=g, dtype=torch.int32).to(DEV)
    rgb_h = Head(g, 3, basis, ll, 1)
    brdf_h = Head(g, 4, basis, ll, 2)
    norm_h = Head(g, 3, basis, ll, 2)
    # (head, role, point set, x_in, light mode, act)
    spec = [(rgb_h, 0, 0, 0, 1, 0), (brdf_h, 1, 0, 1, 2, 0), (brdf_h, 2, 1, 1, 2, 0), (norm_h, 3, 0, 1, 2, 1)]
    jobs = (_lib.TirHeadJob * 4)()
    for j, (h, role, ps, x_in, lm, act) in enumerate(spec):
        jobs[j].mlp, jobs[j].point_set, jobs[j].x_in, jobs[j].light_mode, jobs[j].act, jobs[j].role = \
            h.mlp, ps, x_in, lm, act, role
    noise = torch.zeros(ws.cap_app, 3, device=DEV)
    noise[:n] = torch.randn(n, 3, generator=g).to(DEV)
    w = ws.work_struct(noise, 4, True)
    maps = _lib.TirRayMaps()
    keep = []
    for k, c in zip(("rgb", "depth", "normal", "albedo", "rough", "fresnel", "nd", "no"), (3, 1, 3, 3, 1, 3, 1, 1)):
        keep.append(torch.empty(n_rays, c, device=DEV))
        setattr(maps, k, keep[-1].data_ptr())
    mask = torch.empty(n_rays, dtype=torch.bool, device=DEV)
    losses = torch.empty(2, device=DEV)
    _lib.check(lib.tir_primary_heads(C.byref(field.struct), jobs, 4, 1, _lib.dptr(rays), _lib.dptr(li, torch.int32),
                                     n_rays, C.byref(w), 0.04, 1, C.byref(maps), _lib.dptr(mask, torch.bool),
                                     _lib.dptr(losses), None, _lib.stream_ptr()), "tir_primary_heads")
    torch.cuda.synchronize()
    t = {k: v[:n].double() for k, v in ws.t.items() if v.shape[0] == ws.cap_app and v.is_floating_point()}
    pts = [t["a_xn"], t["a_xj"]]
    check(pts[1], pts[0] + noise[:n].double() * 0.01, 2 * EPS32 * (pts[0].abs() + 0.01 * noise[:n].double().abs()),
          "jittered points")
    planes, lines = [p.to(DEV) for p in field.aplane], [p.to(DEV) for p in field.aline]
    for ps in (0, 1):
        check_gather(planes, lines, V.GRID, pts[ps], t[f"x0_{ps}"], f"n {n}: x0 of point set {ps}")
    for j, (h, role, ps, x_in, lm, act) in enumerate(spec):
        assert bool((ws.t[f"out{j}"][n:] == 3.0).all()), j
        W, B = h.w64()
        vec = rays[ray, 3:6].double() if x_in == 0 else pts[ps]
        out = t[f"out{j}"][:, :h.od]
        st = Stages(n, lm, act, L, W, B, basis.double(), ll.double(), li[ray], vec, t[f"x0_{ps}"], t[f"inp{j}"],
                    t[f"h1_{j}"], t[f"h2_{j}"], out)
        st.forward(f"n {n}: job {j}")


@pytest.mark.gpu
def test_shrunk_state_a_training_step_stages():
    """The stage checks on the radiance-only training step of shrunk state A (the step of
    test_radiance_primary_gpu.py), on the dumps the step left in the model's workspace: the gather, every head stage,
    and the renderModule, basis_mat, light_line and appearance-factor gradients the step produced."""
    from gpu_helpers import load_shrunk_state, model_from_fixture
    from test_radiance_primary_gpu import _fused_step, _loss
    fx = load_shrunk_state("A")
    m = model_from_fixture(fx, DEV, with_mask=True)
    rays, li_all = fx["rays"].to(DEV), fx["light_idx"].to(DEV)
    out, _ = _fused_step(m, rays, li_all, seed=31)
    torch.cuda.synchronize()
    ws = m.__dict__["_tir_radiance_ws"]
    n = int(ws.t["a_offsets"][-1])
    assert n > 0
    t = {k: v[:n].double() for k, v in ws.t.items() if v.shape[0] == ws.cap_app and v.is_floating_point()}
    ray = ws.t["a_ray"][:n].long()
    grid = [int(x) for x in m.gridSize]
    planes = [p.detach() for p in m.app_plane]
    lines = [p.detach() for p in m.app_line]
    check_gather(planes, lines, grid, t["a_xn"], t["x0_0"], "state A: x0")
    mlp = m.renderModule.mlp
    W = [mlp[i].weight.detach().double() for i in (0, 2, 4)]
    B = [mlp[i].bias.detach().double() for i in (0, 2, 4)]
    ll = m.light_line.weight.detach().double()
    li = li_all.reshape(-1)[ray]
    st = Stages(n, 1, 0, ll.shape[0], W, B, m.basis_mat.weight.detach().double(), ll, li, rays[ray, 3:6].double(),
                t["x0_0"], t["inp0"], t["h1_0"], t["h2_0"], t["out0"][:, :3])
    st.forward("state A")
    # the ray gradient of the step's loss
    rgb = out[0].detach().requires_grad_(True)
    (g_rgb,) = torch.autograd.grad(_loss(rgb, out[1].detach(), out[6].detach()), rgb)
    want_gout = t["a_w"][:, None] * g_rgb.double()[ray]
    check(t["g_out0"][:, :3], want_gout, EPS32 * want_gout.abs() + 1e-30, "state A: g_out")
    grads = dict(w0=mlp[0].weight.grad, b0=mlp[0].bias.grad, w1=mlp[2].weight.grad, b1=mlp[2].bias.grad,
                 w2=mlp[4].weight.grad, b2=mlp[4].bias.grad, basis=m.basis_mat.weight.grad)
    st.backward("state A", t["g_out0"], t["gz2_0"], t["gz1_0"], t["gfeat0"][:, :NF], t["gx0_0"], grads,
                m.light_line.weight.grad)
    gp = [p.grad[0].permute(1, 2, 0) for p in m.app_plane]
    gl = [p.grad[0].permute(1, 2, 0) for p in m.app_line]
    check_factor_grads(planes, lines, grid, t["a_xn"], t["gx0_0"], gp, gl, "state A: factor gradients")
