"""The kernels that write the parameters against float64: the optimiser step (csrc/tir_adam.cu through
``optim.FusedAdam``: Adam, the density L1 term and the gradient clearing) and the TV regulariser (csrc/tir_tv.cu through
``tv.tv_planes``: value and gradient), at the sizes and layouts of a training step.

Adam.  The reference starts from the kernel's own fp32 inputs, saved just before each step (parameter, gradient, both
moments, the step count, the learning rate as the fp32 value the kernel reads), and restates the kernel's expression in
float64 with its fp32 constants: ``1.f - beta1`` and ``1.f - beta2`` (exact, by Sterbenz), the bias corrections
``1 - powf(beta1, t)`` and ``sqrtf(1 - powf(beta2, t))`` at the fp32 step count t, and the L1 term ``l1 * sign(p)`` with
sign(+-0) = 0.  Every intermediate x carries a bound e on |x32 - x|.  With u = eps32 = 2^-23 (twice the unit roundoff):
  * a + b:  e_a + e_b + u (|a + b| + e_a + e_b)
  * a * b:  |a| e_b + |b| e_a + e_a e_b + u (|ab| + that)
  * a / b:  (e_a + |a / b| e_b) / (|b| - e_b) + u (...)        (the bound must stay finite: e_b < |b|)
  * sqrtf:  min(e / sqrt(x), sqrt(e)) + u (...)                 (correctly rounded without --use_fast_math)
  * powf:   4 ulp (CUDA Math API), i.e. 4 u x^t plus 4 subnormal ulps 2^-149 once x^t leaves the normal range
These bounds hold per entry whatever order the compiler evaluates in: an FMA contraction rounds once where they round
twice.  After every step p, exp_avg and exp_avg_sq are within their bounds, every parameter's step count is exact
(torch.optim.Adam's per-parameter count: advanced only when the parameter has a gradient and the step is not skipped),
the gradients are bit-zero with clear_grad and bit-identical without it, and a step with ``found_inf`` set leaves the
parameters, moments and counts bit-identical.

Cases: the real parameter list of the 300^3 benchmark model with the bench's groups, device learning rates and density
L1 (eager, then one step captured in a CUDA graph and replayed with new learning rates copied in between, as the
trainer does); the same model with the gradients as views of one ``dp.GradBucket``, where gradients after the
renderModule's 3-float bias are not 16-byte aligned, so whole tensors take the kernel's scalar path; a synthetic table of
~40 tensors with numel 0, 1, 3, 4, 4095, 4096, 4097 and 3 * 4096 + 1, a parameter at storage offset 1 (p misaligned, the
moments aligned) and entries at exactly +0, -0 and +-1e-30 under an L1 weight; the skip flag; a state loaded at step
29 999.  Against torch.optim.Adam (fp32, 2e-6 as test_gpu_parity.py): a parameter whose gradient is None for the first 5
steps, and state_dicts moved from torch to FusedAdam and back.

TV.  tir_tv_loss sums fmaf(d, d, .) over a grid-stride loop per thread (V terms per unit, V = 4 on the float4 path, 1
on the scalar one), scales by the fp32 scale_h / scale_w, reduces 8 tree levels per CTA (5 shuffle + 3) and adds every
CTA's sum into one float with atomics.  All terms are non-negative, so sum |terms| = value and the error is at most
u (n_serial + 8 + n_atomics + 4) value: n_serial = V * the passes of the grid-stride loop, n_atomics = CTAs per plane *
planes, and 4 for d^2, the fp32 scale, its product and the sh + sw sum.  The reference is float64 ``TVLoss`` itself, with
the grid size taken from the device's SM count.  tir_tv_loss_bwd adds at most 4 stencil terms kh (x[h] - x[h-1]) etc. to
the ``.grad`` in place: each term rounds at most 4 times (d, the scale, kh = 2 gout scale, the product) and the chain of
at most 4 additions rounds relative to sum |terms| + |grad|, so every entry is within 8 u (sum |terms| + |grad|) of
float64 autograd of TVLoss plus the initial grad, a factor 2 to spare.  The grads start nonzero, so in-place
accumulation is checked.  Cases: the benchmark model's own planes (3 x [1,16,300,300] and 3 x [1,48,300,300],
channel-last, several grid-stride passes); NCHW planes whose channels sit 1000 apart, so a stencil coupling one channel's
last row to the next channel's first would dominate; channel-last planes with C % 4 != 0 and misaligned views into one
flat buffer (scalar path); 2 x 2 planes in the same call as 300 x 300 ones."""
import copy
import math

import numpy as np
import pytest
import torch

DEV = "cuda:0"
EPS = 2.0 ** -23
ULP_POW = 4.0                                    # CUDA Math API maximum ulp error of powf
SUBNORMAL = 2.0 ** -149
TV_THREADS = 256                                 # kThreads of csrc/tir_tv.cu
TV_CTAS_PER_SM = 8


def f32(x):
    return float(np.float32(float(x)))


def bits(t):
    return t.detach().view(torch.int32)


def check(got, want, bnd, what):
    got, want = got.detach().double(), want.detach().double()
    bnd = torch.as_tensor(bnd, dtype=torch.float64, device=want.device).expand(want.shape)
    assert bool(torch.isfinite(bnd).all()), (what, "vacuous bound")
    assert bool(torch.isfinite(got).all()), what
    err = (got - want).abs()
    bad = err > bnd
    if bool(bad.any()):
        k = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError((what, int(bad.sum()), "of", want.numel(), float(got.reshape(-1)[k]),
                              float(want.reshape(-1)[k]), float(bnd.reshape(-1)[k])))


# ------------------------------------------------------------------------------------------------------------------
# error propagation (module docstring): python floats or float64 tensors
# ------------------------------------------------------------------------------------------------------------------
def _abs(x):
    return x.abs() if torch.is_tensor(x) else abs(x)


def _add(s, e):
    return e + EPS * (_abs(s) + e)


def _mul(a, ea, b, eb):
    e = _abs(a) * eb + _abs(b) * ea + ea * eb
    return a * b, e + EPS * (_abs(a * b) + e)


def _div(a, ea, b, eb):
    q = a / b
    e = (ea + _abs(q) * eb) / (_abs(b) - eb)
    return q, e + EPS * (_abs(q) + e)


def _sqrt(x, e):
    if torch.is_tensor(x):
        r = x.sqrt()
        d = torch.minimum(torch.where(x > 0, e / r, torch.full_like(x, math.inf)), e.sqrt())
    else:
        r = math.sqrt(x)
        d = min(e / r if x > 0 else math.inf, math.sqrt(e))
    return r, d + EPS * (r + d)


def _pow(b, t):
    w = b ** t
    return w, ULP_POW * (EPS * w + SUBNORMAL)


def adam_reference(p, g, m, v, t, lr, l1, beta1, beta2, eps):
    """One step of tir_adam.cu in float64 from the kernel's fp32 inputs at step count t (after the increment).
    -> ((p, e_p), (m, e_m), (v, e_v))"""
    p, g, m, v = (x.double() for x in (p, g, m, v))
    c1, c2 = 1.0 - beta1, 1.0 - beta2                    # 1.f - beta (exact in fp32)
    w1, e_w1 = _pow(beta1, t)
    bc1 = 1.0 - w1
    e_bc1 = _add(bc1, e_w1)
    w2, e_w2 = _pow(beta2, t)
    q2 = 1.0 - w2
    bc2, e_bc2 = _sqrt(q2, _add(q2, e_w2))
    ss, e_ss = _div(lr, 0.0, bc1, e_bc1)
    if l1 != 0.0:
        ge = g + l1 * torch.sign(p)                      # sign(+-0) = 0, like (p > 0) - (p < 0)
        e_ge = EPS * ge.abs()
    else:
        ge, e_ge = g, torch.zeros_like(g)
    d = ge - m
    e_d = _add(d, e_ge)
    cd, e_cd = _mul(c1, 0.0, d, e_d)
    m1 = m + cd
    e_m1 = _add(m1, e_cd)
    bv = beta2 * v
    e_bv = EPS * bv.abs()
    cg, e_cg = _mul(c2, 0.0, ge, e_ge)                   # (1.f - beta2) * ge * ge, left to right
    sq, e_sq = _mul(cg, e_cg, ge, e_ge)
    v1 = bv + sq
    e_v1 = _add(v1, e_bv + e_sq)
    sv, e_sv = _sqrt(v1, e_v1)
    q, e_q = _div(sv, e_sv, bc2, e_bc2)
    den = q + eps
    e_den = _add(den, e_q)
    r, e_r = _div(m1, e_m1, den, e_den)
    st, e_st = _mul(ss, e_ss, r, e_r)
    p1 = p - st
    e_p1 = _add(p1, e_st)
    return (p1, e_p1), (m1, e_m1), (v1, e_v1)


def emulate_kernel(p, g, m, v, t, lr, l1, beta1, beta2, eps, sign=np.sign):
    """tir_adam.cu's update in numpy float32, one rounding per operation."""
    f = np.float32
    one, beta1, beta2 = f(1), f(beta1), f(beta2)
    bc1 = one - np.power(beta1, f(t))
    bc2s = np.sqrt(one - np.power(beta2, f(t)))
    ss = f(lr) / bc1
    ge = g + f(l1) * sign(p).astype(np.float32)
    m1 = m + (one - beta1) * (ge - m)
    v1 = beta2 * v + (one - beta2) * ge * ge
    return p - ss * (m1 / (np.sqrt(v1) / bc2s + f(eps))), m1, v1


def test_adam_reference_bounds_cpu():
    """The bounds of adam_reference hold for an fp32 evaluation of the kernel's expression and fail for the two bugs
    they are there to catch: a step count off by one and sign(-0) = -1 under the L1 term."""
    rng = np.random.default_rng(0)
    n = 20000
    p = rng.standard_normal(n).astype(np.float32)
    p[:4] = [0.0, -0.0, 1e-30, -1e-30]
    g = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    g[:2] = 0.0
    m = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    v = (rng.random(n) * 1e-6).astype(np.float32)
    m[:2] = v[:2] = 0.0
    args = (0.02, 3e-3, f32(0.9), f32(0.99), f32(1e-8))
    T = [torch.from_numpy(x) for x in (p, g, m, v)]

    def ok(t_kernel, t_ref, sign=np.sign):
        got = emulate_kernel(p, g, m, v, t_kernel, *args, sign=sign)
        ref = adam_reference(*T, t_ref, *args)
        return all(bool(((torch.from_numpy(x).double() - r).abs() <= e).all()) for x, (r, e) in zip(got, ref))
    for t in (1.0, 2.0, 10.0, 30000.0):
        assert ok(t, t), t
    assert not ok(1.0, 2.0) and not ok(2.0, 3.0)
    assert not ok(5.0, 5.0, sign=lambda x: np.where(x > 0, 1.0, -1.0))


# ------------------------------------------------------------------------------------------------------------------
# one FusedAdam step against the reference
# ------------------------------------------------------------------------------------------------------------------
def snapshot(opt):
    """The kernel's fp32 inputs of the next step, per parameter with a gradient."""
    b1, b2 = opt.param_groups[0]["betas"]
    snap = dict(beta1=f32(b1), beta2=f32(b2), eps=f32(opt.param_groups[0]["eps"]), rows=[])
    for grp in opt.param_groups:
        for p in grp["params"]:
            if p.grad is None:
                continue
            st = opt.state[p]
            snap["rows"].append(dict(
                p=p, p0=p.detach().clone(memory_format=torch.preserve_format),
                g0=p.grad.detach().clone(memory_format=torch.preserve_format),
                m0=st["exp_avg"].clone() if st else torch.zeros_like(p.detach()),
                v0=st["exp_avg_sq"].clone() if st else torch.zeros_like(p.detach()),
                t0=float(st["step"]) if st else 0.0,
                lr=f32(grp["lr"]), l1=f32(opt.l1.get(id(p), 0.0))))
    return snap


def check_step(opt, snap, what, skipped=False, clear_grad=True):
    """p, exp_avg and exp_avg_sq within their bounds (bit-identical when skipped), exact step counts, gradients
    bit-zero (clear_grad) or untouched."""
    for k, r in enumerate(snap["rows"]):
        p, st = r["p"], opt.state[r["p"]]
        tag = (what, k, tuple(p.shape))
        assert torch.is_tensor(st["step"]) and st["step"].is_cuda and st["step"].dtype == torch.float32, tag
        want_t = r["t0"] + (0.0 if skipped else 1.0)
        assert float(st["step"]) == want_t, (tag, float(st["step"]), want_t)
        if clear_grad:
            assert bool((bits(p.grad) == 0).all()), (tag, "gradient not cleared to +0")
        else:
            assert torch.equal(bits(p.grad), bits(r["g0"])), (tag, "gradient changed")
        if skipped:
            assert torch.equal(bits(p), bits(r["p0"])), (tag, "parameter changed by a skipped step")
            assert torch.equal(bits(st["exp_avg"]), bits(r["m0"])), (tag, "exp_avg changed by a skipped step")
            assert torch.equal(bits(st["exp_avg_sq"]), bits(r["v0"])), (tag, "exp_avg_sq changed by a skipped step")
            continue
        if p.numel() == 0:
            continue
        (p1, ep), (m1, em), (v1, ev) = adam_reference(r["p0"], r["g0"], r["m0"], r["v0"], want_t, r["lr"], r["l1"],
                                                      snap["beta1"], snap["beta2"], snap["eps"])
        check(st["exp_avg"], m1, em, tag + ("exp_avg",))
        check(st["exp_avg_sq"], v1, ev, tag + ("exp_avg_sq",))
        check(p, p1, ep, tag + ("param",))


def checked_step(opt, what, **kw):
    snap = snapshot(opt)
    opt.step()
    check_step(opt, snap, what, clear_grad=opt.clear_grad, **kw)


# ------------------------------------------------------------------------------------------------------------------
# the benchmark model
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lego300():
    from tensoir_b200.synthetic import make_lego_model
    return make_lego_model(300, DEV)


def bench_optimizer(model):
    """bench.py's FusedAdam: the model's groups with device learning rates and the density L1 term."""
    from bench import L1_WEIGHT
    from tensoir_b200.optim import FusedAdam
    from tensoir_b200.static_step import lr_tensors
    groups = lr_tensors(model.get_optparam_groups(0.02, 0.001), DEV)
    opt = FusedAdam(groups, betas=(0.9, 0.99))
    opt.density_l1(model, L1_WEIGHT)
    return opt


def model_params(opt):
    return [p for grp in opt.param_groups for p in grp["params"]]


def fill_grads(params, gen, scale=1e-3):
    for p in params:
        new = torch.randn(p.shape, generator=gen, device=DEV) * scale
        if p.grad is None:
            p.grad = new.contiguous(memory_format=torch.channels_last) if p.dim() == 4 and not p.is_contiguous() else new
        else:
            p.grad.copy_(new)


@pytest.mark.gpu
def test_adam_bench_model_eager_and_graph_replays(lego300):
    opt = bench_optimizer(lego300)
    params = model_params(opt)
    n = sum(p.numel() for p in params)
    assert n > 15_000_000 and len(params) > 20, (n, len(params))
    assert any(l1 != 0.0 for l1 in opt.l1.values())
    gen = torch.Generator(device=DEV).manual_seed(1)
    for it in range(3):
        fill_grads(params, gen)
        checked_step(opt, f"eager step {it}")
    # one step captured, replayed with new gradients and new learning rates copied in from pinned host memory
    fill_grads(params, gen)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    torch.cuda.synchronize()
    for it in range(3):
        host = torch.tensor([0.02 * 0.97 ** (it + 1) if k < 4 else 1e-3 * 0.9 ** (it + 1)
                             for k in range(len(opt.param_groups))], dtype=torch.float32).pin_memory()
        for k, grp in enumerate(opt.param_groups):
            grp["lr"].copy_(host[k], non_blocking=True)
        fill_grads(params, gen)
        snap = snapshot(opt)
        assert [r["lr"] for r in snap["rows"]][0] == f32(host[0])
        graph.replay()
        check_step(opt, snap, f"graph replay {it}")
    del graph


@pytest.mark.gpu
def test_adam_bench_model_grad_bucket_layout(lego300):
    from tensoir_b200.dp import GradBucket
    opt = bench_optimizer(lego300)
    params = model_params(opt)
    for p in params:
        p.grad = None
    bucket = GradBucket(params)
    gen = torch.Generator(device=DEV).manual_seed(2)
    for p, v in zip(bucket.params, bucket.views):
        v.copy_(torch.randn(p.shape, generator=gen, device=DEV) * 1e-3)
        p.grad = v
    big_misaligned = [tuple(p.shape) for p in params if p.numel() > 4096 and p.grad.data_ptr() % 16]
    assert big_misaligned, "no large gradient off 16-byte alignment: the whole-tensor scalar path is not reached"
    for it in range(3):
        if it:
            for p, v in zip(bucket.params, bucket.views):
                v.copy_(torch.randn(p.shape, generator=gen, device=DEV) * 1e-3)
        checked_step(opt, f"bucket step {it}")
    for p in params:
        p.grad = None


# ------------------------------------------------------------------------------------------------------------------
# synthetic table
# ------------------------------------------------------------------------------------------------------------------
SIZES = (0, 1, 3, 4, 4095, 4096, 4097, 3 * 4096 + 1)


def synthetic_params(gen):
    """~40 tensors of the edge sizes (1-D and channel-last 4-D), one at storage offset 1, with exact +0, -0 and +-1e-30
    entries."""
    ps = []
    for rep in range(5):
        for n in SIZES:
            if rep == 1 and n == 4097:
                ps.append(torch.nn.Parameter(torch.randn(4097 + 1, generator=gen, device=DEV)[1:]))
            elif rep == 2 and n == 4096:
                ps.append(torch.nn.Parameter(torch.randn(1, 16, 16, 16, generator=gen, device=DEV)
                                             .contiguous(memory_format=torch.channels_last)))
            else:
                ps.append(torch.nn.Parameter(torch.randn(n, generator=gen, device=DEV)))
    specials = torch.tensor([0.0, -0.0, 1e-30, -1e-30], device=DEV)
    for p in ps:
        if p.numel() >= 8:
            in_memory_order(p.data)[:4] = specials
    assert ps[SIZES.index(4097) + len(SIZES)].data_ptr() % 16 == 4
    return ps


def in_memory_order(t):
    return t.permute(0, 2, 3, 1).view(-1) if t.dim() == 4 else t.view(-1)


def synthetic_grads(ps, gen):
    for p in ps:
        g = torch.randn(p.shape, generator=gen, device=DEV)
        if p.dim() == 4:
            g = g.contiguous(memory_format=torch.channels_last)
        if p.numel() >= 8:
            in_memory_order(g)[:4] = 0.0             # so +-0 stay 0 and meet sign(+-0) = 0 at every step
        if p.grad is None:
            p.grad = g
        else:
            p.grad.copy_(g)


def synthetic_optimizer(ps, clear_grad=True):
    from tensoir_b200.optim import FusedAdam
    k = len(ps) // 3
    lr_dev = torch.tensor(5e-3, device=DEV)
    groups = [{"params": ps[:k], "lr": 0.02}, {"params": ps[k:2 * k], "lr": lr_dev}, {"params": ps[2 * k:], "lr": 1e-3}]
    l1 = {p: 3e-3 * (1 + i % 3) for i, p in enumerate(ps) if i % 2 == 0}
    return FusedAdam(groups, betas=(0.9, 0.99), l1=l1, clear_grad=clear_grad)


@pytest.mark.gpu
@pytest.mark.parametrize("clear_grad", [True, False])
def test_adam_synthetic_table(clear_grad):
    gen = torch.Generator(device=DEV).manual_seed(3)
    ps = synthetic_params(gen)
    assert len(ps) == 40
    opt = synthetic_optimizer(ps, clear_grad)
    flag = torch.zeros((), device=DEV)
    opt.found_inf = flag
    for it in range(5):
        synthetic_grads(ps, gen)
        if it == 2:                                  # skipped: only the gradients are cleared
            flag.fill_(1.0)
            checked_step(opt, "found_inf", skipped=True)
            flag.zero_()
            synthetic_grads(ps, gen)
        checked_step(opt, f"synthetic step {it}")
    for p in ps:
        if p.numel() >= 8:
            first = in_memory_order(p.detach())[:2]
            assert bits(first).tolist() == [0, -2 ** 31], "+0 / -0 entries moved under the L1 term"


@pytest.mark.gpu
def test_adam_end_of_training_state():
    """A state loaded at step 29 999: bias corrections at 1 (powf underflows), moments of a long run, loaded in the
    default contiguous layout also for the channel-last parameter (FusedAdam lays them out like the parameter)."""
    gen = torch.Generator(device=DEV).manual_seed(4)
    ps = synthetic_params(gen)
    opt = synthetic_optimizer(ps)
    sd = opt.state_dict()
    for i, p in enumerate(ps):
        sd["state"][i] = {"step": torch.tensor(29999.0),
                          "exp_avg": torch.randn(p.shape, generator=gen, device=DEV) * 1e-3,
                          "exp_avg_sq": torch.rand(p.shape, generator=gen, device=DEV) * 1e-6}
    opt.load_state_dict(sd)
    for it in range(2):
        synthetic_grads(ps, gen)
        checked_step(opt, f"end of training {it}")
    assert all(float(opt.state[p]["step"]) == 30001.0 for p in ps)


# ------------------------------------------------------------------------------------------------------------------
# against torch.optim.Adam: per-parameter step counts
# ------------------------------------------------------------------------------------------------------------------
SHAPES = [(1, 16, 13, 11), (4099,), (7,), (64, 33)]


def twin_params(seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for sh in SHAPES:
        t = torch.randn(sh, generator=gen, device=DEV)
        out.append(t.contiguous(memory_format=torch.channels_last) if len(sh) == 4 else t)
    return [torch.nn.Parameter(t.clone(memory_format=torch.preserve_format)) for t in out], \
        [torch.nn.Parameter(t.clone(memory_format=torch.preserve_format)) for t in out]


def groups_of(ps):
    return [{"params": ps[:2], "lr": 0.02}, {"params": ps[2:], "lr": 1e-3}]


def assign_grads(pa, pb, gen, live):
    for i, (p, q) in enumerate(zip(pa, pb)):
        if i not in live:
            p.grad = q.grad = None
            continue
        g = torch.randn(p.shape, generator=gen, device=DEV)
        g = g.contiguous(memory_format=torch.channels_last) if g.dim() == 4 else g
        p.grad, q.grad = g.clone(memory_format=torch.preserve_format), g.clone(memory_format=torch.preserve_format)


def same_as_torch(oa, pa, ob, pb, what):
    for i, (p, q) in enumerate(zip(pa, pb)):
        err = float((p - q).abs().max())
        assert err < 2e-6 * max(1.0, float(p.abs().max())), (what, i, err)
        ta = float(oa.state[p]["step"]) if oa.state[p] else 0.0
        tb = float(ob.state[q]["step"]) if ob.state[q] else 0.0
        assert ta == tb, (what, i, "step count", ta, tb)


@pytest.mark.gpu
def test_adam_parameter_joining_late_matches_torch():
    """A parameter whose gradient is None for the first 5 steps starts its own bias corrections at step 1, as
    torch.optim.Adam's per-parameter count does (the warm-up phase leaves the BRDF / normal heads without gradients)."""
    from tensoir_b200.optim import FusedAdam
    pa, pb = twin_params(5)
    oa = torch.optim.Adam(groups_of(pa), betas=(0.9, 0.99))
    ob = FusedAdam(groups_of(pb), betas=(0.9, 0.99), clear_grad=False)
    gen = torch.Generator(device=DEV).manual_seed(6)
    for it in range(10):
        assign_grads(pa, pb, gen, live={0, 1, 3} if it < 5 else {0, 1, 2, 3})
        snap = snapshot(ob)
        oa.step()
        ob.step()
        same_as_torch(oa, pa, ob, pb, f"step {it}")
        check_step(ob, snap, f"step {it}", clear_grad=False)
    assert float(ob.state[pb[2]]["step"]) == 5.0 and float(ob.state[pb[0]]["step"]) == 10.0


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["torch_to_fused", "fused_to_torch"])
def test_adam_state_dict_round_trip_with_torch(direction):
    """7 steps of one optimizer, its state_dict loaded into the other, 3 more steps of both: the loaded step counts
    carry on (torch keeps them on the CPU without capturable; FusedAdam moves them to the device on first use)."""
    from tensoir_b200.optim import FusedAdam
    pa, pb = twin_params(7)
    gen = torch.Generator(device=DEV).manual_seed(8)
    first = torch.optim.Adam(groups_of(pa), betas=(0.9, 0.99)) if direction == "torch_to_fused" else \
        FusedAdam(groups_of(pb), betas=(0.9, 0.99), clear_grad=False)
    for it in range(7):
        assign_grads(pa, pb, gen, live={0, 1, 2, 3})
        first.step()
    src, dst = (pa, pb) if direction == "torch_to_fused" else (pb, pa)
    with torch.no_grad():
        for s, d in zip(src, dst):
            d.copy_(s)
    if direction == "torch_to_fused":
        oa, ob = first, FusedAdam(groups_of(pb), betas=(0.9, 0.99), clear_grad=False)
        ob.load_state_dict(copy.deepcopy(oa.state_dict()))      # a checkpoint: load_state_dict alone shares tensors
    else:
        ob, oa = first, torch.optim.Adam(groups_of(pa), betas=(0.9, 0.99))
        oa.load_state_dict(copy.deepcopy(ob.state_dict()))
    assert all(float(ob.state[q]["step"]) == 7.0 for q in pb)
    for it in range(3):
        assign_grads(pa, pb, gen, live={0, 1, 2, 3})
        snap = snapshot(ob)
        oa.step()
        ob.step()
        same_as_torch(oa, pa, ob, pb, f"{direction} step {7 + it}")
        check_step(ob, snap, f"{direction} step {7 + it}", clear_grad=False)


# ------------------------------------------------------------------------------------------------------------------
# TV
# ------------------------------------------------------------------------------------------------------------------
class TVLoss(torch.nn.Module):
    """utils.TVLoss (utils.py:143-162), restated; float64 in, float64 out."""

    def __init__(self, TVLoss_weight=1.0):
        super().__init__()
        self.TVLoss_weight = TVLoss_weight

    def forward(self, x):
        b, _, h, w = x.shape
        ch, cw = x[:, :, 1:, :].numel() // b, x[:, :, :, 1:].numel() // b
        return self.TVLoss_weight * 2 * (torch.pow(x[:, :, 1:, :] - x[:, :, :h - 1, :], 2).sum() / ch
                                         + torch.pow(x[:, :, :, 1:] - x[:, :, :, :w - 1], 2).sum() / cw) / b


def tv_launch(planes, need_grad):
    """(vector width, CTAs per plane, largest number of grid-stride passes) of tir_tv.cu's launch for these planes."""
    vec = 4
    for p in planes:
        c = 1 if p.is_contiguous() else p.shape[1]          # NCHW (tv._layout): C images of one channel each
        al = p.data_ptr() | (p.grad.data_ptr() if need_grad else 0)
        if c % 4 or al % 16:
            vec = 1
    units = [p.numel() // vec for p in planes]
    cap = torch.cuda.get_device_properties(0).multi_processor_count * TV_CTAS_PER_SM
    grid = max(1, min(cap, -(-max(units) // TV_THREADS)))
    passes = max(-(-u // (grid * TV_THREADS)) for u in units)
    return vec, grid, passes, units


def stencil_magnitude(x, kh, kw):
    """per entry: sum of |terms| of the backward stencil (float64, logical [1,C,H,W])."""
    a = torch.zeros_like(x)
    th = (kh * (x[:, :, 1:, :] - x[:, :, :-1, :])).abs()
    tw = (kw * (x[:, :, :, 1:] - x[:, :, :, :-1])).abs()
    a[:, :, 1:, :] += th
    a[:, :, :-1, :] += th
    a[:, :, :, 1:] += tw
    a[:, :, :, :-1] += tw
    return a


def check_tv(planes, what, w=0.05 * 0.9993, factor=1e-2):
    """tv.tv_planes on ``planes`` (CUDA parameters with a nonzero .grad): value and in-place gradient vs float64."""
    from tensoir_b200 import tv, _lib
    reg = TVLoss(w)
    g0 = [p.grad.detach().clone(memory_format=torch.preserve_format) for p in planes]
    held = [p.grad for p in planes]
    before = _lib.launch_count
    val = tv.tv_planes(planes, reg, factor)
    assert _lib.launch_count - before == 1, what
    xs = [p.detach().double().requires_grad_(True) for p in planes]
    ref = sum(reg(x) * factor for x in xs)
    vec, grid, passes, _ = tv_launch(planes, need_grad=False)
    n = vec * passes + 8 + grid * len(planes) + 4
    check(val.reshape(1), ref.detach().reshape(1), EPS * n * float(ref), (what, "value", vec, grid, passes))
    gout = torch.tensor(0.9993, device=DEV)
    (val * gout).backward()
    assert _lib.launch_count - before == 2, what
    (ref * float(gout)).backward()
    for k, (p, x) in enumerate(zip(planes, xs)):
        assert p.grad is held[k], (what, k, "gradient not accumulated in place")
        _, C, H, W = p.shape
        kh = 2.0 * float(gout) * 2.0 * w * factor / (C * (H - 1) * W)
        kw = 2.0 * float(gout) * 2.0 * w * factor / (C * H * (W - 1))
        mag = stencil_magnitude(x.detach(), kh, kw) + g0[k].double().abs()
        check(p.grad, g0[k].double() + x.grad, 8.0 * EPS * mag, (what, "grad", k, tuple(p.shape)))
    return vec, grid, passes


def with_grads(planes, gen, w=0.05):
    """nonzero .grad of the size of one stencil term (kh with |x[h+1] - x[h]| ~ 1), so that an error in the terms is not
    hidden under the rounding of a larger gradient"""
    for p in planes:
        g = torch.randn(p.shape, generator=gen, device=DEV) * (4.0 * w * 1e-2 / p.numel())
        p.grad = g.contiguous(memory_format=torch.channels_last) if not p.is_contiguous() else g
    return planes


@pytest.mark.gpu
def test_tv_bench_planes(lego300):
    gen = torch.Generator(device=DEV).manual_seed(9)
    m = lego300
    dens, app = list(m.density_plane), list(m.app_plane)
    assert [tuple(p.shape) for p in dens] == [(1, 16, 300, 300)] * 3
    assert [tuple(p.shape) for p in app] == [(1, 48, 300, 300)] * 3
    assert all(p.is_contiguous(memory_format=torch.channels_last) and not p.is_contiguous() for p in dens + app)
    saved = [p.grad for p in dens + app]
    vec, grid, passes = check_tv(with_grads(dens, gen), "density planes")
    assert vec == 4 and passes >= 2, (vec, grid, passes)
    vec, grid, passes = check_tv(with_grads(app, gen), "app planes")
    _, _, _, units = tv_launch(app, True)
    assert units[0] > grid * TV_THREADS and passes >= 4, (units, grid, passes)
    for p, g in zip(dens + app, saved):
        p.grad = g


@pytest.mark.gpu
def test_tv_nchw_planes_keep_channels_apart():
    gen = torch.Generator(device=DEV).manual_seed(10)
    planes = []
    for C, H, W in ((5, 37, 29), (8, 64, 50), (3, 300, 300)):
        x = torch.randn(1, C, H, W, generator=gen, device=DEV) + 1000.0 * torch.arange(C, device=DEV).view(1, C, 1, 1)
        planes.append(torch.nn.Parameter(x))
    vec, grid, passes = check_tv(with_grads(planes, gen), "NCHW")
    assert vec == 1


@pytest.mark.gpu
def test_tv_scalar_path():
    gen = torch.Generator(device=DEV).manual_seed(11)
    cl = [torch.nn.Parameter(torch.randn(1, C, H, W, generator=gen, device=DEV)
                             .contiguous(memory_format=torch.channels_last))
          for C, H, W in ((6, 37, 29), (5, 29, 41), (7, 300, 300))]
    assert check_tv(with_grads(cl, gen), "C % 4 != 0")[0] == 1
    # views at float offsets 1, 6 and 11 of one buffer (gradients too): 16-byte misaligned, channel-last and NCHW
    shapes = [(16, 33, 31, True), (16, 40, 37, True), (4, 50, 45, False)]
    total = sum(C * H * W for C, H, W, _ in shapes) + 64
    xbuf = torch.randn(total, generator=gen, device=DEV)
    gbuf = torch.randn(total, generator=gen, device=DEV) * 1e-7
    planes, off = [], 1
    for C, H, W, channel_last in shapes:
        n = C * H * W

        def view(buf):
            if channel_last:
                return buf[off:off + n].view(1, H, W, C).permute(0, 3, 1, 2)
            return buf[off:off + n].view(1, C, H, W)
        p = torch.nn.Parameter(view(xbuf))
        p.grad = view(gbuf)
        assert p.data_ptr() % 16 and p.grad.data_ptr() % 16
        planes.append(p)
        off += n + 5
    assert check_tv(planes, "misaligned views")[0] == 1


@pytest.mark.gpu
def test_tv_mixed_sizes():
    gen = torch.Generator(device=DEV).manual_seed(12)
    planes = [torch.nn.Parameter(torch.randn(1, 16, H, W, generator=gen, device=DEV)
                                 .contiguous(memory_format=torch.channels_last))
              for H, W in ((2, 2), (300, 300), (2, 2))]
    vec, grid, passes = check_tv(with_grads(planes, gen), "2x2 with 300x300")
    assert vec == 4
