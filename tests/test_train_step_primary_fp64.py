"""The primary path's float64 stage checks (test_primary_kernels_fp64.check_stages / check_radiance_stages) on the
dumps and upstream gradients of real eager training steps, rather than on random map gradients.

A real step's g_weight is a sum over many map channels whose terms largely cancel along a ray, and the compositing
backward's g_alpha = gw_i T_i - suffix_i / om_i is where such sums lose digits; the launches of
test_primary_kernels_fp64 seed the backward with independent random map gradients and never see that structure.  Here
the fused autograd nodes (primary_fused._PrimaryRelight / _PrimaryRadiance) are wrapped for one step: the wrapper keeps
the forward's inputs and maps, the gradients the step's loss sends into them, and the parameter gradients the node's
backward returns (``_tir_grad_inplace`` off, so each is the node's own contribution in a fresh zeroed buffer); the
workspace still holds every dump of that forward and backward.  Every stage must hold its per-entry bound.  The
in-place accumulation into an existing ``.grad`` (what training with FusedAdam takes) is not what is checked here: the
kernels' writes are the same, only the buffer they add to differs.

These are stage checks: each stage is bounded from its own inputs.  They do not bound how the errors of earlier
stages propagate to the parameter gradients, so they do not replace test_general_train_gpu.py's comparison with the
reference's step.  ``test_node_gradient_unpacking_cpu`` pins how the node's gradient tuple is read back to the
parameter order of primary_fused._params.

Cases:
  * general_g20: the three runs of general_g20_train.pt (relight with mixed ids, relight without light 1, phase 1),
    with the fixture's rays, ids and seeds (test_general_train_gpu.fixture_step);
  * the bench's lego field at 64^3 as a general model with 3 and 9 lights (9: past the 8 light tables kept in shared
    memory), 1 024-ray batches, relight and phase 1, phase 1 with white_bg on and off;
  * the bench shape: the lego field at 128^3, a 4 096-ray phase-1 batch and n_samples_for(128), so rays span several
    32-sample chunks of the radiance path's compositing backward."""
import contextlib
import io

import pytest
import torch

import test_primary_kernels_fp64 as P
from gpu_helpers import load_fixture, model_from_fixture, renderer_args
from test_general_train_gpu import train_loss

DEV = "cuda:0"
MAP_ORDER = (0, 1, 2, 3, 4, 5, 7, 8)          # the node's outputs / incoming gradients of P.MAP_NAMES (6 is acc_map)
HEADS = ("renderModule", "renderModule_brdf", "renderModule_normal")


def unpack_node_grads(res, model, is_relight):
    """The parameter gradients a fused primary node's backward returns, after its leading Nones, in the order of
    primary_fused._params -> (VM-factor buffers in P.grad_bufs' channel-last layout: density planes, density lines,
    app planes, app lines; basis_mat; light_line or None; head module -> its six tensors)"""
    cl = [v[0].permute(1, 2, 0) for v in res[:12]]          # parameter-shaped views of channel-last buffers
    nl = 1 if getattr(model, "light_line", None) is not None else 0
    mod = {}
    for k, head in enumerate(HEADS if is_relight else HEADS[:1]):
        ts = res[13 + nl + 6 * k:19 + nl + 6 * k]
        if ts[0] is not None:
            mod[head] = list(ts)
    return [cl[0:3], cl[3:6], cl[6:9], cl[9:12]], res[12], res[13] if nl else None, mod


@contextlib.contextmanager
def own_stats():
    """P.STATS holds only this case's err / bound while it runs, and what it held before afterwards"""
    saved = dict(P.STATS)
    P.STATS.clear()
    try:
        yield
    finally:
        P.STATS.clear()
        P.STATS.update(saved)


@pytest.mark.parametrize("is_relight", [True, False], ids=["relight", "phase1"])
@pytest.mark.parametrize("kind", ["derived_plus_predicted", "purely_derived"])
def test_node_gradient_unpacking_cpu(golden_general, is_relight, kind):
    """unpack_node_grads on a stand-in of the backward's tuple, every gradient filled with its parameter's index in
    primary_fused._params (both normals kinds: purely_derived has no renderModule_normal job)"""
    from tensoir_b200 import primary_fused as F
    m = model_from_fixture(golden_general, "cpu")
    m.normals_kind = kind
    heads = HEADS if is_relight else HEADS[:1]
    params = F._params(m, heads)
    idx = {id(p): i for i, p in enumerate(params)}
    res = [torch.full_like(p, float(i)) for i, p in enumerate(params)]
    if is_relight and kind == "purely_derived":
        res[-6:] = [None] * 6                              # the backward returns None for a head without a job
    vmg, basis, ll, mod = unpack_node_grads(res, m, is_relight)
    names = ("density_plane", "density_line", "app_plane", "app_line")
    for name, bufs in zip(names, vmg):
        for p, b in zip(getattr(m, name), bufs):
            assert b.shape == (p.shape[2], p.shape[3], p.shape[1]) and bool((b == idx[id(p)]).all()), name
    assert bool((basis == idx[id(m.basis_mat.weight)]).all())
    assert bool((ll == idx[id(m.light_line.weight)]).all())
    want = [h for h in heads if not (h == "renderModule_normal" and kind == "purely_derived")]
    assert list(mod) == want
    for head in want:
        mlp = getattr(m, head).mlp
        for t, p in zip(mod[head], (mlp[0].weight, mlp[0].bias, mlp[2].weight, mlp[2].bias, mlp[4].weight,
                                    mlp[4].bias)):
            assert t.shape == p.shape and bool((t == idx[id(p)]).all()), head


@pytest.mark.parametrize("is_relight", [True, False], ids=["relight", "phase1"])
@pytest.mark.parametrize("kind", ["derived_plus_predicted", "purely_derived"])
def test_grad_targets_follow_params_cpu(golden_general, is_relight, kind):
    """primary_fused._grad_targets (``_tir_grad_inplace`` off): every kernel gradient buffer is the one returned for
    its parameter in the order of primary_fused._params, job slot j writes into the head of job j, and a head without
    a job gets None"""
    from tensoir_b200 import primary_fused as F
    m = model_from_fixture(golden_general, "cpu")
    m.normals_kind = kind
    m.__dict__["_tir_grad_inplace"] = False
    heads = HEADS if is_relight else HEADS[:1]
    _, n_jobs, job_heads, _ = F._jobs(m, [], heads)
    gr, grads = F._grad_targets(m, heads, job_heads)
    params = F._params(m, heads)
    assert len(grads) == len(params) and n_jobs == len(job_heads)
    vm = [gr.dplane[k] for k in range(3)] + [gr.dline[k] for k in range(3)] + [gr.aplane[k] for k in range(3)] + \
        [gr.aline[k] for k in range(3)]
    for k in range(12):
        assert vm[k] == grads[k].data_ptr() and grads[k].shape == params[k].shape
    assert gr.basis == grads[12].data_ptr() and gr.light_line == grads[13].data_ptr()
    for j, head in enumerate(job_heads):
        g = grads[14 + 6 * heads.index(head):20 + 6 * heads.index(head)]
        assert [gr.w0[j], gr.b0[j], gr.w1[j], gr.b1[j], gr.w2[j], gr.b2[j]] == [t.data_ptr() for t in g]
    for i, head in enumerate(heads):
        g = grads[14 + 6 * i:20 + 6 * i]
        if head in job_heads:
            assert all(t.shape == p.shape and not t.any() for t, p in zip(g, params[14 + 6 * i:20 + 6 * i]))
        else:
            assert head == "renderModule_normal" and kind == "purely_derived" and list(g) == [None] * 6


def captured_step(monkeypatch, m, rays, li, seed, is_relight, n_samples, args, white_bg=True):
    """One eager training step of train_loss with the fused primary node wrapped -> P.Dump of its forward/backward"""
    from tensoir_b200 import Renderer_TensoIR_train
    from tensoir_b200 import primary_fused as F
    m.__dict__["_tir_grad_inplace"] = False
    node = F._PrimaryRelight if is_relight else F._PrimaryRadiance
    rec = {}
    fwd, bwd = node.forward, node.backward

    def forward(ctx, *a):
        out = fwd(ctx, *a)
        assert "out" not in rec, "one primary forward per step"
        rec["args"], rec["out"] = a, out
        return out

    def backward(ctx, *g):
        res = bwd(ctx, *g)
        rec["grads"], rec["keep"], rec["res"] = g, ctx.keep, res
        return res
    monkeypatch.setattr(node, "forward", staticmethod(forward))
    monkeypatch.setattr(node, "backward", staticmethod(backward))
    for p in m.parameters():
        p.grad = None
    torch.manual_seed(seed)
    ret = Renderer_TensoIR_train(rays, None, li, m, N_samples=n_samples, white_bg=white_bg, is_train=True,
                                 is_relight=is_relight, sample_method='stratified_sampling', chunk_size=160000,
                                 device=DEV, args=args)
    train_loss(ret, is_relight).backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert "res" in rec
    out, g = rec["out"], rec["grads"]
    if is_relight:
        _, _, _, _, _, noise, li_, rays_, ws, jitter = rec["keep"]
        n_rays = rays_.shape[0]
        n_samples, bg = rec["args"][5], int(bool(rec["args"][6]))
        shapes = (3, 1, 3, 3, 1, 3, 1, 1)
        maps = [out[k].detach().reshape(n_rays, c) for k, c in zip(MAP_ORDER, shapes)]
        gm = {name: (None if g[k] is None else g[k].float().reshape(n_rays, c))
              for name, k, c in zip(P.MAP_NAMES, MAP_ORDER, shapes)}
        res = rec["res"][8:]
        extra = dict(mask=out[9], losses=torch.stack([out[10].detach(), out[11].detach()]), gm=gm, g_acc_map=g[6],
                     g_la=g[10], g_lr=g[11], noise=noise)
    else:
        _, _, li_, rays_, ws, jitter, bg = rec["keep"]
        n_rays = rays_.shape[0]
        n_samples = rec["args"][4]
        maps = [out[0].detach(), out[1].detach().reshape(n_rays, 1)]
        gm = dict(rgb=g[0], depth=g[1])
        res = rec["res"][7:]
        extra = dict(mask=None, losses=None, gm=gm, g_acc_map=g[2], g_la=None, g_lr=None, noise=None)
    vmg, g_basis, g_ll, mod = unpack_node_grads(res, m, is_relight)
    return P.Dump(m=m, ws=ws, rays=rays_, li=li_, jitter=jitter, table=None, n_samples=n_samples, cv=ws.cap_valid,
                  ca=ws.cap_app, bg=bg, maps=maps, vmg=vmg, g_basis=g_basis, g_ll=g_ll, mod=mod, pre=0.0, guards=False,
                  fresh=False, **extra)


def run(d, is_relight, key):
    with own_stats():
        if is_relight:
            r = P.check_stages(d, stats_key=key)
            P.assert_gates(r["gates"], r["total_app"], key)
        else:
            r = P.check_radiance_stages(d, stats_key=key)
        P.report(f"{key}, bg {d.bg}")
    assert r["total_app"] > 0
    return r


# ------------------------------------------------------------------------------------------------------ general_g20
@pytest.fixture(scope="module")
def train_fx():
    from tensoir_b200 import _lib
    _lib.load()
    return load_fixture("general_g20_train.pt")


@pytest.mark.parametrize("name", ("relight_mixed", "relight_no1", "phase1"))
@pytest.mark.gpu
def test_general_g20_step_stages(monkeypatch, golden_general, train_fx, name):
    run_ = train_fx["runs"][name]
    m = model_from_fixture(golden_general, DEV)
    m.__dict__["_tir_randn_like"] = lambda t: torch.randn(t.shape).to(t.device)   # CPU stream like the reference's
    d = captured_step(monkeypatch, m, train_fx["rays"], run_["light_idx"], run_["seed"], run_["is_relight"],
                      train_fx["n_samples"], renderer_args(train_fx["second_nsample"]))
    run(d, run_["is_relight"], f"general_g20 {name}")


# ---------------------------------------------------------------------------------------------- lego at training size
def _lego(n_lights, grid=64):
    from tensoir_b200.synthetic import make_lego_model
    with contextlib.redirect_stdout(io.StringIO()):
        m = make_lego_model(grid, DEV, general=True, lights=[f"light{k}" for k in range(n_lights)])
    m.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)
    return m


def _coin_seed(n_rays, want_bg):
    """a seed whose background coin (drawn on the CPU after the per-ray jitter, primary_fused._host_draws) is want_bg"""
    for s in range(100):
        g = torch.Generator().manual_seed(s)
        torch.rand(n_rays, 1, generator=g)
        if bool(torch.rand((1,), generator=g) < 0.5) == want_bg:
            return s
    raise AssertionError


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["relight", "phase1", "phase1_no_white_bg"])
@pytest.mark.parametrize("n_lights", [3, 9])
def test_lego_general_step_stages(monkeypatch, n_lights, mode):
    from tensoir_b200.synthetic import hemisphere_poses, training_batch
    m = _lego(n_lights)
    rays, li = training_batch(hemisphere_poses(100), 1024, 1, n_lights=n_lights)
    assert set(li.view(-1).tolist()) == set(range(n_lights))
    white = mode != "phase1_no_white_bg"
    seed = 7 if white else _coin_seed(1024, False)
    d = captured_step(monkeypatch, m, rays.to(DEV), li.to(DEV), seed, mode == "relight", m.nSamples,
                      renderer_args(96), white_bg=white)
    assert d.bg == int(white)
    run(d, mode == "relight", f"lego 64, {n_lights} lights, {mode}")


@pytest.mark.gpu
def test_lego_bench_shape_phase1_stages(monkeypatch):
    """The bench's field and phase-1 batch: rays longer than two 32-sample chunks in the radiance path."""
    from tensoir_b200.synthetic import hemisphere_poses, make_lego_model, n_samples_for, training_batch
    with contextlib.redirect_stdout(io.StringIO()):
        m = make_lego_model(128, DEV)
    rays, li = training_batch(hemisphere_poses(100), 4096, 0)
    d = captured_step(monkeypatch, m, rays.to(DEV), li.to(DEV), 11, False, n_samples_for(128), renderer_args(96))
    r = run(d, False, "lego 128 phase 1")
    assert int(r["lengths"].max()) > 64
