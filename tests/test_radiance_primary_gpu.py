"""The fused radiance-only primary march (TensorBase.forward with is_relight=False, the warm-up phase of training):
tir_primary_radiance / tir_primary_radiance_backward against the oracle's autograd, against the modular per-op path,
on the edge cases, and as the CUDA-graph step of phase 1 (StaticTrainStep(is_relight=False))."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import tensoir_oracle as O            # noqa: E402
from helpers import oracle_field, named_oracle_params   # noqa: E402
from gpu_helpers import load_fixture, load_shrunk_state, model_from_fixture, renderer_args   # noqa: E402
from test_gpu_parity import DEV, TOL, close, _FixedRand      # noqa: E402

N_SAMPLES = 60


def _cases():
    return [("rotated", True), ("rotated", False), ("general", True), ("shrunk_A", True)]


def _fixture(name):
    if name == "rotated":
        return load_fixture("rotated_g24.pt")
    if name == "general":
        return load_fixture("general_g20.pt")
    return load_shrunk_state("A")


def _loss(rgb, depth, acc):
    """mse(rgb, pixel colours) is the phase-1 loss (the target is a fixed draw of colours in [0, 1], like the pixels of
    a training batch); the acc / depth terms exercise the compositing gradients of the other two maps."""
    target = torch.rand(rgb.shape, generator=torch.Generator().manual_seed(2)).to(rgb.device, rgb.dtype)
    return ((rgb - target) ** 2).mean() + 0.3 * acc.mean() + 0.05 * depth.mean()


APP_SIDE = ("app_plane.", "app_line.", "basis_mat.", "light_line.", "renderModule.")


def _fused_step(m, rays, li, seed, n_samples=N_SAMPLES):
    torch.manual_seed(seed)
    out = m(rays.to(DEV), li.to(DEV), white_bg=True, is_train=True, is_relight=False, N_samples=n_samples)
    loss = _loss(out[0], out[1], out[6])
    loss.backward()
    return out, loss


def _kink_correction(m, fx, out):
    """Gradient change of the renderModule head when its two ReLUs take the kernel's branches instead of the float64
    ones -> {parameter name: delta (float64, CPU)}, empty when every branch agrees.

    A pre-activation within the split-BF16 error of 0 can come out on either side of the ReLU kink in the kernel's
    forward (tests/test_heads_kernels_fp64.py bounds that error), and the gradient of that sample then differs by its
    whole d z entry.  The head is evaluated in float64 on the fused step's own appearance list (points, weights, ray
    gradient), once with float64's branches and once with the kernel's dumped ones; every differing branch must lie
    within twice the split-BF16 bound of its pre-activation."""
    from test_heads_kernels_fp64 import gemm_bound, EPS32
    ws = m.__dict__["_tir_radiance_ws"]
    n = int(ws.t["a_offsets"][-1])
    ray = ws.t["a_ray"][:n].long()
    kmask = [ws.t["h1_0"][:n] > 0, ws.t["h2_0"][:n] > 0]
    rgb = out[0].detach().requires_grad_(True)
    (g_rgb,) = torch.autograd.grad(_loss(rgb, out[1].detach(), out[6].detach()), rgb)
    rays, li = fx["rays"].to(DEV).double(), fx["light_idx"].reshape(-1).to(DEV)[ray].view(-1, 1).long()
    grads = []
    for use_kernel in (False, True):
        old = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)
        try:
            f = oracle_field(fx).to(DEV, torch.float64)
            for p in f.parameters():
                p.requires_grad_(True)
            feat = O.app_feature(f, ws.t["a_xn"][:n].double(), li)
            vd = rays[ray, 3:6]
            x = torch.cat([feat, vd, O.positional_encoding(feat, f.fea_pe), O.positional_encoding(vd, f.view_pe)], -1)
            mm = f.mlp_rgb
            z1 = F.linear(x, mm.w0, mm.b0)
            h1 = z1 * (kmask[0] if use_kernel else z1 > 0)
            z2 = F.linear(h1, mm.w1, mm.b1)
            h2 = z2 * (kmask[1] if use_kernel else z2 > 0)
            o = torch.sigmoid(F.linear(h2, mm.w2, mm.b2))
            aw = ws.t["a_w"][:n].double()[:, None]
            rgb_map = torch.zeros(rays.shape[0], 3, device=DEV).index_add_(0, ray, aw * o)
            if not use_kernel:
                flips = [(kmask[0] != (z1 > 0)), (kmask[1] != (z2 > 0))]
                if not any(bool(fl.any()) for fl in flips):
                    return {}
                for fl, z, a, w, b in ((flips[0], z1, x, mm.w0, mm.b0), (flips[1], z2, h1, mm.w1, mm.b1)):
                    bnd = 2 * gemm_bound(a.detach().abs() @ w.detach().abs().t(), a.shape[1]) + EPS32 * b.detach().abs()
                    assert bool((z.detach().abs() <= bnd)[fl].all()), "a ReLU branch differs outside the kernel's error"
            (rgb_map * g_rgb.double()).sum().backward()
        finally:
            torch.set_default_dtype(old)
        grads.append({k: p.grad for k, p in named_oracle_params(f).items() if p.grad is not None})
    return {k: (grads[1][k] - grads[0][k]).cpu() for k in grads[0]}


def _oracle_step(name, with_mask):
    """One phase-1 training step (recorded CPU jitter, white background) against the oracle differentiated by torch
    autograd: lists bit-exact, maps and loss 1e-4 (1 + |x|) asserted here -> {parameter: max gradient error / max}.
    Where the fused head's forward took the other branch of a ReLU at a pre-activation within its arithmetic error of
    0, the oracle's gradient is moved to that branch (``_kink_correction``)."""
    fx = _fixture(name)
    rays, li = fx["rays"], fx["light_idx"]
    m = model_from_fixture(fx, DEV, with_mask=with_mask)
    out, loss = _fused_step(m, rays, li, seed=31)
    assert "_tir_radiance_ws" in m.__dict__ and "_tir_primary_ws" not in m.__dict__     # the fused radiance node ran
    assert all(out[k] is None for k in (2, 3, 4, 5, 7, 8, 9, 10, 11))

    f = oracle_field(fx, with_mask=with_mask, requires_grad=True)
    jit = torch.rand(rays.shape[0], 1, generator=torch.Generator().manual_seed(31))        # the same CPU draw
    want = O.primary_forward(f, rays, li, True, True, False, N_SAMPLES, jitter=jit, return_aux=True)
    aux = want[-1]
    close(out[0], want[0], TOL, "rgb_map")
    close(out[1], want[1], TOL, "depth_map")
    close(out[6], want[6], TOL, "acc_map")
    # the valid list and the appearance list are the reference's masks, row for row
    ws = m.__dict__["_tir_radiance_ws"]
    n_valid = int(ws.t["offsets"][-1])
    idx = aux["valid"].nonzero()
    assert n_valid == idx.shape[0]
    assert torch.equal(ws.t["v_ray"][:n_valid].cpu().long(), idx[:, 0])
    assert torch.equal(ws.t["v_sample"][:n_valid].cpu().long(), idx[:, 1])
    n_app = int(ws.t["a_offsets"][-1])
    src = ws.t["a_src"][:n_app].cpu()
    app = torch.stack([ws.t["v_ray"][:n_valid].cpu().long()[src], ws.t["v_sample"][:n_valid].cpu().long()[src]], 1)
    assert n_app > 0 and torch.equal(app, aux["app_mask"].nonzero())
    wl = _loss(want[0], want[1], want[6])
    close(loss, wl, TOL, "loss")
    wl.backward()
    corr = _kink_correction(m, fx, out)
    worst, n = {}, 0
    named = named_oracle_params(f)
    for k, p in m.named_parameters():
        w = named.get(k)
        if w is None or w.grad is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        want = w.grad.double() + corr[k] if k in corr else w.grad.double()
        scale = float(want.abs().max()) + 1e-12
        worst[k] = float((p.grad.detach().cpu().double() - want).abs().max()) / scale
        n += 1
    assert n >= 12 + 1 + 6, sorted(worst)           # VM factors, basis, renderModule (+ light_line)
    return worst


@pytest.mark.parametrize("name,with_mask", _cases())
def test_radiance_step_matches_oracle_autograd(name, with_mask):
    """Lists, maps and loss on every case; every parameter gradient within 5e-4 of its largest entry, except the
    appearance-side gradients of shrunk state A (the next test)."""
    worst = _oracle_step(name, with_mask)
    if name == "shrunk_A":
        worst = {k: v for k, v in worst.items() if not k.startswith(APP_SIDE)}
        assert len(worst) == 6                       # the density factors are still checked
    bad = {k: v for k, v in worst.items() if v > 5e-4}
    assert not bad, (bad, max(worst.values()))


def test_shrunk_state_a_appearance_gradients_match_oracle():
    """Appearance factors, basis and renderModule gradients on shrunk state A, within 5e-4 of their max.  One
    first-layer pre-activation of this step (sample 241, unit 45) is 1.6e-7 in float64, 0.0013 of the split-BF16
    error bound of the head's forward: the kernel puts it on the other side of the ReLU, which alone moves these
    gradients by up to 1.1e-2 of their max.  The oracle's gradient is taken on the kernel's branch there
    (DESIGN.md §9)."""
    worst = {k: v for k, v in _oracle_step("shrunk_A", True).items() if k.startswith(APP_SIDE)}
    bad = {k: v for k, v in worst.items() if v > 5e-4}
    assert not bad, (bad, max(worst.values()))


@pytest.mark.parametrize("name,with_mask", _cases())
def test_fused_radiance_matches_modular_path(name, with_mask):
    """Fused radiance node against the modular path (march + fused_head + segment sum, torch autograd): maps 2e-5,
    gradients 2e-4 of their largest entry."""
    fx = _fixture(name)
    outs = []
    for modular in (True, False):
        m = model_from_fixture(fx, DEV, with_mask=with_mask)
        m.__dict__["_tir_modular"] = modular
        out, loss = _fused_step(m, fx["rays"], fx["light_idx"], seed=7)
        outs.append((out, loss, {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}))
    (o0, l0, g0), (o1, l1, g1) = outs
    for k in (0, 1, 6):
        close(o1[k], o0[k], 2e-5, f"map {k}")
    close(l1, l0, 2e-5, "loss")
    nz = lambda g: {k for k, v in g.items() if float(v.abs().max()) > 0}      # noqa: E731
    assert nz(g0) == nz(g1), nz(g0) ^ nz(g1)
    worst = {k: float((g0[k] - g1[k]).abs().max()) / (float(g0[k].abs().max()) + 1e-12) for k in nz(g0)}
    bad = {k: v for k, v in worst.items() if v > 2e-4}
    assert not bad, bad


def test_radiance_eval_matches_golden_and_light_index():
    """No-grad evaluation through the fused node against the reference's is_relight=False maps of the rotated fixture,
    and the general model's per-ray light index: every ray rendered under each light equals the oracle."""
    fx = load_fixture("rotated_g24.pt")
    m = model_from_fixture(fx, DEV)
    with torch.no_grad():
        got = m(fx["rays"].to(DEV), fx["light_idx"].to(DEV), white_bg=True, is_train=False, is_relight=False,
                N_samples=-1)
    assert "_tir_radiance_ws" in m.__dict__
    for k, g, w in zip(range(12), got, fx["primary_eval_norelight"]):
        if w is None:
            assert g is None, k
        else:
            close(g, w, TOL, f"golden {k}")
    fx = load_fixture("general_g20.pt")
    m = model_from_fixture(fx, DEV)
    f = oracle_field(fx)
    rays = fx["rays"]
    for light in range(3):
        li = torch.full((rays.shape[0], 1), light, dtype=torch.int32)
        with torch.no_grad():
            got = m(rays.to(DEV), li.to(DEV), white_bg=True, is_train=False, is_relight=False, N_samples=-1)
        want = O.primary_forward(f, rays, li, True, False, False, -1)
        close(got[0], want[0], TOL, f"general rgb, light {light}")
    mixed = (torch.arange(rays.shape[0]) % 3).view(-1, 1).to(torch.int32)
    with torch.no_grad():
        got = m(rays.to(DEV), mixed.to(DEV), white_bg=True, is_train=False, is_relight=False, N_samples=-1)
    close(got[0], O.primary_forward(f, rays, mixed, True, False, False, -1)[0], TOL, "general rgb, mixed lights")


def test_radiance_edge_cases():
    """Zero rays; a batch in which every ray misses the aabb (no valid sample: white, acc 0, depth = 1 * rays[..., -1],
    zero gradients); no alpha mask; rays with no appearance sample next to rays with many; a non-white background
    coin drawn on the CPU after the jitter."""
    fx = load_fixture("rotated_g24.pt")
    m = model_from_fixture(fx, DEV)
    # (i) zero rays
    out = m(torch.zeros(0, 6, device=DEV), torch.zeros(0, 1, dtype=torch.int32, device=DEV), is_train=True,
            is_relight=False, N_samples=N_SAMPLES)
    assert out[0].shape == (0, 3) and out[1].shape == (0,) and out[6].shape == (0,)
    # (ii) every ray misses the box
    o = torch.tensor([[0., 0., 4.]]).repeat(5, 1)
    d = torch.nn.functional.normalize(torch.tensor([[0.1, 0.2, 1.0]]), dim=-1).repeat(5, 1)
    away = torch.cat([o, d], 1).to(DEV)
    out = m(away, torch.zeros(5, 1, dtype=torch.int32, device=DEV), is_train=True, is_relight=False,
            N_samples=N_SAMPLES)
    assert torch.equal(out[6].detach().cpu(), torch.zeros(5))
    assert torch.equal(out[0].detach().cpu(), torch.ones(5, 3))
    assert torch.equal(out[1].detach().cpu(), away[:, 5].cpu())
    assert int(m.__dict__["_tir_radiance_ws"].t["offsets"][-1]) == 0
    for p in m.parameters():
        p.grad = None
    _loss(out[0], out[1], out[6]).backward()
    for k, p in m.named_parameters():
        assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
    # (iii) a mixed batch without alpha mask, white_bg=False: the coin is the CPU draw after the jitter
    m2 = model_from_fixture(fx, DEV, with_mask=False)
    f2 = oracle_field(fx, with_mask=False)
    rays = torch.cat([fx["rays"][:24], away.cpu()[:3]])
    li = torch.zeros(rays.shape[0], 1, dtype=torch.int32)
    for seed in range(6):                                   # both outcomes of the coin
        torch.manual_seed(seed)
        got = m2(rays.to(DEV), li.to(DEV), white_bg=False, is_train=True, is_relight=False, N_samples=N_SAMPLES)
        torch.manual_seed(seed)
        jit = torch.rand(rays.shape[0], 1)
        coin = torch.rand((1,))
        want = O.primary_forward(f2, rays, li, False, True, False, N_SAMPLES, jitter=jit, bg_coin=coin)
        close(got[0], want[0], TOL, f"rgb, seed {seed}")
        close(got[1], want[1], TOL, f"depth, seed {seed}")
        close(got[6], want[6], TOL, f"acc, seed {seed}")


def _phase1_loss(ret, target):
    return ((ret["rgb_map"] - target) ** 2).mean()


def test_phase1_graph_replay_tracks_eager_training_for_50_steps():
    """50 phase-1 steps of the bench scene at 128^3 without an alpha mask (the state of a fresh training run),
    1024-ray batches, Adam: CUDA-graph replay of StaticTrainStep(is_relight=False) against the eager fused step on
    identical batches and identical per-ray jitter.  Losses agree to 2e-3 relative step by step; no replay overflowed."""
    from tensoir_b200 import Renderer_TensoIR_train
    from tensoir_b200.static_step import StaticTrainStep
    from tensoir_b200.synthetic import make_lego_model, hemisphere_poses, training_batch, n_samples_for
    import bench
    grid, n_rays, steps = 128, 1024, 50
    n_s = n_samples_for(grid)
    poses = hemisphere_poses(100)
    batches = [tuple(t.to(DEV) for t in training_batch(poses, n_rays, it)) for it in range(steps)]
    target = torch.full((n_rays, 3), 0.5, device=DEV)
    g = torch.Generator().manual_seed(5)
    jit = [torch.rand(n_rays, 1, generator=g) for _ in range(steps)]
    runs, caps = [], None
    for graphed in (False, True):
        model = make_lego_model(grid, DEV)
        model.alphaMask = None
        opt = torch.optim.Adam(model.get_optparam_groups(0.02, 0.001), betas=(0.9, 0.99), fused=True,
                               capturable=graphed)
        losses = []
        if graphed:
            # the appearance list grows ~20x while the density forms: lists sized by the eager run (whose workspace
            # grew to fit every step) keep every replay from overflowing, so each recorded loss is that step's
            st = StaticTrainStep(model, opt, n_rays, n_s, bench.Args, lambda ret, m: _phase1_loss(ret, target),
                                 device=DEV, lag=1, is_relight=False, cap_valid=caps[0], cap_app=caps[1])
            it_box = [0]

            def stage(slot, st=st):
                st.static["jitter"].copy_(jit[min(it_box[0], steps - 1)])
            st._stage_host_randoms = stage
            st.capture(warmup=1)
            for it, (rays, li) in enumerate(batches):
                it_box[0] = it
                losses.append(st.run(rays, li).detach().clone())
            st.flush()
            assert st.overflowed() == 0 and st.redone == 0
            st.release()
        else:
            for it, (rays, li) in enumerate(batches):
                torch.rand = _FixedRand(jit[it])
                try:
                    ret = Renderer_TensoIR_train(rays, None, li, model, N_samples=n_s, white_bg=True, is_train=True,
                                                 is_relight=False, device=DEV, args=bench.Args)
                finally:
                    torch.rand = _FixedRand.orig
                loss = _phase1_loss(ret, target)
                opt.zero_grad(set_to_none=True)
                loss.backward()
                opt.step()
                losses.append(loss.detach().clone())
            ws = model.__dict__["_tir_radiance_ws"]
            caps = (ws.cap_valid, ws.cap_app)
        runs.append(torch.stack(losses).cpu())
    l0, l1 = runs
    assert torch.isfinite(l0).all() and torch.isfinite(l1).all()
    assert float(l0[-1]) < float(l0[0])
    rel = ((l0 - l1).abs() / l0.abs().clamp_min(1e-6)).max()
    assert float(rel) < 2e-3, float(rel)


def test_phase1_graph_step_overflow_is_redone():
    """Lists that are too short never change a phase-1 step: the overflowed replay is an exact no-op (Adam's step
    counters do not move), the host grows the lists, re-captures and redoes the batch, and the Adam moments and the
    parameters end where a run with large enough lists ends (same batch and jitter every step, so only the order of
    the gradient atomics differs).

    The large-list run starts with the valid list at its largest possible length, n_rays * n_samples: without an alpha
    mask the valid samples fill ~87 % of it, above the 80 % high-water mark, and a list that cannot grow must not be
    re-captured for (it used to be, and the next step raised "cannot grow any further")."""
    from tensoir_b200.static_step import StaticTrainStep
    fx = load_fixture("rotated_g24.pt")
    rays, li = fx["rays"].to(DEV), fx["light_idx"].to(DEV)
    n_max = rays.shape[0] * N_SAMPLES
    outs = []
    for tiny in (False, True):
        m = model_from_fixture(fx, DEV, with_mask=False)
        opt = torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), betas=(0.9, 0.99), fused=True, capturable=True)
        st = StaticTrainStep(m, opt, rays.shape[0], N_SAMPLES, renderer_args(24),
                             lambda ret, mm: ((ret["rgb_map"] - 0.5) ** 2).mean(), device=DEV, lag=1,
                             is_relight=False, cap_valid=n_max, cap_app=n_max)

        def stage(slot, st=st):
            st.static["jitter"].fill_(0.5)
        st._stage_host_randoms = stage
        if tiny:
            st._set_caps(n_max // 8, n_max // 64)
        st.capture(warmup=1)
        for _ in range(3):
            st.run(rays, li)
        st.flush()
        if tiny:
            assert st.redone >= 1 and st.recaptures >= 1
        else:
            assert st._seen[0] > st.grow_at * n_max, st._seen           # the valid list is past its high-water mark
            assert st.redone == 0 and st.overflowed() == 0 and st.recaptures == 0, (st.redone, st.recaptures)
        steps = {int(v["step"].item()) for v in opt.state.values()}
        assert steps == {3}, steps
        names = {id(p): k for k, p in m.named_parameters()}
        outs.append(({k: p.detach().clone() for k, p in m.named_parameters()},
                     {names[id(p)]: (s["exp_avg"].clone(), s["exp_avg_sq"].clone()) for p, s in opt.state.items()}))
        st.release()
    (p0, s0), (p1, s1) = outs
    assert set(s0) == set(s1) and len(s0) >= 19
    for k in s0:
        for a, b, what in ((s0[k][0], s1[k][0], "exp_avg"), (s0[k][1], s1[k][1], "exp_avg_sq")):
            scale = float(a.abs().max())
            assert float((a - b).abs().max()) <= 1e-5 * scale, (k, what, float((a - b).abs().max()) / max(scale, 1e-30))
    for k in p0:
        # a step applied twice or partly moves a parameter by ~lr = 0.02; Adam's 1 / (sqrt(v) + eps) turns the rounding
        # noise of gradients far below eps = 1e-8 into updates of up to ~lr * noise / eps, hence not 1e-5 here
        assert float((p0[k] - p1[k]).abs().max()) < 1e-3 * max(float(p0[k].abs().max()), 1.0), k
