"""The general multi-light model's training step on the CUDA path: one SG set per light in ``lgtSGs_list`` (outside
``named_parameters()`` and the state_dict) and one light_line row per light.

* On general_g20.pt's state, the eager step against the real reference's (tests/golden/make_general_train_golden.py):
  relight steps with mixed light ids and without light 1, and a phase-1 (radiance-only) step.  Maps to
  1e-4 (1 + |x|), every gradient, each SG set's included, to 5e-4 of its max (the density factors to DENSITY_TOL); an
  absent light's SG set exactly 0.
* At training size (the bench's lego field at 64^3, 1 024-ray batches, stratified light directions, 3 and 9 lights,
  9 being past the 8 light tables the kernels keep in shared memory), two exact identities, each up to the float
  atomics order of the scatters: relabelling the lights permutes every light gradient and changes nothing else, and
  with identical lights the mixed-id step equals the all-zero-id step.
* Graph replays of ``StaticTrainStep`` on the three-light model, with an optimizer that records each replay's
  gradients: every recorded gradient equals the eager step's from the same parameters and host draws."""
import contextlib
import io

import pytest
import torch

pytestmark = pytest.mark.gpu

from gpu_helpers import load_fixture, model_from_fixture, renderer_args   # noqa: E402

DEV = "cuda:0"
RUNS = ("relight_mixed", "relight_no1", "phase1")
GRID, N_RAYS = 64, 1024
# new light j is old light PERM[j]: light 8 moves to 0, light 4 to 8, and no light keeps its index
PERMS = {3: [2, 0, 1], 9: [8, 3, 1, 0, 5, 7, 2, 6, 4]}
MAP_TOL, GRAD_TOL = 2e-6, 1e-5
# The density factors' gradients on general_g20.pt cancel heavily: against a float64 oracle with the same draws, the fp32
# reference's own density_line.2 is 2.0e-4 of its max away, the modular autograd path 3.6e-4 and the fused primary
# backward 1.7e-3 (relight_mixed; relight_no1 6.0e-4, phase 1 1.6e-4; H100).  Leaving normals_diff_map out of the
# loss does not shrink it, and the build before the run-merged VM scatters gives the same numbers.  Every other
# gradient holds the 5e-4 of tests/test_gpu_parity.py.
DENSITY_TOL = 2e-3


def train_loss(ret, is_relight):
    """make_general_train_golden.train_loss."""
    target = torch.full_like(ret["rgb_map"], 0.5)
    loss = ((ret["rgb_map"] - target) ** 2).mean()
    if is_relight:
        loss = (loss + 0.2 * ((ret["rgb_with_brdf_map"] - target) ** 2).mean()
                + 0.0005 * ret["normals_diff_map"].mean() + 0.001 * ret["normals_orientation_loss_map"].mean()
                + 0.001 * ret["albedo_smoothness_loss"] + 0.001 * ret["roughness_smoothness_loss"])
    return loss


def all_params(model):
    """named_parameters() plus each light's SG set as ``lgtSGs_list.k``."""
    return dict(model.named_parameters()) | {f"lgtSGs_list.{k}": p for k, p in enumerate(model.lgtSGs_list)}


def step(model, rays, light_idx, seed, is_relight, n_samples, args):
    """One eager training step from the model's current parameters -> (maps, loss, gradients)."""
    from tensoir_b200 import Renderer_TensoIR_train
    params = all_params(model)
    for p in params.values():
        p.grad = None
    torch.manual_seed(seed)
    ret = Renderer_TensoIR_train(rays, None, light_idx, model, N_samples=n_samples, white_bg=True, is_train=True,
                                 is_relight=is_relight, sample_method='stratified_sampling', chunk_size=160000,
                                 device=DEV, args=args)
    loss = train_loss(ret, is_relight)
    loss.backward()
    maps = {k: v.detach().clone() for k, v in ret.items() if torch.is_tensor(v) and v.dtype != torch.bool}
    grads = {k: p.grad.detach().clone() for k, p in params.items() if p.grad is not None}
    return maps, loss.detach().clone(), grads


def rel_err(got, want):
    return float((got - want).abs().max()) / max(float(want.abs().max()), 1e-30)


# ----------------------------------------------------------------------------------------------- the reference's step
@pytest.fixture(scope="module")
def train_fx():
    from tensoir_b200 import _lib
    _lib.load()
    return load_fixture("general_g20_train.pt")


def fixture_step(golden_general, train_fx, run, is_relight=None):
    m = model_from_fixture(golden_general, DEV)
    m.__dict__["_tir_randn_like"] = lambda t: torch.randn(t.shape).to(t.device)   # CPU stream like the reference's
    is_relight = run["is_relight"] if is_relight is None else is_relight
    from tensoir_b200 import Renderer_TensoIR_train
    params = all_params(m)
    torch.manual_seed(run["seed"])
    got = Renderer_TensoIR_train(train_fx["rays"], None, run["light_idx"], m, N_samples=train_fx["n_samples"],
                                 white_bg=True, is_train=True, is_relight=is_relight,
                                 sample_method='stratified_sampling', chunk_size=160000, device=DEV,
                                 args=renderer_args(train_fx["second_nsample"]))
    loss = train_loss(got, is_relight)
    loss.backward()
    return got, loss, params


@pytest.mark.parametrize("name", RUNS)
def test_general_train_step_matches_reference(golden_general, train_fx, name):
    run, want_grads = train_fx["runs"][name], train_fx[name]
    got, loss, params = fixture_step(golden_general, train_fx, run)
    for k, w in run["maps"].items():
        if w is None:
            assert got[k] is None, k
            continue
        g = got[k].detach().cpu()
        if w.dtype == torch.bool:
            assert torch.equal(g, w), k
            continue
        err = (g.float() - w).abs()
        assert bool((err <= 1e-4 * (1 + w.abs())).all()), (k, float(err.max()))
    assert float((loss.detach().cpu() - run["loss"]).abs()) <= 1e-4 * (1 + float(run["loss"].abs()))
    assert set(params) == set(want_grads), set(params) ^ set(want_grads)
    worst = {}
    for k, w in want_grads.items():
        g = params[k].grad
        if w is None:
            assert g is None or float(g.abs().max()) == 0.0, k
            continue
        worst[k] = rel_err(g.detach().cpu(), w)
    print(f"{name}: worst gradient err / max", {k: f"{v:.2e}" for k, v in sorted(worst.items(), key=lambda kv: -kv[1])})
    assert len(worst) >= (20 if run["is_relight"] else 10)
    bad = {k: v for k, v in worst.items() if v > (DENSITY_TOL if k.startswith("density_") else 5e-4)}
    assert not bad, bad
    ids = set(run["light_idx"].view(-1).tolist())
    for k in range(3):
        g = params[f"lgtSGs_list.{k}"].grad
        if not run["is_relight"]:
            assert g is None or float(g.abs().max()) == 0.0, k
        elif k not in ids:
            assert float(g.abs().max()) == 0.0, k                 # exactly: no ray of the batch reads light k
        else:
            assert float(g.abs().max()) > 0.0, k


def test_general_phase1_absent_light_row_is_zero(golden_general, train_fx):
    """A radiance-only step reads light_line only at each ray's own light (no intrinsic mean over the rows), so the row of
    a light outside the batch gets exactly zero gradient; the SG sets get none."""
    run = train_fx["runs"]["relight_no1"]
    got, _, params = fixture_step(golden_general, train_fx, run, is_relight=False)
    rows = params["light_line.weight"].grad.abs().amax(1).tolist()
    assert rows[1] == 0.0 and rows[0] > 0 and rows[2] > 0, rows
    for k in range(3):
        g = params[f"lgtSGs_list.{k}"].grad
        assert g is None or float(g.abs().max()) == 0.0, k


# ------------------------------------------------------------------------------------------ identities at training size
@pytest.fixture(scope="module")
def lego():
    """The bench's lego field at 64^3 with 3 and with 9 lights, a 1 024-ray batch of each (mixed light ids)."""
    from tensoir_b200 import _lib
    from tensoir_b200.synthetic import hemisphere_poses, make_lego_model, training_batch
    _lib.load()
    out = {}
    for n in PERMS:
        with contextlib.redirect_stdout(io.StringIO()):
            m = make_lego_model(GRID, DEV, general=True, lights=[f"light{k}" for k in range(n)])
        m.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)     # xyz noise fixed per row
        # The intrinsic feature reads the mean of all light_line rows.  Rows on a 2^-10 grid sum exactly in fp32, so
        # that mean is the same float in every order of the rows; with the rows as initialised, relabelling the lights
        # reorders the sum, and its last-bit change moved normal_map by up to 4.7e-6 of its max (H100).
        with torch.no_grad():
            m.light_line.weight.copy_(torch.round(m.light_line.weight * 1024) / 1024)
        rays, li = training_batch(hemisphere_poses(100), N_RAYS, 1, n_lights=n)
        assert set(li.view(-1).tolist()) == set(range(n))
        out[n] = (m, rays.to(DEV), li.to(DEV))
    return out


def _set_lights(model, sgs, rows):
    with torch.no_grad():
        for p, v in zip(model.lgtSGs_list, sgs):
            p.copy_(v)
        model.light_line.weight.copy_(rows)


def _light_state(model):
    return [p.detach().clone() for p in model.lgtSGs_list], model.light_line.weight.detach().clone()


def _check_maps(got, want, what):
    assert got.keys() == want.keys()
    for k in want:
        err = rel_err(got[k], want[k])
        assert err <= MAP_TOL, (what, k, err)


def _max_errs(got, want, keys):
    return {k: rel_err(got[k], want[k]) for k in keys}


@pytest.mark.parametrize("is_relight", [True, False], ids=["relight", "phase1"])
@pytest.mark.parametrize("n_lights", sorted(PERMS))
def test_relabelling_lights_permutes_their_gradients(lego, n_lights, is_relight):
    """Light j of the relabelled model is light PERM[j]: its SG set, its light_line row and the ids that name it.  The
    maps must not move and every light gradient must come out permuted; two runs of one input bound both sides."""
    model, rays, li = lego[n_lights]
    n_s = model.nSamples
    args = renderer_args(96)
    perm = torch.tensor(PERMS[n_lights])
    inv = torch.argsort(perm)
    sgs, rows = _light_state(model)
    try:
        m0, _, g0 = step(model, rays, li, 7, is_relight, n_s, args)
        m1, _, g1 = step(model, rays, li, 7, is_relight, n_s, args)
        _set_lights(model, [sgs[int(j)] for j in perm], rows[perm.to(DEV)])
        m2, _, g2 = step(model, rays, inv.to(DEV)[li.long()].to(torch.int32), 7, is_relight, n_s, args)
    finally:
        _set_lights(model, sgs, rows)
    _check_maps(m1, m0, "repeat")
    _check_maps(m2, m0, "relabelled")
    sg = [f"lgtSGs_list.{k}" for k in range(n_lights)]
    assert set(g0) == set(g1) == set(g2)
    assert all((k in g0) == is_relight for k in sg)
    rest = [k for k in g0 if k not in sg and k != "light_line.weight"]
    noise = _max_errs(g1, g0, g0.keys())
    moved = _max_errs(g2, g0, rest)
    ll = g0["light_line.weight"]
    moved["light_line.weight"] = float((g2["light_line.weight"] - ll[perm.to(DEV)]).abs().max()) / float(ll.abs().max())
    if is_relight:
        scale = max(float(g0[k].abs().max()) for k in sg)
        for j in range(n_lights):
            moved[sg[j]] = float((g2[sg[j]] - g0[sg[int(perm[j])]]).abs().max()) / scale
    print(f"{n_lights} lights, relight {is_relight}: repeat {max(noise.values()):.2e}, relabelled "
          f"{max(moved.values()):.2e} ({max(moved, key=moved.get)})")
    assert max(noise.values()) <= GRAD_TOL, noise
    bad = {k: v for k, v in moved.items() if v > GRAD_TOL}
    assert not bad, bad


@pytest.mark.parametrize("is_relight", [True, False], ids=["relight", "phase1"])
@pytest.mark.parametrize("n_lights", sorted(PERMS))
def test_identical_lights_make_light_ids_irrelevant(lego, n_lights, is_relight):
    """Every SG set and light_line row equal to light 0's: the mixed-id step renders and trains what the all-zero-id step
    does.  The light gradients split over the lights of the batch: summed over the lights they equal the all-zero
    step's.  (The all-zero step's SG sets 1.. get exactly nothing; its light_line rows 1.. do get the intrinsic
    feature's share in a relight step, which reads the mean of all rows, so the rows are compared summed on both
    sides.)"""
    model, rays, li = lego[n_lights]
    n_s = model.nSamples
    args = renderer_args(96)
    sgs, rows = _light_state(model)
    try:
        _set_lights(model, [sgs[0]] * n_lights, rows[:1].expand(n_lights, -1))
        mm, _, gm = step(model, rays, li, 8, is_relight, n_s, args)
        mz, _, gz = step(model, rays, torch.zeros_like(li), 8, is_relight, n_s, args)
        mr, _, gr = step(model, rays, torch.zeros_like(li), 8, is_relight, n_s, args)
    finally:
        _set_lights(model, sgs, rows)
    _check_maps(mr, mz, "repeat")
    _check_maps(mm, mz, "mixed ids")
    sg = [f"lgtSGs_list.{k}" for k in range(n_lights)]
    rest = [k for k in gz if k not in sg and k != "light_line.weight"]
    noise = _max_errs(gr, gz, gz.keys())
    diff = _max_errs(gm, gz, rest)
    zr = gz["light_line.weight"]
    diff["light_line rows summed"] = rel_err(gm["light_line.weight"].sum(0), zr.sum(0))
    if not is_relight:
        assert float(zr[1:].abs().max()) == 0.0                       # phase 1: only each ray's own row
    if is_relight:
        for k in sg[1:]:
            assert float(gz[k].abs().max()) == 0.0, k
        diff["SG sets summed"] = rel_err(sum(gm[k] for k in sg), gz[sg[0]])
        assert all(float(gm[k].abs().max()) > 0 for k in sg)         # every light of the batch got its share
    print(f"{n_lights} lights, relight {is_relight}: repeat {max(noise.values()):.2e}, mixed vs zero "
          f"{max(diff.values()):.2e} ({max(diff, key=diff.get)})")
    assert max(noise.values()) <= GRAD_TOL, noise
    bad = {k: v for k, v in diff.items() if v > GRAD_TOL}
    assert not bad, bad


# --------------------------------------------------------------------------------------------------- graph replays
class RecordingSGD(torch.optim.Optimizer):
    """Capturable plain SGD that keeps a copy of every gradient it applies: the copies of a replayed step are that
    step's gradients.  ``clear_grad``: gradients are zeroed in place after the update (StaticTrainStep then keeps the
    gradient buffers of the first warm-up step); ``found_inf`` (a 0-dim device tensor set by StaticTrainStep) turns the
    update into a no-op."""
    clear_grad = True

    def __init__(self, params, lrs):
        super().__init__([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], {})
        self.found_inf = None
        self.record = {p: torch.zeros_like(p) for p in params}

    @torch.no_grad()
    def step(self):
        keep = 1.0 - self.found_inf
        for grp in self.param_groups:
            for p in grp["params"]:
                if p.grad is None:
                    continue
                self.record[p].copy_(p.grad)
                p.sub_(p.grad * keep * grp["lr"])
                p.grad.zero_()


@pytest.mark.parametrize("is_relight", [True, False], ids=["relight", "phase1"])
def test_graph_replays_equal_eager_steps(lego, is_relight):
    """Four replays back to back (mixed ids, all light 2, lights 0 and 1 only, a new mixed batch), each against the eager
    step from the parameters the replay started from, with the same host draws: loss and every recorded gradient, each
    SG set's included.  The update moves each parameter by 1 % of its largest entry per step, so a replay that read a
    stale light table or the previous batch's light ids would be far outside the bound."""
    from tensoir_b200.static_step import StaticTrainStep
    from tensoir_b200.synthetic import hemisphere_poses, training_batch
    model0, rays0, li0 = lego[3]
    with contextlib.redirect_stdout(io.StringIO()):
        from tensoir_b200.synthetic import make_lego_model
        model = make_lego_model(GRID, DEV, general=True, lights=["light0", "light1", "light2"])
        eager = make_lego_model(GRID, DEV, general=True, lights=["light0", "light1", "light2"])
    for m in (model, eager):
        m.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)
        _set_lights(m, *_light_state(model0))
    n_s = model.nSamples
    args = renderer_args(96)
    rays1, _ = training_batch(hemisphere_poses(100), N_RAYS, 2, n_lights=3)
    rays1 = rays1.to(DEV)
    batches = [(rays0, li0), (rays0, torch.full_like(li0, 2)), (rays1, (torch.arange(N_RAYS, device=DEV) % 2).view(-1, 1)
                                                                 .to(torch.int32)), (rays1, li0)]
    params = all_params(model)
    names = list(params)
    # per-parameter learning rate from one eager step: each update moves a parameter by 1 % of its largest entry
    _, _, g = step(model, rays0, li0, 1, is_relight, n_s, args)
    lrs = [0.01 * float(params[k].detach().abs().max()) / float(g[k].abs().max()) if k in g and float(g[k].abs().max()) > 0
           else 0.0 for k in names]
    for p in params.values():
        p.grad = None
    opt = RecordingSGD([params[k] for k in names], lrs)
    st = StaticTrainStep(model, opt, N_RAYS, n_s, args, lambda ret, mm: train_loss(ret, is_relight), device=DEV,
                         is_relight=is_relight)
    st.calibrate(batches)
    st.capture(warmup=2)
    start = {k: p.detach().clone() for k, p in params.items()}
    worst = {}
    try:
        for b, (rays, li) in enumerate(batches):
            before = {k: p.detach().clone() for k, p in params.items()}
            loss = float(st.run(rays, li, seed=100 + b))
            torch.cuda.synchronize()
            rec = {k: opt.record[params[k]].clone() for k in names if params[k].grad is not None}
            with torch.no_grad():
                for k, p in all_params(eager).items():
                    p.copy_(before[k])
            _, want_loss, want = step(eager, rays, li, 100 + b, is_relight, n_s, args)
            assert set(rec) == set(want), set(rec) ^ set(want)
            assert abs(loss - float(want_loss)) <= 1e-5 * abs(float(want_loss)), (b, loss, float(want_loss))
            errs = {k: rel_err(rec[k], want[k]) for k in want if float(want[k].abs().max()) > 0}
            for k in want:
                if float(want[k].abs().max()) == 0:
                    assert float(rec[k].abs().max()) == 0.0, (b, k)
            if is_relight:
                ids = set(li.view(-1).tolist())
                for k in range(3):
                    nz = float(rec[f"lgtSGs_list.{k}"].abs().max()) > 0
                    assert nz == (k in ids), (b, k, ids)
            worst[b] = max(errs.items(), key=lambda kv: kv[1])
            bad = {k: v for k, v in errs.items() if v > GRAD_TOL}
            assert not bad, (b, bad)
        st.flush()
        assert st.redone == 0 and st.recaptures == 0 and st.overflowed() == 0
    finally:
        st.release()
    moved = max(float((params[k].detach() - start[k]).abs().max()) / max(float(start[k].abs().max()), 1e-30) for k in names)
    print(f"relight {is_relight}: worst recorded gradient err / max per replay {worst}, parameters moved up to "
          f"{moved:.2e} of their max")
    assert moved > 0.02
