"""The overflow redo of the graph-replayed training step, as the trainer drives it (tensoir_b200.train.reconstruction
with graphed=True): which replays apply, in what order, with which learning rates and loss weights, and what the loss
log keeps.

The run is the shrunk armadillo schedule of tests/golden/schedule_shrunk.pt cut to 130 iterations (lr_decay_iters kept,
so every iteration has its own learning rates): phase 1, the mask update with shrink and the upsample at 50, the first
relight capture at 51, evaluations at 74, 99 and 124, the mask updates at 75, 100 and 125, the upsample at 100, saves
at 0, 50 and 100.  It trains on synthetic lego views from the lego-density checkpoint, with the deterministic xyz
noise of tests/test_train_gpu.py.

A test-local StaticTrainStep re-captures with lists far below the real lengths right before the replays in FORCED, and
back at the trainer's sizes right after, with the steps in flight kept.  Each forced replay overflows; the step's own
grow logic then recovers.  After every replay it records the replay's iteration (its seed - train.SEED), found_inf,
the trainer's scalar vector (the device vector behind the optimizer's learning rates: every rate, then the TV density,
TV appearance, normal and BRDF weights) and the loss-term vector.  Its release(), which the trainer calls right after
flush(), records every FusedAdam step count, and at the first release (the end of phase 1) the parameters and both
Adam moments.
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_ITERS = 130
FORCED_CAPS = (1024, 256)     # valid / appearance lists: a 4096-ray batch has several times more valid samples
# forced iteration -> (what it covers, steps redone).  An overflow makes its own replay and every replay launched after
# it no-ops until the host settles it, re-captures and redoes them all in order.  The trainer settles a step when its
# slot comes round again three launches later, or earlier at a flush: every read of the loss ring (each 10th iteration
# and at each event, so at 0 and 50 too), an evaluation, a save, a grid event.
FORCED = {
    0: ("first replay of phase 1, flushed at 0", 1),
    23: ("mid-phase, 24 and 25 in flight behind it, settled when 26 reuses its slot", 3),
    # 31 and 32 come right after the flush at 30, so no step launched on the normal lists is settled (and judged
    # against the forced ones) between them
    31: ("first of two consecutive overflows, settled at 34 with 32 and 33", 3),
    32: ("second of two consecutive overflows, redone with 31", 0),
    49: ("pending at the grid event of 50, redone with 50", 2),
    51: ("first replay of phase 2, the first relight capture, redone with 52 and 53", 3),
    73: ("pending when the evaluation at 74 flushes, redone with 74", 2),
}
RECAPTURES = 6                # one grow per group of overflows: {0}, {23}, {31, 32}, {49}, {51}, {73}


def _args(ckpt, n_iters):
    fx = torch.load(os.path.join(HERE, "golden", "schedule_shrunk.pt"), weights_only=False)
    a = types.SimpleNamespace(**fx["config"])
    a.expname, a.ckpt, a.config = "lego", ckpt, None
    a.N_vis = 2
    a.n_iters = n_iters
    a.render_test = 0
    return a


def _train(tmp, name, ckpt, views, n_iters, forced):
    from tensoir_b200 import train
    from tensoir_b200.primary_fused import Workspace
    from tensoir_b200.static_step import StaticTrainStep

    run = {"trace": [], "weights": {}, "adam": [], "snapshot": None, "opts": 0}
    holder = {}

    class Model(train.TensorVMSplit):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)

    class Schedule(train.TrainSchedule):
        def begin(self, it):
            w = super().begin(it)
            run["weights"][it] = w
            return w

    orig_loss = train._loss

    def loss(*a):
        holder["terms"] = a[-1]                    # the trainer's terms list: terms[0] is the captured vector
        return orig_loss(*a)

    class Step(StaticTrainStep):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            if not hasattr(self.opt, "_redo_test_serial"):
                self.opt._redo_test_serial = run["opts"]
                run["opts"] += 1
            self._home = None                      # the trainer's capacities
            self._normal = None                    # capacities to go back to while a forced capture is in place

        def _capture_keeping(self, caps):
            """Re-capture at ``caps`` with the steps in flight kept: their slots, the skip flag, the overflow count."""
            torch.cuda.synchronize()
            kept = [(s["event"], s["batch"]) for s in self._slots]
            skip, over = self.found_inf.clone(), self.static["overflow"].clone()
            # the primary march's workspace only ever grows: drop it, so that the capture allocates lists of ``caps``
            for key in [k for k, v in self.model.__dict__.items() if isinstance(v, Workspace)]:
                del self.model.__dict__[key]
            self._set_caps(*caps)
            self.capture(warmup=1)
            for s, (ev, b) in zip(self._slots, kept):
                s["event"], s["batch"] = ev, b
            self.found_inf.copy_(skip)
            self.static["overflow"].copy_(over)

        def run(self, rays, light_idx, target=None, seed=None, *rest, **kw):
            it = seed - train.SEED
            if self._home is None:
                self._home = self.capacities()
            if it in forced:
                if self._normal is None:
                    # settle the step whose slot this run reuses first, as run() would: a step launched on the normal
                    # lists must not be judged against the forced ones (its high-water mark would grow them back)
                    self._settle(self._slots[self._step % len(self._slots)])
                    self._normal = self.capacities()
                    self._capture_keeping(FORCED_CAPS)
            elif self._normal is not None:
                normal, self._normal = self._normal, None
                self._capture_keeping(normal)
            return super().run(rays, light_idx, target, seed, *rest, **kw)

        def _recapture(self, caps):
            # the grow after a forced overflow goes back to at least the trainer's lists, so that the rest of the phase
            # runs on the lists an undisturbed run has; the forced shrinks are not growth that could fail to converge
            self._normal = None
            self.__dict__.pop("_last_grow", None)
            super()._recapture(tuple(max(c, h) for c, h in zip(caps, self._home)))

        def _launch(self, *a, **k):
            super()._launch(*a, **k)
            scal = self.opt.param_groups[0]["lr"]._base          # the learning rates are views of the trainer's vector
            run["trace"].append((torch.initial_seed() - train.SEED, self.opt._redo_test_serial, self.found_inf.clone(),
                                 scal.clone(), holder["terms"][0].clone()))

        def release(self):
            torch.cuda.synchronize()
            last = max(r[0] for r in run["trace"])
            run["adam"].append((last, self.opt._redo_test_serial,
                                [int(s["step"].item()) for s in self.opt.state.values()]))
            if run["snapshot"] is None:
                run["snapshot"] = [(p.detach().clone(), s["exp_avg"].clone(), s["exp_avg_sq"].clone())
                                   for g in self.opt.param_groups for p in g["params"]
                                   for s in [self.opt.state.get(p)] if s]
            super().release()

    args = _args(ckpt, n_iters)
    np.random.seed(train.SEED)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(train, "TensorVMSplit", Model)
        mp.setattr(train, "TrainSchedule", Schedule)
        mp.setattr(train, "_loss", loss)
        mp.setattr(train, "StaticTrainStep", Step)
        with open(os.devnull, "w") as out:
            res = train.reconstruction(args, views[0], views[1], str(tmp / name), graphed=True, device=DEV, out=out)
    run["trace"] = [(it, serial, float(fi), scal.cpu(), terms.cpu()) for it, serial, fi, scal, terms in run["trace"]]
    run["res"] = res
    return run


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    import __graft_entry__ as g
    g.build()
    from tensoir_b200.synthetic import SyntheticTrainViews, SyntheticViews, hemisphere_poses, make_lego_model
    tmp = tmp_path_factory.mktemp("redo")
    poses = hemisphere_poses(14)
    views = (SyntheticTrainViews(poses[:12], 64, 64), SyntheticViews(poses[12:], 32, 32))
    ckpt = str(tmp / "start.th")
    m = make_lego_model(64, DEV)
    m.alphaMask = None
    m.alphaMask_thres = 0.05            # as tests/test_train_gpu.py: the first mask's aabb comes from the box faces
    m.save(ckpt)
    forced = _train(tmp, "forced", ckpt, views, N_ITERS, set(FORCED))
    # the undisturbed runs stop after the grid event at 50: their phase 1 is the forced run's (same batches, seeds,
    # learning rates and TV weights; lr_decay_iters fixes the decay)
    calm = [_train(tmp, f"calm{k}", ckpt, views, 51, set()) for k in range(3)]
    return {"forced": forced, "calm": calm}


def _applied(run):
    return [row for row in run["trace"] if row[2] == 0.0]


def test_the_run_has_the_events_the_checks_need(runs):
    res = runs["forced"]["res"]
    kinds = {(ev[0], ev[1]) for ev in res["events"]}
    for want in ((0, "save"), (50, "shrink"), (50, "upsample_volume_grid"), (74, "evaluation"), (75, "updateAlphaMask"),
                 (100, "upsample_volume_grid")):
        assert want in kinds, want
    assert not res["relight"][50] and res["relight"][51]
    first = {}
    for it, _, fi, _, _ in runs["forced"]["trace"]:
        first.setdefault(it, fi)
    assert set(FORCED) <= {it for it, fi in first.items() if fi != 0.0}    # every forced replay was a no-op


def test_applied_replays_are_every_iteration_once_in_order(runs):
    got = [row[0] for row in _applied(runs["forced"])]
    assert got == list(range(N_ITERS)), [(k, it) for k, it in enumerate(got) if k != it][:8]


def test_each_applied_replay_reads_its_own_iterations_scalars(runs):
    run = runs["forced"]
    bad = []
    for it, _, _, scal, _ in _applied(run):
        w = run["weights"][it]
        want = torch.tensor([np.float32(v) for v in list(w.lrs) + [w.tv_density, w.tv_app, w.normal_factor,
                                                                   w.brdf_factor]], dtype=torch.float32)
        if scal.shape != want.shape or not torch.equal(scal.view(torch.int32), want.view(torch.int32)):
            bad.append((it, scal.tolist(), want.tolist()))
    assert not bad, bad[:3]


def test_adam_step_counts_equal_the_applied_iterations_at_every_retire(runs):
    run = runs["forced"]
    assert len(run["adam"]) >= 6
    for last, serial, steps in run["adam"]:
        want = len({it for it, s, _, _, _ in run["trace"] if s == serial and it <= last})
        assert steps and set(steps) == {want}, (last, serial, sorted(set(steps)), want)


def test_loss_ring_holds_every_iterations_applied_replay(runs):
    run = runs["forced"]
    losses = run["res"]["losses"]
    bad = [(it, losses[it].tolist(), terms.tolist()) for it, _, _, _, terms in _applied(run)
           if not torch.equal(losses[it], terms)]
    assert not bad, bad[:3]


def test_forced_overflows_leave_phase_1_as_an_undisturbed_run(runs):
    """Parameters and both Adam moments at the end of phase 1 (the retire at 50): the forced run against an undisturbed
    one, within 4x the largest spread of three undisturbed runs (atomics order, amplified by 50 Adam steps) plus 1e-6 of
    the tensor's largest value.  Applying a forced step after the two behind it, or with their learning rates, moves
    the end of phase 1 by thousands of times that."""
    f = runs["forced"]["snapshot"]
    calm = [c["snapshot"] for c in runs["calm"]]
    assert len(f) > 0 and all(len(c) == len(f) for c in calm)
    worst, ratio = [], (0.0, None)
    for k in range(len(f)):
        for j, name in enumerate(("param", "exp_avg", "exp_avg_sq")):
            a, ref = f[k][j], [c[k][j] for c in calm]
            assert all(r.shape == a.shape for r in ref), (k, name)
            spread = max(float((ref[u] - ref[v]).abs().max()) for u in range(3) for v in range(u))
            diff = float((a - ref[0]).abs().max())
            tol = 4 * spread + 1e-6 * float(ref[0].abs().max())
            if diff > tol:
                worst.append((k, name, tuple(a.shape), diff, spread, tol))
            ratio = max(ratio, (diff / tol, (k, name, tuple(a.shape))), key=lambda r: r[0])
    print(f"largest difference from an undisturbed run: {ratio[0]:.3f} of the tolerance, at {ratio[1]}")
    assert not worst, worst[:6]


def test_redo_and_recapture_counts(runs):
    res = runs["forced"]["res"]
    assert res["redone"] == sum(n for _, n in FORCED.values()), res["redone"]
    assert res["recaptures"] == RECAPTURES, res["recaptures"]
    for calm in runs["calm"]:
        assert calm["res"]["redone"] == 0 and calm["res"]["recaptures"] == 0
