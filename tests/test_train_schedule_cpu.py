"""TrainSchedule against the reference's own train_tensoIR.py schedule, recorded on the CPU by
tests/golden/make_schedule_golden.py (configs/single_light/armadillo.txt at 80 000 iterations, and the same config
shrunk to 400), plus the sampler and the trainer's up-front rejections."""
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from tensoir_b200.schedule import MaskUpdate, SimpleSampler, TrainSchedule  # noqa: E402


def _fixture(name):
    return torch.load(os.path.join(HERE, "golden", f"schedule_{name}.pt"), weights_only=False)


def _replay(fx):
    """Drive TrainSchedule the way the trainer does, against a model that behaves like the recording one (shrink takes
    the fixture's box as the new aabb); -> (events in the fixture's format, per-iteration columns)."""
    args = types.SimpleNamespace(**fx["config"])
    aabb = fx["initial_aabb"].clone()
    sched = TrainSchedule(args, aabb, lambda lr, lr_basis: [lr, lr_basis, 0.001])
    events = [(-1, "init", list(sched.reso_cur)), (-1, "get_optparam_groups", args.lr_init, args.lr_basis),
              (-1, "optimizer"), (-1, "filtering_rays", True)]
    rows = []
    for it in range(args.n_iters):
        w = sched.begin(it)
        rows.append(list(w.lrs) + [w.tv_density, w.tv_app, w.l1,
                                   w.normal_factor * args.normals_diff_weight if w.relight else 0.0,
                                   w.normal_factor * args.normals_orientation_weight if w.relight else 0.0,
                                   w.brdf_factor * args.roughness_smoothness_loss_weight if w.relight else 0.0,
                                   w.brdf_factor * args.albedo_smoothness_loss_weight if w.relight else 0.0,
                                   float(w.relight), float(w.n_samples)])
        end = sched.end(it)
        assert end.progress == (it % args.progress_refresh_rate == 0)
        if end.evaluate:
            events.append((it, "evaluation", "imgs_vis", f"{it:06d}_", int(w.n_samples), False, False))
        if end.save:
            events.append((it, "save", f"checkpoints/{args.expname}_{it}.th"))
        for ev in end.grid:
            if isinstance(ev, MaskUpdate):
                events.append((it, "updateAlphaMask", list(ev.reso)))
                if ev.shrink:
                    aabb = fx["new_aabb"].clone()
                    events.append((it, "shrink"))
                if ev.refilter:
                    events.append((it, "filtering_rays", True))
            else:
                events.append((it, "upsample_volume_grid", list(sched.upsample(ev, aabb))))
                events += [(it, "get_optparam_groups", ev.lr, ev.lr_basis), (it, "optimizer")]
    last = args.n_iters - 1
    events.append((last, "save", f"{args.expname}.th"))
    if args.render_test:
        events.append((last, "evaluation", "imgs_test_all", "", -1, True, True))
    return events, np.asarray(rows, dtype=np.float64)


@pytest.mark.parametrize("name", ["shrunk", "armadillo"])
def test_schedule_reproduces_the_reference_events(name):
    """Grid events (order, resolutions on the shrunk aabb), optimizer creations with their learning rates, saves and
    evaluations (iteration, folder, prefix, nSamples) are the reference's, bit for bit."""
    fx = _fixture(name)
    events, _ = _replay(fx)
    assert events == fx["events"]


@pytest.mark.parametrize("name", ["shrunk", "armadillo"])
def test_schedule_reproduces_the_reference_per_iteration_values(name):
    """Every param group's learning rate, the TV / L1 / normal / BRDF weights, the relight flag and nSamples of every
    iteration equal the reference's in float64, bit for bit (the armadillo run is compared through a SHA-256 of each
    column, with samples around every event to show where a difference starts)."""
    fx = _fixture(name)
    _, cols = _replay(fx)
    if "per_iter" in fx:
        want = fx["per_iter"].numpy()
        assert cols.shape == want.shape
        for c, col in enumerate(fx["columns"]):
            bad = np.nonzero(cols[:, c] != want[:, c])[0]
            assert bad.size == 0, (col, int(bad[0]), cols[bad[0], c], want[bad[0], c])
        return
    keep = fx["sample_iters"].numpy()
    want = fx["samples"].numpy()
    for c, col in enumerate(fx["columns"]):
        bad = np.nonzero(cols[keep, c] != want[:, c])[0]
        assert bad.size == 0, (col, int(keep[bad[0]]), cols[keep[bad[0]], c], want[bad[0], c])
        digest = hashlib.sha256(np.ascontiguousarray(cols[:, c]).tobytes()).hexdigest()
        assert digest == fx["sha256"][c], col


def test_learning_rate_decay_is_one_multiplication_per_iteration():
    """Rounding matters at 80 000 iterations: the reference multiplies each group's rate by lr_factor once per
    iteration; a closed form lr0 * f**k differs from it in the last bits."""
    fx = _fixture("armadillo")
    args = types.SimpleNamespace(**fx["config"])
    sched = TrainSchedule(args, fx["initial_aabb"], lambda lr, lr_basis: [lr, lr_basis, 0.001])
    lrs = []
    for it in range(9999):
        lrs.append(sched.begin(it).lrs[0])
        sched.end(it)
    closed = [args.lr_init * sched.lr_factor ** k for k in range(9999)]
    assert lrs != closed
    want = fx["samples"].numpy()[:, 0]
    keep = fx["sample_iters"].numpy()
    assert [lrs[i] for i in keep if i < 9999] == [want[j] for j, i in enumerate(keep) if i < 9999]


def test_sampler_matches_the_reference_ids():
    """The first 3 epochs of ray ids under the scripts' numpy seed are the ones the reference's sampler drew."""
    fx = _fixture("shrunk")
    np.random.seed(20211202)
    s = SimpleSampler(fx["n_rays"], fx["config"]["batch_size"])
    got = torch.stack([s.nextids() for _ in range(fx["ids"].shape[0])])
    assert torch.equal(got, fx["ids"].long())


def _args(**kw):
    a = types.SimpleNamespace(**_fixture("shrunk")["config"])
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("change, message", [
    (dict(ndc_ray=1), "ndc_ray"),
    (dict(model_name="TensorCP"), "TensorVMSplit"),
    (dict(shadingMode="MLP_PE"), "MLP_Fea"),
    (dict(update_AlphaMask_list=[400, 500]), "before n_iters"),
    (dict(update_AlphaMask_list=None), "before n_iters"),
])
def test_reconstruction_rejects_what_it_does_not_run(change, message, tmp_path):
    from tensoir_b200.train import reconstruction
    with pytest.raises(ValueError, match=message):
        reconstruction(_args(**change), None, None, str(tmp_path))
    assert not os.listdir(tmp_path)              # rejected before anything is written


def test_schedule_needs_a_mask_resolution():
    """The reference only sets reso_mask from a grid under 256^3 voxels: a first mask update above that is an error
    (a NameError in the reference), reported clearly here."""
    a = _args(N_voxel_init=300 ** 3)
    sched = TrainSchedule(a, _fixture("shrunk")["initial_aabb"], lambda lr, lr_basis: [lr, lr_basis])
    with pytest.raises(ValueError, match="256"):
        for it in range(a.update_AlphaMask_list[0] + 1):
            sched.begin(it)
            sched.end(it)
