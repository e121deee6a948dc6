"""The native trainer (tensoir_b200.train.reconstruction) on the shrunk armadillo schedule recorded from the reference
(tests/golden/schedule_shrunk.pt: 400 iterations, four upsamples, six mask updates, both phases), trained on synthetic
lego views from the lego-density checkpoint, once graphed and once eagerly on the same batches."""
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


def _args(tmp, ckpt):
    fx = torch.load(os.path.join(HERE, "golden", "schedule_shrunk.pt"), weights_only=False)
    a = types.SimpleNamespace(**fx["config"])
    a.expname, a.ckpt, a.config = "lego", ckpt, None
    a.N_vis = 2
    return a, fx


def _psnr(model, views, n_samples):
    from tensoir_b200 import Renderer_TensoIR_train
    out = []
    with torch.no_grad():
        for i in range(len(views)):
            item = views[i]
            ret = Renderer_TensoIR_train(item['rays'].to(DEV), None, item['light_idx'][0].to(DEV), model,
                                         N_samples=n_samples, white_bg=True, is_train=False, is_relight=False,
                                         device=DEV)
            mse = torch.mean((ret['rgb_map'] - item['rgbs'][0].to(DEV)) ** 2)
            out.append(float(-10 * torch.log10(mse)))
    return float(np.mean(out))


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import train
    from tensoir_b200.static_step import StaticTrainStep
    from tensoir_b200.synthetic import SyntheticTrainViews, SyntheticViews, hemisphere_poses, make_lego_model
    tmp = tmp_path_factory.mktemp("train")
    poses = hemisphere_poses(14)
    train_views = SyntheticTrainViews(poses[:12], 64, 64)
    test_views = SyntheticViews(poses[12:], 32, 32)
    ckpt = str(tmp / "start.th")
    m = make_lego_model(64, DEV)
    m.alphaMask = None
    # a mask threshold well above what the empty space can reach in 50 steps, so the aabb that the first mask update
    # finds comes from the box faces, not from faint floaters whose alpha differs between the two runs by atomics order
    m.alphaMask_thres = 0.05
    m.save(ckpt)

    class Model(train.TensorVMSplit):
        """Deterministic xyz noise of the smoothness terms, so that the padded device draw of the graphed step and
        the eager draw agree."""
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)

    orig_model, orig_run = train.TensorVMSplit, StaticTrainStep.run
    readback = []

    def run(self, *a, **k):
        loss = orig_run(self, *a, **k)
        readback.append(float(loss))          # a per-step host readback of the same replay
        return loss

    out = {}
    train.TensorVMSplit = Model
    try:
        for graphed in (True, False):
            args, fx = _args(tmp, ckpt)
            log = str(tmp / ("graphed" if graphed else "eager"))
            np.random.seed(20211202)
            StaticTrainStep.run = run if graphed else orig_run
            res = train.reconstruction(args, train_views, test_views, log, graphed=graphed, device=DEV,
                                       out=open(os.devnull, "w"))
            res["log"] = log
            out[graphed] = res
    finally:
        train.TensorVMSplit, StaticTrainStep.run = orig_model, orig_run
    start = train.TensorVMSplit(**torch.load(ckpt, map_location=DEV, weights_only=False)["kwargs"] | {"device": DEV})
    start.load(torch.load(ckpt, map_location=DEV, weights_only=False))
    return {"graphed": out[True], "eager": out[False], "readback": readback, "fx": fx, "test_views": test_views,
            "start": start, "args": args}


def test_graphed_and_eager_runs_make_the_same_events(runs):
    g, e = runs["graphed"], runs["eager"]
    assert g["events"] == e["events"]
    kinds = [ev[1] for ev in g["events"]]
    for k in ("updateAlphaMask", "shrink", "filtering_rays", "upsample_volume_grid", "save", "evaluation"):
        assert k in kinds
    # the iterations and names of the reference's schedule (resolutions depend on the trained aabb)
    want = [(ev[0], ev[1]) for ev in runs["fx"]["events"] if ev[0] >= 0 and ev[1] != "optimizer"]
    assert [(ev[0], ev[1]) for ev in g["events"]] == want


def test_graphed_losses_track_eager_for_the_first_50_iterations_of_each_phase(runs):
    """Per-iteration total loss over the first 50 iterations of each phase, each window cut at the next mask update: a
    mask update thresholds the trained density, and two runs whose densities differ by atomics order can flip a few
    voxels of the new mask near the threshold, after which they march different sample sets (here the phase-2 window
    ends at the mask update at 75).  Phase 1 starts both runs from one checkpoint and holds the 2e-3 of the 50-step
    graph-replay parity test.  Phase 2 starts from models that already differ by 51 steps of atomics-order noise, which
    Adam turns into parameter steps of up to ~lr: its losses start ~1e-3 apart and drift apart (6e-3 after 20 steps
    on an H100), so it is held to 1e-2."""
    g, e = runs["graphed"], runs["eager"]
    lg, le = g["losses"][:, 0], e["losses"][:, 0]
    assert torch.isfinite(lg).all() and torch.isfinite(le).all()
    masks = [ev[0] for ev in g["events"] if ev[1] == "updateAlphaMask"]
    first2 = int(np.argmax(g["relight"]))
    for lo, tol in ((0, 2e-3), (first2, 1e-2)):
        hi = min([lo + 50] + [m + 1 for m in masks if m >= lo])
        rel = ((lg[lo:hi] - le[lo:hi]).abs() / le[lo:hi].abs().clamp_min(1e-6))
        k = lo + int(rel.argmax())
        assert float(rel.max()) < tol, (lo, hi, float(rel.max()), k, g["losses"][k].tolist(), e["losses"][k].tolist())
    assert first2 >= 50                      # phase 1 is compared over a full 50 iterations
    assert g["redone"] == 0, g["redone"]     # an overflow would be redone; none is expected at this size


def test_device_ring_equals_per_step_readback(runs):
    got = runs["graphed"]["losses"][:, 0].tolist()
    assert got == [float(np.float32(v)) for v in runs["readback"]]


def test_held_out_psnr_rises_by_more_than_3_db(runs):
    n_s = runs["graphed"]["model"].nSamples
    before = _psnr(runs["start"], runs["test_views"], n_s)
    for key in ("graphed", "eager"):
        after = _psnr(runs[key]["model"], runs["test_views"], n_s)
        assert after - before > 3.0, (key, before, after)


def test_final_checkpoint_renders_like_the_trained_model(runs):
    from tensoir_b200 import Renderer_TensoIR_train
    from tensoir_b200.tensorf import TensorVMSplit
    res, args = runs["graphed"], runs["args"]
    ckpt = torch.load(os.path.join(res["log"], f"{args.expname}.th"), map_location=DEV, weights_only=False)
    kw = dict(ckpt["kwargs"], device=DEV)
    fresh = TensorVMSplit(**kw)
    fresh.load(ckpt)
    item = runs["test_views"][0]
    maps = []
    for m in (res["model"], fresh):
        with torch.no_grad():
            maps.append(Renderer_TensoIR_train(item['rays'].to(DEV), None, item['light_idx'][0].to(DEV), m,
                                               N_samples=-1, white_bg=True, is_train=False, is_relight=True,
                                               sample_method='fixed_envirmap', device=DEV, args=args))
    for k in ("rgb_map", "rgb_with_brdf_map", "depth_map", "normal_map", "albedo_map", "roughness_map"):
        assert float((maps[0][k] - maps[1][k]).abs().max()) <= 1e-6, k


def test_output_folders_hold_the_reference_names(runs):
    res, args = runs["graphed"], runs["args"]
    log = res["log"]
    assert os.path.isfile(os.path.join(log, f"{args.expname}.th"))
    saves = [ev[2] for ev in res["events"] if ev[1] == "save"]
    for name in saves:
        assert os.path.isfile(os.path.join(log, name)), name
    assert f"checkpoints/{args.expname}_0.th" in saves
    for ev in res["events"]:
        if ev[1] == "evaluation" and ev[2] == "imgs_vis":
            for sub in ("nvs_with_radiance_field", "nvs_with_brdf", "normal", "brdf", "acc_map"):
                assert os.path.isfile(os.path.join(log, "imgs_vis", sub, f"{ev[3]}000.png")), (ev, sub)
    assert os.listdir(os.path.join(log, "imgs_test_all"))
