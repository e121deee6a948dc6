"""The native trainer's general multi-light and simple variants (tensoir_b200.train, variant="general" / "simple") on the
shrunk armadillo schedule of tests/golden/schedule_shrunk.pt and synthetic lego views, set up like test_train_gpu.py;
render_test and the entry scripts' mesh export on the checkpoints these runs write."""
import importlib.util
import os
import shutil
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 20211202
LIGHTS = ("sunset", "snow", "courtyard")
SUBDIRS = {"nvs_with_radiance_field", "nvs_with_brdf", "normal", "normal_vis", "brdf", "envir_map", "acc_map"}


def _args(ckpt, **kw):
    fx = torch.load(os.path.join(HERE, "golden", "schedule_shrunk.pt"), weights_only=False)
    a = types.SimpleNamespace(**fx["config"])
    a.expname, a.ckpt, a.config = "lego", ckpt, None
    a.N_vis = 2
    for k, v in kw.items():
        setattr(a, k, v)
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


def _load(path):
    from tensoir_b200.tensorf import TensorVMSplit
    ckpt = torch.load(path, map_location=DEV, weights_only=False)
    m = TensorVMSplit(**(ckpt["kwargs"] | {"device": DEV}))
    m.load(ckpt)
    return m


class _Writer:
    """SummaryWriter stand-in that keeps the scalar tags."""
    def __init__(self, tags):
        self.tags = tags

    def add_scalar(self, tag, *a, **k):
        self.tags.append(tag)

    def add_image(self, *a, **k):
        pass

    def close(self):
        pass


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import train
    from tensoir_b200.synthetic import SyntheticTrainViews, SyntheticViews, hemisphere_poses, make_lego_model
    tmp = tmp_path_factory.mktemp("train_variants")
    poses = hemisphere_poses(14)
    starts = {}
    for name, general in (("general", True), ("simple", False)):
        m = make_lego_model(64, DEV, general=general, lights=LIGHTS if general else ("000",))
        m.alphaMask = None
        m.alphaMask_thres = 0.05              # as in test_train_gpu.py: the first mask update's aabb from the box faces
        starts[name] = str(tmp / f"start_{name}.th")
        m.save(starts[name])
    data = {"general": (SyntheticTrainViews(poses[:12], 64, 64, n_lights=3), SyntheticViews(poses[12:], 32, 32,
                                                                                            n_lights=3)),
            "simple": (SyntheticTrainViews(poses[:12], 64, 64), SyntheticViews(poses[12:], 32, 32))}
    del data["simple"][0].all_masks          # the simple script's datasets need not have masks

    class Model(train.TensorVMSplit):
        """Deterministic xyz noise of the smoothness terms (test_train_gpu.py)."""
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)

    drawn = []

    class Sampler(train.SimpleSampler):
        def nextids(self):
            ids = super().nextids()
            drawn.append((self.total, ids.clone()))
            return ids

    tags = []
    orig = train.TensorVMSplit, train.SimpleSampler, train._summary_writer
    out = {}
    train.TensorVMSplit, train.SimpleSampler = Model, Sampler
    try:
        for key, variant, graphed in (("general", "general", True), ("general_eager", "general", False),
                                      ("simple", "simple", True)):
            kw = {"light_name_list": list(LIGHTS)} if variant == "general" else {}
            args, fx = _args(starts[variant], **kw)
            log = str(tmp / key)
            drawn.clear()
            tags.clear()
            train._summary_writer = (lambda _: _Writer(tags)) if variant == "simple" else orig[2]
            np.random.seed(SEED)
            res = train.reconstruction(args, *data[variant], log, variant=variant, graphed=graphed, device=DEV,
                                       out=open(os.devnull, "w"))
            res.update(log=log, args=args, drawn=list(drawn), tags=list(tags))
            out[key] = res
    finally:
        train.TensorVMSplit, train.SimpleSampler, train._summary_writer = orig
    out.update(fx=fx, starts=starts, data=data, tmp=tmp)
    return out


def _schedule(fx):
    return [(ev[0], ev[1]) for ev in fx["events"] if ev[0] >= 0 and ev[1] != "optimizer"]


def test_general_graphed_and_eager_make_the_schedules_events(runs):
    g, e = runs["general"], runs["general_eager"]
    assert g["events"] == e["events"]
    assert [(ev[0], ev[1]) for ev in g["events"]] == _schedule(runs["fx"])


def test_general_graphed_losses_track_eager(runs):
    """The windows of test_train_gpu.py's test_graphed_losses_track_eager_for_the_first_50_iterations_of_each_phase.

    Phase 1 holds its 2e-3.  The first relight iteration is held to 5e-3: its loss is the captured relight forward on
    models that differ only by phase 1's noise, so a ray lit or shaded with the wrong light would show there at once
    (measured on an H100: 1.6e-3).  The rest of the phase-2 window is held to 5e-2, not 1e-2.  What differs between
    two runs is the float atomics order of the gradient scatters: two eager backwards of one batch from one state
    differ by at most 5e-6 of each gradient's max, in every parameter, by the same amount with mixed and with all-zero
    light ids and for a single-light model (test_general_gradients_vary_only_by_atomics_order).  The three-light run's
    relight phase grows that noise much further than the single-light run: over this window two eager runs differ by
    up to 2.0e-2 and two graphed runs by 1.7e-2 (single light: 3e-5 and 5e-4); the graphed-eager gap measured 1.7e-2
    and 2.9e-2."""
    g, e = runs["general"], runs["general_eager"]
    lg, le = g["losses"][:, 0], e["losses"][:, 0]
    assert torch.isfinite(lg).all() and torch.isfinite(le).all()
    masks = [ev[0] for ev in g["events"] if ev[1] == "updateAlphaMask"]
    first2 = int(np.argmax(g["relight"]))
    assert first2 >= 50
    rel = lambda lo, hi: (lg[lo:hi] - le[lo:hi]).abs() / le[lo:hi].abs().clamp_min(1e-6)  # noqa: E731
    assert float(rel(first2, first2 + 1)[0]) < 5e-3, (g["losses"][first2].tolist(), e["losses"][first2].tolist())
    for lo, tol in ((0, 2e-3), (first2, 5e-2)):
        hi = min([lo + 50] + [m + 1 for m in masks if m >= lo])
        r = rel(lo, hi)
        k = lo + int(r.argmax())
        assert float(r.max()) < tol, (lo, hi, float(r.max()), k, g["losses"][k].tolist(), e["losses"][k].tolist())
    assert g["redone"] == 0, g["redone"]


def test_general_gradients_vary_only_by_atomics_order(runs):
    """Eager backwards of one relight batch of the three-light model from one state: every gradient, the light_line
    rows and each light's SG set included, repeats to within 1e-5 of its max (float atomics order), with the batch's
    mixed light ids as with all of them set to 0; and only the SG sets of the lights a batch holds get a gradient."""
    from tensoir_b200 import Renderer_TensoIR_train
    model = _load(runs["starts"]["general"])
    model.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)
    args = runs["general"]["args"]
    views = runs["data"]["general"][0]
    ids = torch.randint(0, views.all_rays.shape[0], (4096,), generator=torch.Generator().manual_seed(1))
    rays, rgb = views.all_rays[ids].to(DEV), views.all_rgbs[ids].to(DEV)
    li = views.all_light_idx[ids].to(torch.int32).to(DEV)
    params = dict(model.named_parameters()) | {f"lgtSGs_list.{k}": p for k, p in enumerate(model.lgtSGs_list)}

    def grads(light_idx):
        for p in params.values():
            p.grad = None
        torch.manual_seed(SEED)
        ret = Renderer_TensoIR_train(rays, None, light_idx, model, N_samples=model.nSamples, white_bg=True,
                                     device=DEV, sample_method=args.light_sample_train, is_train=True,
                                     is_relight=True, args=args)
        (torch.mean((ret['rgb_map'] - rgb) ** 2) + torch.mean((ret['rgb_with_brdf_map'] - rgb) ** 2)).backward()
        return {k: p.grad.detach().clone() for k, p in params.items() if p.grad is not None}

    for light_idx in (li, torch.zeros_like(li)):
        ref = grads(light_idx)
        for _ in range(3):
            got = grads(light_idx)
            assert got.keys() == ref.keys()
            for k in ref:
                err = float((got[k] - ref[k]).abs().max()) / max(float(ref[k].abs().max()), 1e-30)
                assert err < 1e-5, (k, err)
    with_sg = lambda g: sorted(k for k in g if k.startswith("lgtSGs_list") and float(g[k].abs().max()) > 0)  # noqa
    assert with_sg(grads(li)) == [f"lgtSGs_list.{k}" for k in range(len(LIGHTS))]
    assert with_sg(grads(torch.zeros_like(li))) == ["lgtSGs_list.0"]


def test_general_graphed_run_trains_every_light(runs):
    """Every light's SG set and light_line row moved: each ray's light index reached the captured step."""
    start, model = _load(runs["starts"]["general"]), runs["general"]["model"]
    assert len(model.lgtSGs_list) == len(LIGHTS)
    for k in range(len(LIGHTS)):
        assert float((model.lgtSGs_list[k].detach() - start.lgtSGs_list[k].detach()).abs().max()) > 1e-4, k
        row = model.light_line.weight.detach()[k] - start.light_line.weight.detach()[k]
        assert float(row.abs().max()) > 1e-4, k


def test_general_final_evaluation_runs_once_per_light(runs):
    from tensoir_b200 import Renderer_TensoIR_train, evaluation
    res = runs["general"]
    for name in LIGHTS:
        d = os.path.join(res["log"], "imgs_test_all", name)
        assert SUBDIRS <= set(os.listdir(d)), (name, os.listdir(d))
        assert os.path.isfile(os.path.join(d, "nvs_with_radiance_field", "000.png"))
    per_light = [np.mean(evaluation.evaluation_iter_TensoIR_general_multi_lights(
        runs["data"]["general"][1], res["model"], res["args"], Renderer_TensoIR_train, None, N_samples=-1,
        white_bg=True, ndc_ray=False, device=DEV, test_all=True, light_idx_to_test=l)[0]) for l in range(len(LIGHTS))]
    assert abs(res["psnr_test"] - float(np.mean(per_light))) <= 1e-4, (res["psnr_test"], per_light)


def test_general_sampler_shares_numpy_stream_with_evaluation_draws(runs):
    """A SimpleSampler replay that makes each in-training evaluation's np.random.randint(light_num) draws (one per
    evaluated view) after that iteration's batch draws the trained run's ids, across the new permutations drawn after
    the first evaluation."""
    from tensoir_b200.schedule import SimpleSampler
    res = runs["general"]
    evals = {ev[0] for ev in res["events"] if ev[1] == "evaluation" and ev[2] == "imgs_vis"}
    n_views = min(res["args"].N_vis, len(runs["data"]["general"][1]))
    first = min(evals)
    refilters = {ev[0] for ev in res["events"] if ev[1] == "filtering_rays"}
    np.random.seed(SEED)
    s, redrawn = None, 0
    for it, (total, ids) in enumerate(res["drawn"]):
        if it == 0 or it - 1 in refilters:        # the trainer's new sampler after each re-filter
            s = SimpleSampler(total, res["args"].batch_size)
        if it > first and s.curr + 2 * s.batch > s.total:
            redrawn += 1                          # this call draws a new permutation after the first evaluation
        assert torch.equal(s.nextids(), ids), it
        if it in evals:
            for _ in range(n_views):
                np.random.randint(len(LIGHTS))
    assert len(res["drawn"]) == res["args"].n_iters and redrawn > 0


def test_simple_run_follows_the_schedule_and_learns(runs):
    res = runs["simple"]
    assert [(ev[0], ev[1]) for ev in res["events"]] == _schedule(runs["fx"])
    assert res["redone"] == 0, res["redone"]
    views = runs["data"]["simple"][1]
    n_s = res["model"].nSamples
    before, after = _psnr(_load(runs["starts"]["simple"]), views, n_s), _psnr(res["model"], views, n_s)
    assert after - before > 3.0, (before, after)


def test_simple_run_writes_the_simple_outputs(runs):
    res = runs["simple"]
    d = os.path.join(res["log"], "imgs_test_all")
    assert set(os.listdir(d)) == SUBDIRS | {"metrics_record.txt"}, os.listdir(d)
    assert os.path.isfile(os.path.join(d, "brdf", "000_albedo.png"))
    assert "test/psnr_rgb_all" in res["tags"] and "test/psnr_rgb" in res["tags"]
    assert not [t for t in res["tags"] if t.startswith("test/") and ("albedo" in t or "mae" in t)], res["tags"]


@pytest.mark.parametrize("key,variant", [("general", "general"), ("simple", "simple")])
def test_render_test_of_the_final_checkpoint_matches_the_runs_final_evaluation(runs, key, variant, capsys):
    from tensoir_b200 import train
    res = runs[key]
    args, _ = _args(os.path.join(res["log"], "lego.th"), render_only=1, render_test=1,
                    light_name_list=list(LIGHTS) if variant == "general" else None)
    log = str(runs["tmp"] / f"test_{key}")
    r = train.render_test(args, runs["data"][variant][1], log, variant=variant, device=DEV)
    assert abs(float(r[0]) - res["psnr_test"]) <= 1e-4, (r[0], res["psnr_test"])
    printed = capsys.readouterr().out
    assert f"PSNRs_test: {r[0]}" in printed
    for line in (f"MAE_test: {r[2]}", f"PSNR_albedo_single: {r[3]}", f"PSNR_albedo_three: {r[4]}"):
        assert (line in printed) == (variant == "general"), (line, printed)
    want = [f for f in _files(os.path.join(res["log"], "imgs_test_all"))]
    assert _files(os.path.join(log, "imgs_test_all")) == want


def test_export_mesh_entry_writes_the_checkpoints_mesh_before_rendering(runs, monkeypatch):
    from tensoir_b200 import mesh, train
    res = runs["general"]
    ckpt = str(runs["tmp"] / "export" / "final.th")
    os.makedirs(os.path.dirname(ckpt))
    shutil.copy(os.path.join(res["log"], "lego.th"), ckpt)
    ply = ckpt[:-3] + ".ply"
    args, _ = _args(ckpt, export_mesh=1, render_only=1, render_test=1, light_name_list=list(LIGHTS),
                    basedir=str(runs["tmp"] / "export"), datadir="data", hdrdir="hdr")
    seen = []
    monkeypatch.setattr(train, "render_test", lambda *a, **k: seen.append(os.path.isfile(ply)))
    spec = importlib.util.spec_from_file_location(
        "tool_general", os.path.join(ROOT, "tools", "train_tensoIR_general_multi_lights.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    tool.main(args, lambda *a, **k: runs["data"]["general"][1], device=DEV)
    assert seen == [True]
    want = str(runs["tmp"] / "export" / "want.ply")
    mesh.export_mesh(_load(ckpt), want)
    assert open(ply, "rb").read() == open(want, "rb").read()
