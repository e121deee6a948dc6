"""Material editing on the H100: the tir_material_edit kernel against its host build, edited shading against
relight_chunk_fused on the fixture maps, a region edit on the lego scene, relight_edited end to end against relight(),
and the edited asset export.

The primary render composites with float atomics, and the visibility march's result for a sample can change in its last
bits with the sample's place in the visibility list, which an atomic append fills; so two runs of one chunk agree only
to those bits.  Where a test compares two runs, the forward and the visibility of the first run are replayed in the
second (relight_edited shares one visibility pass between its variants by construction)."""
import ctypes as C
import os
import re
import types

import cv2
import numpy as np
import pytest
import torch

from gpu_helpers import load_fixture, model_from_fixture
from helpers import build_host_lib
from test_material_edit_cpu import np_edit, random_rules

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def fx():
    import __graft_entry__ as g
    g.build()
    return load_fixture("rotated_g24.pt")


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_edit"), "host_edit.cpp", "host_relight.cpp")


def _host_edit(lib, rules, rays, depth, pts, albedo, rough, fresnel, acc, thr, scale):
    from tensoir_b200.editing import rule_table
    n = acc.shape[0]
    outs = (torch.empty(n, 3), torch.empty_like(rough), torch.empty(n, 3), torch.empty(n, dtype=torch.int32))
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    assert lib.tir_material_edit(rule_table(rules), len(rules), p(rays), p(depth), p(pts), p(albedo), p(rough),
                                 rough.shape[1], p(fresnel), p(acc), n, thr, p(scale), *(p(o) for o in outs),
                                 None) == 0
    return outs


@pytest.mark.parametrize("stride,use_rays", [(1, True), (3, False)])
def test_kernel_matches_host_build(fx, host_so, stride, use_rays):
    from tensoir_b200.editing import edit_materials
    g = np.random.default_rng(10 + stride)
    n = 100_000
    rays = torch.from_numpy(np.concatenate([g.uniform(-2, 2, (n, 3)), g.normal(size=(n, 3))], 1).astype(np.float32))
    depth = torch.from_numpy(g.uniform(0, 2, n).astype(np.float32))
    pts = torch.from_numpy(g.uniform(-1.5, 1.5, (n, 3)).astype(np.float32))
    albedo = torch.from_numpy(g.uniform(0, 1.2, (n, 3)).astype(np.float32))
    rough = torch.from_numpy(g.uniform(0.09, 0.99, (n, stride)).astype(np.float32))
    fresnel = torch.from_numpy(g.uniform(0, 1, (n, 3)).astype(np.float32))
    acc = torch.from_numpy(g.uniform(0, 1, n).astype(np.float32))
    scale = torch.tensor([0.9, 1.2, 1.05])
    rules = random_rules(g, 16)
    want = _host_edit(host_so, rules, rays if use_rays else None, depth if use_rays else None,
                      None if use_rays else pts, albedo, rough, fresnel, acc, 0.5, scale)
    maps = tuple(t.to(DEV) for t in (depth, torch.zeros(n, 3), albedo, rough, fresnel, acc))
    kw = dict(rays=rays.to(DEV)) if use_rays else dict(points=pts.to(DEV))
    got = edit_materials(maps, rules, scale.to(DEV), 0.5, **kw)
    again = edit_materials(maps, rules, scale.to(DEV), 0.5, **kw)
    for a, b, w in zip(got, again, want):
        assert torch.equal(a, b)                                    # bit-identical reruns
        assert torch.equal(a.cpu(), w)                              # the host build's bits
    if not use_rays:
        np_want = np_edit(rules, pts.numpy(), albedo.numpy(), rough.numpy(), fresnel.numpy(), acc.numpy(), 0.5,
                          scale.numpy())
        assert all(np.array_equal(a.cpu().numpy(), w) for a, w in zip(got, np_want))
    assert int((got[3] != 0).sum()) > n // 4


def _chunk(fx, names=("sunny", "dim")):
    from tensoir_b200.relight import Environment_Light
    rgb = fx["env_rgb"].numpy()
    hdr = {"sunny": rgb, "dim": rgb[:, ::-1].copy() * 0.4}
    env = Environment_Light({n: hdr[n] for n in names}, device=DEV)
    m = model_from_fixture(fx, DEV)
    return m, env, list(names), tuple(t.to(DEV) for t in fx["relight_maps"]), fx["rays"].to(DEV)


class ReplayVisibility:
    """relighting.relight_visibility recorded on the first pass and its outputs replayed, in call order, on later
    passes (the march still runs, so its launches still count)."""

    def __init__(self, monkeypatch):
        from tensoir_b200 import relighting as R
        self.fn, self.calls, self.i = R.relight_visibility, [], None
        monkeypatch.setattr(R, "relight_visibility", self)

    def __call__(self, *a):
        out = self.fn(*a)
        if self.i is None:
            self.calls.append(out)
            return out
        self.i += 1
        return self.calls[self.i - 1]


def _edited_shade(m, env, names, rays, maps, rules, scale, u, S, vis=None):
    from tensoir_b200 import relighting as R
    from tensoir_b200.editing import edit_materials
    envs, keep = R.env_tables(env, names)
    rays, maps = R.chunk_inputs(rays, maps)
    depth, normal, albedo, rough, fresnel, acc = maps
    L, n = len(names), rays.shape[0]
    if vis is None:
        vis = R.relight_visibility(m, envs, L, rays, depth, normal, acc, u, S, 0.5, 'nerv')
    a, r, f, sel = edit_materials(maps, rules, scale, 0.5, rays=rays)
    out = (torch.empty(L, n, 3, device=DEV), torch.empty(L, n, 3, device=DEV))
    R.relight_shade(envs, L, rays, normal, a, r, f, acc, S, 0.5, torch.ones(3, device=DEV), vis, 'nerv', out, 0)
    return out, sel, vis


def test_identity_edit_is_relight_chunk_fused(fx, monkeypatch):
    from tensoir_b200.relighting import relight_chunk_fused
    rv = ReplayVisibility(monkeypatch)
    m, env, names, maps, rays = _chunk(fx)
    S = 128
    u = torch.rand(2, rays.shape[0], S, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    scale = torch.tensor([1.3, 0.8, 1.1], device=DEV)
    w, wo = relight_chunk_fused(m, env, names, rays, maps, scale, u, S)
    rv.i = 0
    (ew, ewo), sel, _ = _edited_shade(m, env, names, rays, maps, [], scale, u, S)
    assert torch.equal(w, ew) and torch.equal(wo, ewo) and not sel.any()


def test_set_everywhere_is_substituted_maps(fx, monkeypatch):
    from tensoir_b200.editing import MaterialEdit
    from tensoir_b200.relighting import relight_chunk_fused
    rv = ReplayVisibility(monkeypatch)
    m, env, names, maps, rays = _chunk(fx)
    S = 128
    u = torch.rand(2, rays.shape[0], S, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(4))
    A, Rg, Fr = [0.7, 0.2, 0.4], 0.35, [0.3, 0.1, 0.05]
    rules = [MaterialEdit(albedo_set=A, roughness_set=Rg, fresnel_set=Fr)]
    (ew, ewo), sel, _ = _edited_shade(m, env, names, rays, maps, rules, 1.7, u, S)
    rv.i = 0
    depth, normal, albedo, rough, fresnel, acc = maps
    n = rays.shape[0]
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)  # noqa: E731
    sub = (depth, normal, f32(A).expand(n, 3).contiguous(), f32([Rg]).expand(n, rough.reshape(n, -1).shape[1])
           .contiguous(), f32(Fr).expand(n, 3).contiguous(), acc)
    w, wo = relight_chunk_fused(m, env, names, rays, sub, 1.0, u, S)
    assert torch.equal(w, ew) and torch.equal(wo, ewo)
    assert torch.equal(sel != 0, acc.reshape(-1) > 0.5)


def test_region_edit_on_lego_views():
    """A rule whose box is one lego box (the back wall, grown by two voxels) changes only the pixels whose surface point
    it selects, and the selection is the box test of the sampler's surface points."""
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import relighting as R
    from tensoir_b200.editing import MaterialEdit
    from tensoir_b200.relight import Environment_Light
    from tensoir_b200.synthetic import SyntheticViews, _lego_boxes, hemisphere_poses, make_lego_model
    import bench
    grid = 96
    m = make_lego_model(grid, DEV)
    env = Environment_Light({"a": bench.synthetic_hdr(seed=3)}, device=DEV)
    lo, hi, _ = _lego_boxes()[16]                                   # back wall
    pad = 2 * 3.0 / grid
    box = [[c - pad for c in lo], [c + pad for c in hi]]
    rules = [MaterialEdit(aabb=box, albedo_set=[0.9, 0.05, 0.05], roughness_set=0.15)]
    ds = SyntheticViews(hemisphere_poses(3), 48, 48, light_names=["a"])
    S, changed, kept = 64, 0, 0
    for v in range(len(ds)):
        rays = ds[v]["rays"].to(DEV)
        li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=DEV)
        with torch.no_grad():
            _, depth, normal, albedo, rough, fresnel, acc, *_ = m(rays, li, is_train=False, white_bg=True,
                                                                  ndc_ray=False, N_samples=-1)
        maps = (depth, normal, albedo, rough, fresnel, acc)
        u = R._uniforms(1, rays.shape[0], S, DEV)
        (w0, wo0), sel0, vis = _edited_shade(m, env, ["a"], rays, maps, [], 1.0, u, S)
        (w1, wo1), sel, _ = _edited_shade(m, env, ["a"], rays, maps, rules, 1.0, u, S, vis=vis)
        assert not sel0.any()
        p = rays[:, :3] + depth.reshape(-1, 1) * rays[:, 3:]
        blo, bhi = torch.tensor(box, device=DEV)
        hit = acc.reshape(-1) > 0.5
        inside = ((p > blo + 1e-4) & (p < bhi - 1e-4)).all(1) & hit
        outside = (((p < blo - 1e-4) | (p > bhi + 1e-4)).any(1)) | ~hit
        s = sel != 0
        assert bool(s[inside].all()) and not bool(s[outside].any())
        assert torch.equal(wo1[:, ~s], wo0[:, ~s]) and torch.equal(w1[:, ~s], w0[:, ~s])
        diff = (wo1[0, s] != wo0[0, s]).any(-1)
        changed += int(diff.sum())
        kept += int(s.sum())
    assert kept > 100 and changed > 0.9 * kept


class Replay:
    """The model's forward recorded on the first pass and replayed, with the same rays, on later passes."""

    def __init__(self, m):
        self.m, self.calls, self.i, self.fwd = m, [], None, m.forward
        m.forward = self

    def __call__(self, rays, *a, **k):
        if self.i is None:
            out = self.fwd(rays, *a, **k)
            self.calls.append((rays.clone(), [t.detach().clone() if torch.is_tensor(t) else t for t in out]))
            return out
        r, out = self.calls[self.i]
        self.i += 1
        assert torch.equal(r, rays)
        return [t.clone() if torch.is_tensor(t) else t for t in out]


def test_relight_edited_end_to_end(fx, tmp_path, monkeypatch):
    """Two variants and two maps on two 32x24 views, batch_size 300 (three chunks per view): the file list, the
    'original' files byte-identical to relight()'s under the same forward and uniforms, one visibility march per chunk,
    and the metrics text from pair_metrics."""
    import tensoir_b200.relighting as R
    from tensoir_b200 import _lib, editing
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    m, env, names, _, _ = _chunk(fx)
    rgb = fx["env_rgb"].numpy()
    hdr = {"sunny": rgb, "dim": rgb[:, ::-1].copy() * 0.4}
    H, W, B = 24, 32, 300
    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=names)
    n_chunks = -(-H * W // B)
    rep = Replay(m)
    rv = ReplayVisibility(monkeypatch)
    draws = []

    def uniforms(L, n, S, device):
        k = len(draws) % (len(ds) * n_chunks)
        if len(draws) < len(ds) * n_chunks:
            draws.append(torch.rand(L, n, S, dtype=torch.float64, device=device,
                                    generator=torch.Generator(device).manual_seed(100 + k)))
        else:
            draws.append(draws[k])
        return draws[-1].clone()
    monkeypatch.setattr(R, "_uniforms", uniforms)
    ref = tmp_path / "ref"
    R.relight(ds, types.SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(ref), batch_size=B), tensoIR=m)
    rep.i = rv.i = 0

    launches = []
    march = _lib.load().tir_march_density
    monkeypatch.setattr(_lib.load(), "tir_march_density", lambda *a: launches.append(1) or march(*a))
    pm, recorded = R.pair_metrics, []
    monkeypatch.setattr(R, "pair_metrics", lambda *a: recorded.append((a[0].clone(), pm(*a))) or recorded[-1][1])
    out = tmp_path / "edit"
    variants = {"red": [{"aabb": [[-2, -2, -2], [2, 0.0, 2]], "albedo_set": [0.9, 0.1, 0.1]}],
                "glossy": [{"roughness_set": 0.12, "fresnel_set": 0.6}]}
    editing.relight_edited(ds, types.SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(out), batch_size=B), variants,
                           tensoIR=m)
    assert len(launches) == len(ds) * n_chunks
    runs = ["original", "red", "glossy"]
    files = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs
                   if not f.endswith(".mp4"))
    want = [f"{v}/relight_psnr.txt" for v in runs]
    for i in range(len(ds)):
        for v in runs:
            want += [f"test_{i:03d}/{v}/{f}" for f in ("albedo_gamma_corrected.png", "roughness.png", "selection.png",
                                                      "relighting_without_bg/relight_psnr.txt")]
            want += [f"test_{i:03d}/{v}/relighting_{s}/{n}.png" for s in ("with_bg", "without_bg") for n in names]
    assert files == sorted(want)
    for i in range(len(ds)):
        for s in ("with_bg", "without_bg"):
            for n in names:
                assert (ref / f"test_{i:03d}/relighting_{s}/{n}.png").read_bytes() == \
                    (out / f"test_{i:03d}/original/relighting_{s}/{n}.png").read_bytes()
        assert (ref / f"test_{i:03d}/relighting_without_bg/relight_psnr.txt").read_text() == \
            (out / f"test_{i:03d}/original/relighting_without_bg/relight_psnr.txt").read_text()
    assert (ref / "relight_psnr.txt").read_text() == (out / "original/relight_psnr.txt").read_text()
    # one pair_metrics call per view and variant, in view-then-variant order; the text holds its numbers
    assert len(recorded) == len(ds) * len(runs)
    for c, (img, met) in enumerate(recorded):
        i, v = divmod(c, len(runs))
        d = out / f"test_{i:03d}" / runs[v]
        met = met.cpu().numpy()
        for k, n in enumerate(names):
            png = cv2.imread(str(d / "relighting_without_bg" / f"{n}.png"))[..., ::-1].reshape(-1, 3)
            assert np.array_equal(png, (img[k] * 255).to(torch.uint8).cpu().numpy())
        lines = (d / "relighting_without_bg" / "relight_psnr.txt").read_text().splitlines()
        for k, (n, line) in enumerate(zip(names, lines)):
            mt = re.fullmatch(rf"{n}: PNSR (\S+); SSIM (\S+); L_Alex \S+; L_VGG \S+", line)
            assert mt, line
            assert float(mt.group(1)) == -10.0 * np.log(met[k, 0] / (H * W * 3)) / np.log(10.0)
            assert float(mt.group(2)) == float(met[k, 1])
    red = cv2.imread(str(out / "test_000/red/selection.png"), cv2.IMREAD_UNCHANGED)
    assert red.any() and not red.all()


def test_edited_asset(fx, tmp_path, monkeypatch):
    from tensoir_b200 import mesh
    from tensoir_b200.editing import MaterialEdit, edit_materials
    m = model_from_fixture(fx, DEV)
    pts, faces, v = mesh.asset_surface(m)
    p = mesh.probe(m, v, mesh.vertex_normals(m, v))
    monkeypatch.setattr(mesh, "probe", lambda *a, **k: p)              # the same probe outputs for both exports
    rules = [MaterialEdit(aabb=[[-9, -9, -9], [9, 9, float(v[:, 2].median())]], albedo_set=[0.2, 0.6, 0.9]),
             MaterialEdit(roughness_mul=0.5)]
    plain, edited = str(tmp_path / "plain.ply"), str(tmp_path / "edited.ply")
    mesh.export_asset(m, plain, envmaps=False)
    mesh.export_asset(m, edited, envmaps=False, edits=rules)
    a, b = mesh.read_asset_ply(plain), mesh.read_asset_ply(edited)
    for k in ("xyz", "faces", "probed", "normal"):
        assert np.array_equal(a[k], b[k]), k
    V = v.shape[0]
    maps = (None, None, p["albedo"], p["roughness"].reshape(V, 1), torch.zeros(V, 3, device=DEV), p["probed"].float())
    alb, rough, _, sel = edit_materials(maps, rules, 1.0, 0.5, points=v)
    assert np.array_equal(b["albedo"], alb.cpu().numpy()) and np.array_equal(b["roughness"], rough[:, 0].cpu().numpy())
    assert np.array_equal(b["rgb"], mesh.vertex_colors(alb).cpu().numpy())
    probed = p["probed"].cpu().numpy()
    assert (sel.cpu().numpy()[probed] != 0).all() and not sel.cpu().numpy()[~probed].any()
    assert not np.array_equal(a["albedo"][probed], b["albedo"][probed])
    with pytest.raises(ValueError):
        mesh.export_asset(m, str(tmp_path / "f.ply"), edits=[MaterialEdit(fresnel_mul=0.5)])
