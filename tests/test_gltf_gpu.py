"""Textured glTF export on the GPU, on the fixture models of test_asset_gpu.py (the rotated model, shrunk states A and
B): the atlas kernels against their host twin bit for bit, the corner texels of the .glb against the PLY asset's
per-vertex columns, the texel probes against the oracle's eval-mode primary_forward, material edits, and
tools/export_asset.py --glb end to end.

The primary tail composites with float atomics, so probe results of separate runs agree at the map tolerance of
test_gpu_parity.py, not bit for bit."""
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import tensoir_oracle as O                                      # noqa: E402
from helpers import build_host_lib, on_host, oracle_field                   # noqa: E402
from gpu_helpers import load_fixture, load_shrunk_state, model_from_fixture  # noqa: E402
from test_gpu_parity import DEV, TOL, close                                # noqa: E402
from test_asset_gpu import _tool                                           # noqa: E402
from test_gltf_cpu import srgb64                                           # noqa: E402
from tensoir_b200 import gltf, mesh                                        # noqa: E402
from tensoir_b200.editing import MaterialEdit                              # noqa: E402

N_ORACLE_TEXELS = 2048


def smallest_texture(F):
    for T in (256, 512, 1024, 2048, 4096, 8192):
        if (T // gltf.S_MIN) ** 2 >= (F + 1) // 2:
            return T
    raise AssertionError(F)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_atlas_gpu"), "host_atlas.cpp")


@pytest.fixture(scope="module", params=["rotated", "A", "B"])
def baked(request, tmp_path_factory):
    fx = load_fixture("rotated_g24.pt") if request.param == "rotated" else load_shrunk_state(request.param)
    m = model_from_fixture(fx, DEV)
    d = tmp_path_factory.mktemp(f"glb_{request.param}")
    _, faces, v = mesh.asset_surface(m)
    F = faces.shape[0]
    T = smallest_texture(F)
    s = gltf.atlas_cell_size(F, T)
    glb, ply = str(d / "asset.glb"), str(d / "asset.ply")
    unprobed, degenerate = gltf.export_asset_glb(m, glb, texture_size=T)
    mesh.export_asset(m, ply)
    return types.SimpleNamespace(fx=fx, m=m, faces=faces, v=v, F=F, T=T, s=s, glb=glb, ply=ply, unprobed=unprobed,
                                 degenerate=degenerate)


def test_kernels_equal_the_host_twin(baked, host):
    b = baked
    F, T, s = b.F, b.T, b.s
    n = gltf.texel_count(F, s)
    pix, pos = gltf.atlas_texels(b.faces, b.v, T, s, 0, n)
    corners = gltf.atlas_corners(b.faces, b.v, T, s)
    g = torch.Generator().manual_seed(4)
    albedo = torch.rand(n, 3, generator=g) * 1.2 - 0.1
    rough = torch.rand(n, generator=g) * 1.2 - 0.1
    normal = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    probed = torch.rand(n, generator=g) < 0.9
    img = gltf.new_images(T, DEV)
    half = n // 2                  # two calls, to cover a range that starts inside the layout
    for lo, hi in ((0, half), (half, n)):
        gltf.atlas_encode(b.faces, b.v, T, s, lo, albedo[lo:hi].to(DEV), rough[lo:hi].to(DEV), normal[lo:hi].to(DEV),
                          probed[lo:hi].to(DEV), img)
    torch.cuda.synchronize()
    fc, vc = b.faces.cpu(), b.v.cpu()
    himg = gltf.new_images(T, "cpu")
    with on_host(host):
        hpix, hpos = gltf.atlas_texels(fc, vc, T, s, 0, n)
        hcorners = gltf.atlas_corners(fc, vc, T, s)
        gltf.atlas_encode(fc, vc, T, s, 0, albedo, rough, normal, probed, himg)
    assert torch.equal(pix.cpu(), hpix)
    assert torch.equal(pos.cpu().view(torch.int32), hpos.view(torch.int32))
    for k in corners:
        assert torch.equal(corners[k].cpu().view(torch.int32), hcorners[k].view(torch.int32)), k
    assert torch.equal(img.cpu(), himg)
    # repeated calls give the same bits
    pix2, pos2 = gltf.atlas_texels(b.faces, b.v, T, s, 0, n)
    assert torch.equal(pix2, pix) and torch.equal(pos2.view(torch.int32), pos.view(torch.int32))


def _decode_normal(rgb, N, Tw):
    x = rgb.astype(np.float64) / 255 * 2 - 1
    B = np.cross(N, Tw[:, :3]) * Tw[:, 3:]
    d = Tw[:, :3] * x[:, :1] + B * x[:, 1:2] + N * x[:, 2:]
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def test_corner_texels_hold_the_ply_asset_values(baked, capsys):
    b = baked
    got = gltf.read_glb(b.glb)
    ply = mesh.read_asset_ply(b.ply)
    acc = got["accessors"]
    pos, N, Tw, uv = acc[0], acc[1].astype(np.float64), acc[2].astype(np.float64), acc[3]
    assert pos.shape == (3 * b.F, 3)
    vid = ply["faces"].reshape(-1)                          # the PLY vertex of every glb corner row
    assert np.array_equal(pos.view(np.uint32), b.v.cpu().numpy()[vid].view(np.uint32))
    xy = np.rint(uv.astype(np.float64) * b.T - 0.5).astype(np.int64)
    px = xy[:, 1] * b.T + xy[:, 0]
    base, mr, nm = (im.reshape(-1, 4)[px] for im in got["images"])
    # the corner texels' own probe: probe() at the vertex (the same ray), against the PLY's columns within TOL
    pix, tpos = gltf.atlas_texels(b.faces, b.v, b.T, b.s, 0, gltf.texel_count(b.F, b.s))
    order = torch.argsort(pix.long())
    rows = torch.searchsorted(pix.long()[order], torch.from_numpy(px).to(DEV))
    texel_rows = order[rows]
    assert torch.equal(pix[texel_rows].cpu(), torch.from_numpy(px).int())
    assert torch.equal(tpos[texel_rows].cpu().view(torch.int32), torch.from_numpy(pos).view(torch.int32))
    albedo, rough, normal, probed = gltf.probe_texels(b.m, tpos[texel_rows])
    sel = probed.cpu().numpy() & (ply["probed"][vid] == 1)
    assert sel.mean() > 0.3, sel.mean()
    close(albedo.cpu()[sel], torch.from_numpy(ply["albedo"][vid][sel]), TOL, "corner albedo")
    close(rough.cpu()[sel], torch.from_numpy(ply["roughness"][vid][sel]), TOL, "corner roughness")
    close(normal.cpu()[sel], torch.from_numpy(ply["normal"][vid][sel]), TOL, "corner normal")
    # decoded from the images: 1 LSB plus TOL (through the OETF's largest slope, 12.92, for the albedo)
    want = srgb64(ply["albedo"][vid][sel])
    assert np.abs(base[sel, :3] / 255 - want).max() <= 1 / 255 + 12.92 * TOL
    assert np.abs(mr[sel, 1] / 255 - ply["roughness"][vid][sel]).max() <= 1 / 255 + TOL
    dec = _decode_normal(nm[sel, :3], N[sel], Tw[sel])
    want_n = ply["normal"][vid][sel].astype(np.float64)
    want_n /= np.linalg.norm(want_n, axis=1, keepdims=True)
    assert np.linalg.norm(dec - want_n, axis=1).max() <= 2 * np.sqrt(3) / 255 + 2 * TOL
    capsys.readouterr()


def test_texel_attributes_match_the_oracle(baked):
    b = baked
    n = gltf.texel_count(b.F, b.s)
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(7))[:N_ORACLE_TEXELS].to(DEV)
    _, pos = gltf.atlas_texels(b.faces, b.v, b.T, b.s, 0, n)
    v = pos[rows].contiguous()
    nrm = mesh.vertex_normals(b.m, v)
    p = mesh.probe(b.m, v, nrm)
    albedo, rough, normal, probed = gltf.probe_texels(b.m, v)
    has_n = mesh.has_normal(nrm).cpu()
    assert int(has_n.sum()) >= 2000 * 0.9
    rays = p["rays"].cpu()[has_n]
    li = b.fx["light_idx"].new_zeros(rays.shape[0], 1)
    _, _, o_normal, o_albedo, o_rough, _, o_acc, *_ = O.primary_forward(oracle_field(b.fx), rays, li, white_bg=True,
                                                                        is_train=False)
    close(p["acc"].cpu()[has_n], o_acc, TOL, "acc")
    got_probed = probed.cpu()
    near = torch.zeros_like(has_n)
    near[has_n] = (o_acc - mesh.PROBE_ACC_THRESHOLD).abs() <= TOL * (1 + mesh.PROBE_ACC_THRESHOLD)
    want_probed = torch.zeros_like(has_n)
    want_probed[has_n] = o_acc >= mesh.PROBE_ACC_THRESHOLD
    assert torch.equal(got_probed[~near], want_probed[~near])
    sel = got_probed[has_n]
    assert int(sel.sum()) > 200, int(sel.sum())
    close(albedo.cpu()[got_probed], o_albedo[sel], TOL, "albedo")
    close(rough.cpu()[got_probed], o_rough[sel, 0], TOL, "roughness")
    close(normal.cpu()[got_probed], o_normal[sel], TOL, "normal")
    un = ~got_probed
    assert torch.equal(albedo.cpu()[un], torch.zeros(int(un.sum()), 3))
    assert torch.equal(rough.cpu()[un], torch.ones(int(un.sum())))
    assert torch.equal(normal.cpu()[un & has_n], nrm.cpu()[un & has_n])
    assert bool((normal.cpu()[un & ~has_n] == torch.tensor([0.0, 0.0, 1.0])).all())


def test_edits_apply_to_the_texels(baked, tmp_path, capsys):
    b = baked
    lo, hi = b.v.min(0).values.cpu(), b.v.max(0).values.cpu()
    mid = (lo + hi) / 2
    box = (lo.tolist(), [float(mid[0]), *hi[1:].tolist()])
    edits = [MaterialEdit(aabb=box, albedo_set=(0.8, 0.2, 0.1), roughness_mul=0.5)]
    n = gltf.texel_count(b.F, b.s)
    _, pos = gltf.atlas_texels(b.faces, b.v, b.T, b.s, 0, n)
    p = mesh.probe(b.m, pos, mesh.vertex_normals(b.m, pos))
    want_a, want_r = mesh.edit_vertices(p, pos, edits)
    inside = ((pos >= torch.tensor(box[0], device=DEV)) & (pos <= torch.tensor(box[1], device=DEV))).all(1)
    sel = inside & p["probed"]
    assert int(sel.sum()) > 50
    assert torch.equal(want_a[sel], torch.tensor([0.8, 0.2, 0.1], device=DEV).expand(int(sel.sum()), 3))
    albedo, rough, _, probed = gltf.probe_texels(b.m, pos, edits)
    both = probed & p["probed"]
    close(albedo[both], want_a[both], TOL, "edited albedo")
    close(rough[both], want_r[both], TOL, "edited roughness")
    assert torch.equal(albedo[sel & probed], want_a[sel & probed])
    with pytest.raises(ValueError, match="fresnel"):
        gltf.export_asset_glb(b.m, str(tmp_path / "f.glb"), texture_size=b.T,
                              edits=[MaterialEdit(fresnel_set=(0.1, 0.1, 0.1))])
    assert not (tmp_path / "f.glb").exists()
    capsys.readouterr()


def test_glb_summary(baked):
    b = baked
    got = gltf.read_glb(b.glb)
    base = got["images"][0].reshape(-1, 4)
    pix, _ = gltf.atlas_texels(b.faces, b.v, b.T, b.s, 0, gltf.texel_count(b.F, b.s))
    assert 0 <= b.unprobed < pix.numel() and b.degenerate >= 0
    black = (base[pix.cpu().numpy(), :3] == 0).all(1).sum()
    assert black >= b.unprobed                     # unprobed texels have albedo 0
    assert got["json"]["meshes"][0]["primitives"][0]["attributes"]["POSITION"] == 0


def test_export_asset_tool_glb_end_to_end(tmp_path, capsys):
    from tensoir_b200.relight import read_hdr
    m = model_from_fixture(load_shrunk_state("B"), DEV)
    ckpt = str(tmp_path / "model.th")
    m.save(ckpt)
    path = _tool("export_asset").main(types.SimpleNamespace(ckpt=ckpt), glb=True, texture_size=512)
    out = capsys.readouterr().out
    assert path == ckpt[:-3] + "_asset.glb" and f"saving asset to {path}" in out
    got = gltf.read_glb(path)
    assert got["json"]["asset"]["version"] == "2.0" and len(got["images"]) == 3
    assert all(im.shape == (512, 512, 4) for im in got["images"])
    assert got["accessors"][0].shape[0] % 3 == 0
    hdrs = mesh.envmap_paths(path, m.light_num)
    assert hdrs == mesh.envmap_paths(ckpt[:-3] + "_asset.ply", m.light_num)
    assert all(read_hdr(q).shape == (*mesh.ENVMAP_HW, 3) for q in hdrs)
    assert not any(q.suffix == ".ply" for q in tmp_path.iterdir())


def test_export_asset_tool_glb_on_a_general_checkpoint(tmp_path, capsys):
    m = model_from_fixture(load_fixture("general_g20.pt"), DEV)
    ckpt = str(tmp_path / "general.th")
    m.save(ckpt)
    T = smallest_texture(mesh.asset_surface(m)[1].shape[0])
    path = _tool("export_asset").main(types.SimpleNamespace(ckpt=ckpt), glb=True, texture_size=T)
    out = capsys.readouterr().out
    assert path == ckpt[:-3] + "_asset.glb"
    gltf.read_glb(path)
    assert "general multi-light checkpoint" in out and "no environment map is written" in out
    assert not any(q.suffix == ".hdr" for q in tmp_path.iterdir())
