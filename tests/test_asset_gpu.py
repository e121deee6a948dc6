"""Relightable asset export on the GPU, on the fixture models of test_mesh_gpu.py (the rotated model, shrunk states A
and B): the geometry against export_mesh's PLY byte for byte, the probe directions against the oracle's derived normals,
the probed attributes against the oracle's eval-mode primary_forward on the same probe rays, the environment maps
against the oracle's SG lights, and tools/export_asset.py end to end.

The primary tail composites with float atomics, so only the geometry is bit-stable across runs; attributes are compared
at the map tolerance of test_gpu_parity.py."""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import tensoir_oracle as O                                      # noqa: E402
from helpers import oracle_field                                           # noqa: E402
from gpu_helpers import load_fixture, load_shrunk_state, model_from_fixture  # noqa: E402
from test_gpu_parity import DEV, TOL, close                                # noqa: E402
from tensoir_b200 import mesh                                              # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
NORMAL_TOL = 5e-4          # the derived-normal check of test_gpu_parity.test_unit_kernels


def _fixture(name):
    return load_fixture("rotated_g24.pt") if name == "rotated" else load_shrunk_state(name)


@pytest.fixture(scope="module", params=["rotated", "A", "B"])
def exported(request, tmp_path_factory):
    fx = _fixture(request.param)
    m = model_from_fixture(fx, DEV)
    d = tmp_path_factory.mktemp(f"asset_{request.param}")
    path, geo = str(d / "asset.ply"), str(d / "mesh.ply")
    unprobed = mesh.export_asset(m, path)
    mesh.export_mesh(m, geo)
    pts, faces, v = mesh.asset_surface(m)
    n = mesh.vertex_normals(m, v)
    p = mesh.probe(m, v, n)
    return types.SimpleNamespace(fx=fx, m=m, path=path, geo=geo, unprobed=unprobed, v=v, n=n, p=p)


def _body(path):
    data = open(path, "rb").read()
    return data, data.index(b"end_header\n") + len(b"end_header\n")


def test_geometry_is_export_mesh_byte_for_byte(exported):
    e = exported
    data, end = _body(e.path)
    gdata, gend = _body(e.geo)
    V, F = mesh.read_ply(e.geo)[0].shape[0], mesh.read_ply(e.geo)[1].shape[0]
    assert V > 100 and F > 100
    rec = np.frombuffer(data, np.uint8, 44 * V, end).reshape(V, 44)
    assert rec[:, :12].tobytes() == gdata[gend:gend + 12 * V]                     # x y z
    assert data[end + 44 * V:] == gdata[gend + 12 * V:]                            # face records
    got = mesh.read_asset_ply(e.path)
    assert int((got["probed"] == 0).sum()) == e.unprobed
    # the file holds probe()'s attributes (a separate run: equal at the map tolerance, not bit for bit)
    p = e.p
    for k in ("albedo", "roughness", "normal"):
        sel = p["probed"].cpu() & torch.from_numpy(got["probed"] == 1)
        close(torch.from_numpy(got[k])[sel], p[k].cpu()[sel], TOL, k)


def _ill_conditioned(fx, xn):
    """Vertices whose derived normal fp32 cannot pin down to NORMAL_TOL: the fp32 and float64 oracle normals differ by
    more than that (test_shrunk_field_gpu.ill_conditioned_rays' criterion at the vertices)."""
    f, f64 = oracle_field(fx), oracle_field(fx).to("cpu", torch.float64)
    x32 = xn.clone().requires_grad_(True)
    g32 = torch.autograd.grad(O.feature2density(f, O.density_feature_with_xyz_grad(f, x32)).sum(), x32)[0]
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        x64 = xn.double().requires_grad_(True)
        g64 = torch.autograd.grad(O.feature2density(f64, O.density_feature_with_xyz_grad(f64, x64)).sum(), x64)[0]
    finally:
        torch.set_default_dtype(old)
    nrm = torch.nn.functional.normalize
    return (nrm(g32.double(), dim=-1) - nrm(g64, dim=-1)).norm(dim=-1) > NORMAL_TOL


def test_probe_directions_are_the_oracle_derived_normals(exported):
    """Vertices are excluded by test_shrunk_field_gpu's criterion (the fp32 and float64 oracle normals differ by more
    than the tolerance), with the tolerance unchanged.  The cap on excluded vertices is a choice made here from the
    measured counts: 436 of 1512 vertices (29 %) on the rotated model, 496 of 4620 (11 %) on states A and B, more than
    the 1 in 8 that close_maps allows for rays (where a ray's normals_diff_map is a weighted sum over its samples, while a
    vertex is a single point).  The cap is 1 in 3, above both counts."""
    e = exported
    f = oracle_field(e.fx)
    xn = O.normalize_coord(f, e.v.cpu())
    want = O.derived_normals(f, xn.clone()).detach()
    ill = _ill_conditioned(e.fx, xn)
    assert int(ill.sum()) <= ill.numel() // 3, int(ill.sum())
    close(e.n[~ill.to(DEV)], want[~ill], NORMAL_TOL, "derived normals")
    assert torch.equal(e.p["rays"][:, 3:], -e.n)


def test_probed_attributes_match_the_oracle(exported):
    e = exported
    p = e.p
    has_n = mesh.has_normal(e.n).cpu()
    rays = p["rays"].cpu()[has_n]
    f = oracle_field(e.fx)
    li = e.fx["light_idx"].new_zeros(rays.shape[0], 1)
    _, _, normal, albedo, rough, _, acc, *_ = O.primary_forward(f, rays, li, white_bg=True, is_train=False)
    got_acc = p["acc"].cpu()
    close(got_acc[has_n], acc, TOL, "acc")
    assert torch.equal(got_acc[~has_n], torch.zeros(int((~has_n).sum())))
    want_probed = torch.zeros_like(has_n)
    want_probed[has_n] = acc >= mesh.PROBE_ACC_THRESHOLD
    got_probed = p["probed"].cpu()
    near_threshold = torch.zeros_like(has_n)
    near_threshold[has_n] = (acc - mesh.PROBE_ACC_THRESHOLD).abs() <= TOL * (1 + mesh.PROBE_ACC_THRESHOLD)
    assert torch.equal(got_probed[~near_threshold], want_probed[~near_threshold])
    sel = got_probed[has_n]
    assert int(sel.sum()) > 50, int(sel.sum())
    close(p["albedo"].cpu()[got_probed], albedo[sel], TOL, "albedo")
    close(p["roughness"].cpu()[got_probed], rough[sel, 0], TOL, "roughness")
    close(p["normal"].cpu()[got_probed], normal[sel], TOL, "normal")
    # the fallback of unprobed vertices
    un = ~got_probed
    assert torch.equal(p["albedo"].cpu()[un], torch.zeros(int(un.sum()), 3))
    assert torch.equal(p["roughness"].cpu()[un], torch.ones(int(un.sum())))
    assert torch.equal(p["normal"].cpu()[un & has_n], e.n.cpu()[un & has_n])
    assert bool((p["normal"].cpu()[un & ~has_n] == torch.tensor([0.0, 0.0, 1.0])).all())


def _three_light_models():
    """(fixture, model) of the general fixture (three named lights) and of the rotated fixture's field with three
    rotations (its light_line gets a third row)."""
    gen = load_fixture("general_g20.pt")
    rot = load_fixture("rotated_g24.pt")
    sd = dict(rot["state_dict"])
    w = sd["light_line.weight"]
    sd["light_line.weight"] = torch.cat([w, w[:1] * 0.5 + w[-1:] * 0.5])
    rot3 = dict(rot, light_rotation=[0, 120, 240], state_dict=sd)
    return [(fx, model_from_fixture(fx, DEV)) for fx in (gen, rot3)]


def test_three_lights_write_three_envmaps(tmp_path, capsys):
    from tensoir_b200.relight import read_hdr
    H, W = mesh.ENVMAP_HW
    _, dirs = O.generate_envir_map_dir(H, W)
    for i, (fx, m) in enumerate(_three_light_models()):
        assert m.light_num == 3
        path = str(tmp_path / f"model{i}_asset.ply")
        mesh.export_asset(m, path)
        hdrs = sorted(q.name for q in tmp_path.iterdir() if q.name.startswith(f"model{i}_asset_envmap_"))
        assert hdrs == [f"model{i}_asset_envmap_{k}.hdr" for k in range(3)]
        want = O.get_light_rgbs(oracle_field(fx), dirs).clamp(min=0).reshape(3, H, W, 3).numpy()
        assert (want.max(-1) > 0).mean() > 0.99
        for k, q in enumerate(mesh.envmap_paths(path, 3)):
            got = read_hdr(q)
            assert got.shape == (H, W, 3) and got.dtype == np.float32
            # one RGBE mantissa step of the pixel's exponent, plus the fp32 difference of the two SG evaluations
            step = np.ldexp(1.0, np.frexp(want[k].max(-1, keepdims=True) * (1 + 1e-5))[1] - 8)
            err = np.abs(got - want[k])
            assert (err <= step + 1e-5 * (1 + np.abs(want[k]))).all(), float((err / step).max())
    capsys.readouterr()


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(HERE), "tools", f"{name}.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    return tool


def test_export_asset_tool_on_a_general_checkpoint(tmp_path, capsys):
    """A general multi-light checkpoint does not hold its SG lights (lgtSGs_list is not in the state_dict): the tool
    writes the mesh with its attributes and no environment map, and says why."""
    m = model_from_fixture(load_fixture("general_g20.pt"), DEV)
    ckpt = str(tmp_path / "general.th")
    m.save(ckpt)
    path = _tool("export_asset").main(types.SimpleNamespace(ckpt=ckpt))
    out = capsys.readouterr().out
    assert path == ckpt[:-3] + "_asset.ply" and os.path.exists(path)
    assert "general multi-light checkpoint" in out and "no environment map is written" in out
    assert not any(q.suffix == ".hdr" for q in tmp_path.iterdir())
    geo = _tool("export_mesh").main(types.SimpleNamespace(ckpt=ckpt))
    capsys.readouterr()
    asset = mesh.read_asset_ply(path)
    verts, faces = mesh.read_ply(geo)
    assert np.array_equal(asset["xyz"].view(np.uint32), verts.view(np.uint32))
    assert np.array_equal(asset["faces"], faces)


def test_export_asset_tool_end_to_end(tmp_path, capsys):
    m = model_from_fixture(load_shrunk_state("B"), DEV)
    ckpt = str(tmp_path / "model.th")
    m.save(ckpt)
    path = _tool("export_asset").main(types.SimpleNamespace(ckpt=ckpt))
    assert path == ckpt[:-3] + "_asset.ply" and os.path.exists(path)
    out = capsys.readouterr().out
    assert f"saving asset to {path}" in out
    geo = _tool("export_mesh").main(types.SimpleNamespace(ckpt=ckpt))
    capsys.readouterr()
    asset = mesh.read_asset_ply(path)
    verts, faces = mesh.read_ply(geo)
    assert np.array_equal(asset["xyz"].view(np.uint32), verts.view(np.uint32))
    assert np.array_equal(asset["faces"], faces)
    assert 0 < int(asset["probed"].sum()) <= len(verts)
    assert f"{len(verts) - int(asset['probed'].sum())} unprobed" in out
    from tensoir_b200.relight import read_hdr
    hdrs = mesh.envmap_paths(path, m.light_num)
    assert all(os.path.exists(q) and read_hdr(q).shape == (*mesh.ENVMAP_HW, 3) for q in hdrs)
    assert not os.path.exists(mesh.envmap_paths(path, m.light_num + 1)[-1])
