"""Mesh export on the GPU: getDenseAlpha against the reference's volumes (tests/golden/mesh_reference.pt), the
tir_marching_cubes_* kernels against the host build of the same C ABI bit for bit, and tools/export_mesh.py end to
end."""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

from gpu_helpers import load_fixture, load_shrunk_state, model_from_fixture
from helpers import build_host_lib
from mesh_helpers import LEVEL, assert_closed, host_marching_cubes, shared_volumes, signed_volume, sphere_volume
from tensoir_b200 import mesh

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_mesh"), "host_mesh.cpp")


@pytest.fixture(scope="module")
def golden_mesh():
    return load_fixture("mesh_reference.pt")


def _model(name):
    fx = load_fixture("rotated_g24.pt") if name == "rotated" else load_shrunk_state(name)
    return model_from_fixture(fx, "cuda:0")


def _same(lib, vol, level, spacing):
    gv, gf = mesh.marching_cubes(torch.from_numpy(vol).cuda(), level, spacing)
    hv, hf = host_marching_cubes(lib, vol, level, spacing)
    gv, gf = gv.cpu().numpy(), gf.cpu().numpy()
    assert np.array_equal(gv.view(np.uint32), hv.view(np.uint32))
    assert np.array_equal(gf, hf)
    return gv, gf


@pytest.mark.parametrize("name", ["rotated", "A", "B"])
def test_dense_alpha_and_mesh_on_fixture_volumes(lib, golden_mesh, name):
    rec = golden_mesh["models"][name]
    m = _model(name)
    alpha, _ = m.getDenseAlpha()
    want = rec["volume"]
    got = alpha.cpu()
    assert got.shape == want.shape
    assert bool(((got - want).abs() <= 2e-5 * (1 + want.abs())).all()), float((got - want).abs().max())
    assert torch.equal(got[want == 0], want[want == 0])           # exact zeros where the mask excludes
    sp = [float(v) for v in mesh.ply_spacing(tuple(want.shape), rec["aabb"])]
    verts, faces = _same(lib, want.numpy(), golden_mesh["level"], sp)
    assert len(faces) > 100


@pytest.mark.parametrize("case", range(len(shared_volumes())), ids=[n for n, _, _ in shared_volumes()])
def test_gpu_equals_host_build(lib, case):
    _, vol, sp = shared_volumes()[case]
    _, faces = _same(lib, vol, LEVEL, sp)
    assert_closed(faces)


def test_lego_300_bit_identical_and_equal_to_host(lib):
    """the 300^3 synthetic lego alpha: scans over many blocks and more than 2^24 cells"""
    from tensoir_b200.synthetic import make_lego_model
    m = make_lego_model(300, torch.device("cuda:0"))
    alpha, _ = m.getDenseAlpha()
    assert alpha.numel() > 1 << 24
    sp = [float(v) for v in mesh.ply_spacing(tuple(alpha.shape), m.aabb)]
    v1, f1 = mesh.marching_cubes(alpha, 0.005, sp)
    v2, f2 = mesh.marching_cubes(alpha, 0.005, sp)
    assert torch.equal(v1.view(torch.int32), v2.view(torch.int32)) and torch.equal(f1, f2)
    assert len(f1) > 100000
    hv, hf = host_marching_cubes(lib, alpha.cpu().numpy(), 0.005, sp)
    assert np.array_equal(v1.cpu().numpy().view(np.uint32), hv.view(np.uint32))
    assert np.array_equal(f1.cpu().numpy(), hf)


def test_export_mesh_tool_end_to_end(tmp_path, capsys):
    m = _model("B")
    ckpt = str(tmp_path / "model.th")
    m.save(ckpt)
    spec = importlib.util.spec_from_file_location("export_mesh_tool",
                                                  os.path.join(os.path.dirname(HERE), "tools", "export_mesh.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    path = tool.main(types.SimpleNamespace(ckpt=ckpt))
    assert path == ckpt[:-3] + ".ply" and os.path.exists(path)
    want = str(tmp_path / "want.ply")
    mesh.convert_sdf_samples_to_ply(m.getDenseAlpha()[0], want, bbox=m.aabb, level=0.005)
    assert open(path, "rb").read() == open(want, "rb").read()
    assert f"saving mesh to {path}" in capsys.readouterr().out
    verts, faces = mesh.read_ply(path)
    assert len(faces) > 100 and faces.max() < len(verts)


def test_exported_sphere_faces_outward(tmp_path, capsys):
    """marching_cubes winds into the dense region (skimage's default); the written PLY, reversed like the reference's,
    faces outward: positive signed volume of the same size"""
    vol = torch.from_numpy(sphere_volume()).cuda()
    bbox = torch.tensor([[-1.0, -0.5, -2.0], [1.5, 2.0, 1.0]], device="cuda")
    path = str(tmp_path / "sphere.ply")
    mesh.convert_sdf_samples_to_ply(vol, path, bbox=bbox, level=LEVEL)
    capsys.readouterr()
    verts, faces = mesh.read_ply(path)
    assert_closed(faces)
    mv, mf = mesh.marching_cubes(vol, LEVEL, [float(v) for v in mesh.ply_spacing(tuple(vol.shape), bbox)])
    inner = -signed_volume(mv.cpu().numpy(), mf.cpu().numpy())
    got = signed_volume(verts, faces)
    assert got > 0 and abs(got - inner) < 1e-4 * inner, (got, inner)
