"""Relightable asset export on the CPU: the PLY layout and its reader, the field-space probe positions against
getDenseAlpha's sample grid, the probe rays against the primary sampler, the vertex colours and the .hdr round trip."""
import types

import numpy as np
import pytest
import torch

from helpers import build_host_lib
from mesh_helpers import LEVEL, host_marching_cubes, random_volume
from oracle import tensoir_oracle as O
from tensoir_b200 import mesh

HEADER = (b"ply\nformat binary_little_endian 1.0\nelement vertex {V}\nproperty float x\nproperty float y\n"
          b"property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
          b"property uchar green\nproperty uchar blue\nproperty float roughness\nproperty float albedo_r\n"
          b"property float albedo_g\nproperty float albedo_b\nproperty uchar probed\nelement face {F}\n"
          b"property list uchar int vertex_indices\nend_header\n")
RECORD = np.dtype({"names": ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue", "roughness", "albedo_r",
                             "albedo_g", "albedo_b", "probed"],
                   "formats": ["<f4"] * 6 + ["u1"] * 3 + ["<f4"] * 4 + ["u1"],
                   "offsets": [0, 4, 8, 12, 16, 20, 24, 25, 26, 27, 31, 35, 39, 43], "itemsize": 44})


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_mesh"), "host_mesh.cpp")


def _hand_mesh(V=7, F=5, seed=3):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(V, 3, generator=g)
    faces = torch.randint(0, V, (F, 3), generator=g, dtype=torch.int32)
    normal = torch.nn.functional.normalize(torch.randn(V, 3, generator=g), dim=-1)
    albedo = torch.rand(V, 3, generator=g)
    albedo[0] = torch.tensor([0.0, 1.0, 0.5])
    rough = torch.rand(V, generator=g)
    probed = torch.arange(V) % 3 != 0
    return pts, faces, normal, albedo, rough, probed


def test_asset_ply_layout_and_reader(tmp_path):
    pts, faces, normal, albedo, rough, probed = _hand_mesh()
    V, F = pts.shape[0], faces.shape[0]
    data = mesh.asset_ply_bytes(pts, faces, normal, albedo, rough, probed)
    head = HEADER.replace(b"{V}", str(V).encode()).replace(b"{F}", str(F).encode())
    assert data[:len(head)] == head
    assert len(data) == len(head) + 44 * V + 13 * F
    rec = np.frombuffer(data, RECORD, V, len(head))
    assert np.array_equal(np.stack([rec["x"], rec["y"], rec["z"]], -1), pts.numpy())
    assert np.array_equal(np.stack([rec["nx"], rec["ny"], rec["nz"]], -1), normal.numpy())
    assert np.array_equal(np.stack([rec["red"], rec["green"], rec["blue"]], -1),
                          (albedo ** (1 / 2.2) * 255).to(torch.uint8).numpy())
    assert np.array_equal(rec["roughness"], rough.numpy())
    assert np.array_equal(np.stack([rec["albedo_r"], rec["albedo_g"], rec["albedo_b"]], -1), albedo.numpy())
    assert np.array_equal(rec["probed"], probed.numpy().astype(np.uint8))
    # the face element is ply_bytes' (the reference's faces[..., ::-1] records)
    geo = mesh.ply_bytes(torch.zeros(V, 3), faces, torch.zeros(2, 3))
    assert data[-13 * F:] == geo[-13 * F:]

    path = tmp_path / "asset.ply"
    path.write_bytes(data)
    got = mesh.read_asset_ply(str(path))
    assert np.array_equal(got["xyz"], pts.numpy()) and np.array_equal(got["normal"], normal.numpy())
    assert np.array_equal(got["albedo"], albedo.numpy()) and np.array_equal(got["roughness"], rough.numpy())
    assert np.array_equal(got["probed"], probed.numpy().astype(np.uint8))
    assert np.array_equal(got["faces"], faces.flip(-1).numpy())
    for bad in (data[:-1], data + b"\0", geo):        # truncated, over-long, the geometry-only layout
        path.write_bytes(bad)
        with pytest.raises(ValueError):
            mesh.read_asset_ply(str(path))


def test_empty_asset_ply(tmp_path):
    z3 = torch.zeros(0, 3)
    data = mesh.asset_ply_bytes(z3, torch.zeros(0, 3, dtype=torch.int32), z3, z3, torch.zeros(0),
                                torch.zeros(0, dtype=torch.bool))
    assert data == HEADER.replace(b"{V}", b"0").replace(b"{F}", b"0")
    path = tmp_path / "empty.ply"
    path.write_bytes(data)
    got = mesh.read_asset_ply(str(path))
    assert got["xyz"].shape == (0, 3) and got["faces"].shape == (0, 3)


def test_vertex_colors_follow_the_evaluation():
    """relighting.relight's albedo_gamma_corrected.png expression on a linear albedo map"""
    albedo_map = torch.cat([torch.linspace(0, 1, 1001), torch.tensor([0.0, 1.0, 1e-7, 0.9999999])]).reshape(-1, 1)
    albedo_map = albedo_map.expand(-1, 3).contiguous()
    want = (albedo_map ** (1 / 2.2) * 255).to(torch.uint8)
    assert torch.equal(mesh.vertex_colors(albedo_map), want)


def _stub_model(vol, bbox):
    """An object with TensorBase.getDenseAlpha over a given volume (slab i of ``vol`` is its alpha at x index i)."""
    from tensoir_b200.tensorbase import TensorBase
    slabs = iter(torch.from_numpy(vol))
    stub = types.SimpleNamespace(gridSize=torch.tensor(vol.shape), device="cpu", aabb=bbox, stepSize=0.1,
                                 compute_alpha=lambda xyz, length: next(slabs).reshape(-1))
    stub.getDenseAlpha = lambda: TensorBase.getDenseAlpha(stub)
    return stub


def test_field_positions_lie_on_the_dense_alpha_grid(lib, monkeypatch, tmp_path, capsys):
    """asset_surface: the PLY coordinates are convert_sdf_samples_to_ply's, byte for byte; the field positions sit on
    getDenseAlpha's sample grid (dense_xyz), so a vertex on a grid point is that point of dense_xyz."""
    vol = random_volume((13, 9, 11), 21)           # 10 % of the points exactly at the level: vertices on grid points
    bbox = torch.tensor([[-1.25, -0.5, -2.0], [1.5, 0.75, 1.0]])
    monkeypatch.setattr(mesh, "marching_cubes", lambda v, level, spacing: tuple(
        torch.from_numpy(x) for x in host_marching_cubes(lib, v.numpy(), level, spacing)))
    pts, faces, v = mesh.asset_surface(_stub_model(vol, bbox), LEVEL)
    path = tmp_path / "mesh.ply"
    mesh.convert_sdf_samples_to_ply(torch.from_numpy(vol), str(path), bbox=bbox, level=LEVEL)
    capsys.readouterr()
    want_v, want_f = mesh.read_ply(str(path))
    assert np.array_equal(pts.numpy().view(np.uint32), want_v.view(np.uint32))
    assert np.array_equal(faces.flip(-1).numpy(), want_f)

    _, dense_xyz = _stub_model(vol, bbox).getDenseAlpha()
    idx, _ = host_marching_cubes(lib, vol, LEVEL)
    on_grid = (idx == np.round(idx)).all(-1)
    assert on_grid.sum() > 20 and (~on_grid).sum() > 20
    j = np.round(idx[on_grid]).astype(np.int64)
    at = dense_xyz[j[:, 0], j[:, 1], j[:, 2]]
    assert torch.allclose(v[on_grid], at, rtol=0, atol=4e-7), float((v[on_grid] - at).abs().max())
    # every other vertex lies on its grid edge between two points of dense_xyz, at the marching-cubes fraction
    lo = np.floor(idx[~on_grid]).astype(np.int64)
    t = torch.from_numpy(idx[~on_grid] - lo).float()
    hi = np.minimum(lo + 1, np.array(vol.shape) - 1)
    p0, p1 = dense_xyz[lo[:, 0], lo[:, 1], lo[:, 2]], dense_xyz[hi[:, 0], hi[:, 1], hi[:, 2]]
    assert torch.allclose(v[~on_grid], p0 + t * (p1 - p0), rtol=0, atol=1e-6)
    # the PLY vertex is the same vertex at the reference's N-divided spacing, up to a voxel toward bbox[0]
    voxel = (bbox[1] - bbox[0]) / (torch.tensor(vol.shape) - 1)
    shift = v - pts
    assert bool((shift >= -1e-6).all()) and bool((shift <= voxel + 1e-6).all())


@pytest.fixture(scope="module")
def rotated_cpu(golden_rotated):
    from gpu_helpers import model_from_fixture
    from helpers import oracle_field
    return model_from_fixture(golden_rotated, "cpu"), oracle_field(golden_rotated)


def test_probe_rays_start_outside_the_vertex(rotated_cpu):
    """The primary sampler (sample_ray, the reference's; the kernels' lists equal it, test_gpu_parity) on probe rays: the
    first sample is v + r n when the box entry comes earlier, and the box entry when it comes later."""
    m, f = rotated_cpu
    r = mesh.probe_offset(m)
    assert r == pytest.approx(mesh.PROBE_OFFSET_VOXELS * float(m.units.max()))
    near = float(m.near_far[0])
    g = torch.Generator().manual_seed(7)
    lo, hi = f.aabb[0], f.aabb[1]
    n = torch.nn.functional.normalize(torch.randn(64, 3, generator=g), dim=-1)
    inner = lo + (hi - lo) * (0.3 + 0.4 * torch.rand(64, 3, generator=g))         # v + r n well inside the box
    rays = mesh.probe_rays(inner, n, near, r)
    assert torch.equal(rays[:, 3:], -n)
    pts, z, _ = O.sample_ray(f, rays[:, :3], rays[:, 3:6], is_train=False)
    assert torch.allclose(z[:, 0], torch.full((64,), near), rtol=0, atol=1e-6)
    assert torch.allclose(pts[:, 0], inner + r * n, rtol=0, atol=2e-6)
    assert torch.allclose(pts[:, 1] - pts[:, 0], -n * float(m.stepSize), rtol=0, atol=2e-6)

    # vertices half a probe offset inside the +x face, normals leaning out through it: v + r n is outside the box
    edge = inner.clone()
    edge[:, 0] = hi[0] - 0.5 * r
    n_out = torch.nn.functional.normalize(n * torch.tensor([0.0, 0.3, 0.3]) + torch.tensor([1.0, 0.0, 0.0]), dim=-1)
    rays = mesh.probe_rays(edge, n_out, near, r)
    pts, z, _ = O.sample_ray(f, rays[:, :3], rays[:, 3:6], is_train=False)
    entry = (rays[:, 0] - hi[0]) / n_out[:, 0]            # where the ray crosses x = hi[0]
    assert bool((z[:, 0] > near + 1e-4).all())
    assert torch.allclose(z[:, 0], entry, rtol=0, atol=2e-6)
    assert torch.allclose(pts[:, 0, 0], hi[0].expand(64), rtol=0, atol=2e-6)
    between = ((pts[:, 0] - edge) * n_out).sum(-1)        # the first sample lies between the vertex and v + r n
    assert bool(((between > 0) & (between < r)).all())


class _ForwardStub:
    """The model surface probe() uses, with a forward that returns fixed maps and records the rays it is given."""
    near_far = [2.0, 6.0]
    units = torch.tensor([0.1, 0.1, 0.1])

    def __init__(self, acc):
        self.acc, self.seen = acc, []

    def __call__(self, rays, light_idx, is_train, white_bg, ndc_ray, N_samples):
        assert not is_train and white_bg and not ndc_ray and N_samples == -1 and bool((light_idx == 0).all())
        n = rays.shape[0]
        a = self.acc[sum(r.shape[0] for r in self.seen):][:n]
        self.seen.append(rays)
        return (None, None, torch.full((n, 3), 0.6), torch.full((n, 3), 0.25), torch.full((n, 1), 0.3), None, a)


def test_probe_renders_only_unit_normals_and_falls_back():
    """Derived normals shorter than 1 come from a gradient below the normalisation's eps and give no direction: those
    vertices are not rendered and get the (0,0,1) fallback, like zero normals.  A rendered vertex with acc < 0.5 keeps
    its derived normal; every unprobed vertex gets albedo 0 and roughness 1."""
    g = torch.Generator().manual_seed(5)
    v = torch.randn(9, 3, generator=g)
    n = torch.nn.functional.normalize(torch.randn(9, 3, generator=g), dim=-1)
    n[2] = 0.0
    n[5] = n[5] * 0.3                      # |grad| = 3e-7: -grad / 1e-6
    model = _ForwardStub(torch.tensor([0.9, 0.2, 0.5, 0.49, 1.0, 0.7, 0.6]))
    p = mesh.probe(model, v, n, chunk=3)
    rendered = torch.tensor([0, 1, 3, 4, 6, 7, 8])
    assert torch.equal(torch.cat(model.seen), p["rays"][rendered]) and [r.shape[0] for r in model.seen] == [3, 3, 1]
    assert torch.equal(mesh.has_normal(n), torch.tensor([True, True, False, True, True, False, True, True, True]))
    want_acc = torch.zeros(9)
    want_acc[rendered] = model.acc
    assert torch.equal(p["acc"], want_acc)
    probed = want_acc >= 0.5
    assert torch.equal(p["probed"], probed)
    assert torch.equal(p["albedo"][probed], torch.full((int(probed.sum()), 3), 0.25))
    assert torch.equal(p["roughness"][probed], torch.full((int(probed.sum()),), 0.3))
    assert torch.equal(p["normal"][probed], torch.full((int(probed.sum()), 3), 0.6))
    assert torch.equal(p["albedo"][~probed], torch.zeros(int((~probed).sum()), 3))
    assert torch.equal(p["roughness"][~probed], torch.ones(int((~probed).sum())))
    assert torch.equal(p["normal"][[1, 4]], n[[1, 4]])
    assert torch.equal(p["normal"][[2, 5]], torch.tensor([[0.0, 0.0, 1.0]] * 2))


def test_hdr_round_trip_within_rgbe_precision(tmp_path):
    from tensoir_b200.relight import read_hdr, write_hdr
    g = np.random.default_rng(4)
    rgb = (g.random((16, 32, 3)) * 10.0 ** g.uniform(-3, 2, (16, 32, 1))).astype(np.float32)
    rgb[0, 0] = 0.0
    rgb[1, 1] = [5.0, 0.0, 1e-4]
    path = str(tmp_path / "env.hdr")
    write_hdr(path, rgb)
    got = read_hdr(path)
    assert got.shape == rgb.shape and got.dtype == np.float32
    # RGBE: one 8-bit mantissa per channel under the exponent of the pixel's largest channel
    step = np.ldexp(1.0, np.frexp(rgb.max(-1, keepdims=True))[1] - 8)
    assert (np.abs(got - rgb) <= step).all(), float((np.abs(got - rgb) / step).max())
    assert (got[0, 0] == 0).all()


def test_envmap_paths():
    assert mesh.envmap_paths("/a/b/model_asset.ply", 3) == [f"/a/b/model_asset_envmap_{k}.hdr" for k in range(3)]
