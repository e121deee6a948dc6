"""Mesh export on the CPU.

The tir_marching_cubes_* entry points are built for the host (tests/host_mesh.cpp: the same C ABI, argument checks,
scratch layout and per-cell math of csrc/tir_mc_body.h, loops instead of kernels) and driven through the real ctypes
wrapper tensoir_b200.mesh.  They must agree with the numpy restatement oracle/mesh_oracle.py, give closed,
consistently wound meshes, and the PLY post-processing must reproduce the reference's (tests/golden/mesh_reference.pt).
"""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from helpers import build_host_lib
from mesh_helpers import (LEVEL, assert_closed, boundary_edges, euler, host_marching_cubes, random_volume,
                          saddle_volume, shared_volumes, signed_volume, sphere_volume, torus_volume)
from oracle import mesh_oracle as MO
from tensoir_b200 import mesh

HEADER = (b"ply\nformat binary_little_endian 1.0\nelement vertex {V}\nproperty float x\nproperty float y\n"
          b"property float z\nelement face {F}\nproperty list uchar int vertex_indices\nend_header\n")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = build_host_lib(tmp_path_factory.mktemp("host_mesh"), "host_mesh.cpp")
    lib.mc_host_cell.restype, lib.mc_host_cell.argtypes = C.c_int, [C.c_int32, C.c_int32, C.c_void_p]
    lib.mc_host_face_connected.restype = C.c_int
    lib.mc_host_face_connected.argtypes = [C.c_float] * 5
    return lib


def host_cell(lib, mask, connected):
    buf = (C.c_int8 * 36)()
    n = lib.mc_host_cell(mask, connected, buf)
    return [tuple(buf[3 * t:3 * t + 3]) for t in range(n)]


def crossed_edges(mask):
    out = set()
    for e in range(12):
        a = e // 4
        u, w = [b for b in range(3) if b != a]
        c0 = ((e & 1) << u) | (((e >> 1) & 1) << w)
        if (mask >> c0 & 1) != (mask >> (c0 | 1 << a) & 1):
            out.add(e)
    return out


def ambiguous_faces(mask):
    out = []
    for f in range(6):
        a, side = f // 2, f % 2
        u, w = [b for b in range(3) if b != a]
        q = [(side << a) | (du << u) | (dw << w) for du, dw in ((0, 0), (1, 0), (0, 1), (1, 1))]
        i = [mask >> c & 1 for c in q]
        if i[0] == i[3] and i[1] == i[2] and i[0] != i[1]:
            out.append(f)
    return out


def test_every_cell_configuration(lib):
    """All 256 corner patterns under every outcome of the face decider: the loops close, every crossed edge is a vertex
    of the cell's triangles and starts / ends exactly one boundary segment, the triangle count is sum(k-2), and the
    host build equals the oracle's independent derivation."""
    n_cases = 0
    for mask in range(256):
        cross = crossed_edges(mask)
        amb = ambiguous_faces(mask)
        for bits in itertools.product((0, 1), repeat=len(amb)):
            conn = sum(b << f for b, f in zip(bits, amb))
            tris = host_cell(lib, mask, conn)
            assert tris == list(MO.cell_triangles(mask, conn)), (mask, conn)
            used = {e for t in tris for e in t}
            assert used == cross, (mask, conn)
            # directed boundary edges of the cell's patch: one segment out of and one into every crossed edge
            de = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
            assert len(set(de)) == len(de)
            bnd = [d for d in de if (d[1], d[0]) not in de]
            assert sorted(a for a, _ in bnd) == sorted(cross) and sorted(b for _, b in bnd) == sorted(cross)
            # loops: follow the boundary segments
            nxt = dict(bnd)
            loops, seen = 0, set()
            for e in sorted(cross):
                if e in seen:
                    continue
                loops += 1
                while e not in seen:
                    seen.add(e)
                    e = nxt[e]
            assert len(tris) == len(cross) - 2 * loops, (mask, conn)
            n_cases += 1
    assert n_cases == sum(2 ** len(ambiguous_faces(m)) for m in range(256))


@pytest.mark.parametrize("case", range(len(shared_volumes())), ids=[n for n, _, _ in shared_volumes()])
def test_closed_volumes_match_oracle(lib, case):
    name, vol, sp = shared_volumes()[case]
    verts, faces = host_marching_cubes(lib, vol, LEVEL, sp)
    ov, of = MO.marching_cubes(vol, LEVEL, sp)
    assert np.array_equal(verts.view(np.uint32), ov.view(np.uint32)), name
    assert np.array_equal(faces, of), name
    assert len(verts) == MO.crossed_edge_count(vol, LEVEL) > 0
    assert_closed(faces)
    assert faces.min() >= 0 and faces.max() < len(verts)


def test_vertices_on_their_edges(lib):
    """every vertex sits on its grid edge at the fp64-interpolated position, rounded to fp32 once"""
    vol = random_volume((13, 8, 11), 7)
    sp = (0.7, 1.3, 0.45)
    verts, _ = host_marching_cubes(lib, vol, LEVEL, sp)
    ins = vol > np.float32(LEVEL)
    want = []
    for p in range(vol.size):
        i = np.unravel_index(p, vol.shape)
        for a in range(3):
            j = list(i)
            j[a] += 1
            if j[a] >= vol.shape[a] or ins[i] == ins[tuple(j)]:
                continue
            t = (np.float64(np.float32(LEVEL)) - np.float64(vol[i])) / (np.float64(vol[tuple(j)]) - np.float64(vol[i]))
            want.append([np.float32((i[c] + t) * sp[c]) if c == a else np.float32(i[c] * sp[c]) for c in range(3)])
    assert np.array_equal(verts, np.array(want, dtype=np.float32))


def test_open_boundary_edges_lie_on_outer_faces(lib):
    """without the zero border the mesh is open only where it meets the array's outer faces, as with skimage"""
    vol = random_volume((12, 9, 14), 3, border=False)
    verts, faces = host_marching_cubes(lib, vol, LEVEL)
    bnd = boundary_edges(faces)
    assert len(bnd) > 0
    p, q = verts[bnd[:, 0]], verts[bnd[:, 1]]
    hi = np.array(vol.shape, dtype=np.float32) - 1
    on = ((p == 0) & (q == 0)) | ((p == hi) & (q == hi))
    assert on.any(axis=1).all()


def test_sphere_and_torus_topology(lib):
    sp = (0.8, 1.1, 0.9)
    vol = sphere_volume(spacing=sp)
    verts, faces = host_marching_cubes(lib, vol, LEVEL, sp)
    assert_closed(faces)
    assert euler(verts, faces) == 2
    want = 4 / 3 * np.pi * 6.5 ** 3
    vol_got = -signed_volume(verts, faces)                # skimage's winding: normals point into the dense region
    assert abs(vol_got - want) < 0.02 * want, (vol_got, want)
    verts, faces = host_marching_cubes(lib, torus_volume(), LEVEL)
    assert_closed(faces)
    assert euler(verts, faces) == 0
    assert signed_volume(verts, faces) < 0


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_exported_ply_faces_outward(lib, name, tmp_path, monkeypatch, capsys):
    """convert_sdf_samples_to_ply reverses marching_cubes' winding as the reference does: the file's closed surface
    has positive signed volume, equal in size to the volume enclosed by the marching-cubes mesh"""
    vol = sphere_volume() if name == "sphere" else torus_volume()
    monkeypatch.setattr(mesh, "marching_cubes", lambda v, level, spacing: tuple(
        torch.from_numpy(x) for x in host_marching_cubes(lib, v.numpy(), level, spacing)))
    bbox = torch.tensor([[-1.0, -0.5, -2.0], [1.5, 2.0, 1.0]])
    path = tmp_path / "mesh.ply"
    mesh.convert_sdf_samples_to_ply(torch.from_numpy(vol), str(path), bbox=bbox, level=LEVEL)
    capsys.readouterr()
    verts, faces = mesh.read_ply(str(path))
    assert_closed(faces)
    sp = [float(v) for v in mesh.ply_spacing(vol.shape, bbox)]
    mv, mf = host_marching_cubes(lib, vol, LEVEL, sp)
    got, inner = signed_volume(verts, faces), -signed_volume(mv, mf)
    assert got > 0 and abs(got - inner) < 1e-4 * inner, (got, inner)


def test_saddles_take_both_decider_outcomes(lib):
    vol = saddle_volume()
    verts, faces = host_marching_cubes(lib, vol, LEVEL)
    assert_closed(faces)
    # both outcomes of the decider occur on the ambiguous z-normal faces (u = x, w = y) of this volume
    v00, v10, v01, v11 = vol[:-1, :-1], vol[1:, :-1], vol[:-1, 1:], vol[1:, 1:]
    ins = [x > np.float32(LEVEL) for x in (v00, v10, v01, v11)]
    amb = (ins[0] == ins[3]) & (ins[1] == ins[2]) & (ins[0] != ins[1])
    dec = MO._decider(v00, v10, v01, v11, LEVEL)
    assert amb.sum() > 50 and (amb & dec).sum() > 10 and (amb & ~dec).sum() > 10


def _near_ties(n, seed=5):
    """ambiguous face values (v00, v10, v01, v11) whose fp32 decision depends on the order of the denominator's sum:
    the two cells of a face must evaluate the decider on the same order of values"""
    g = np.random.default_rng(seed)
    f, L = np.float32, np.float32(LEVEL)
    out = []
    while len(out) < n:
        a, c, b = (g.random(3) * 0.4 + 0.05).astype(np.float32)
        d = f(a * c / b)
        if not (0 < d < 0.45):
            continue
        v00, v11, v10, v01 = f(L + a), f(L + c), f(L - b), f(L - d)
        num = v00 * v11 - v10 * v01
        one = ((v00 + v11) - v10) - v01
        two = ((v00 + v11) - v01) - v10
        if (num / one > L) != (num / two > L):
            out.append((v00, v10, v01, v11))
    return out


def test_near_tie_faces_keep_the_mesh_closed(lib):
    """a slab of cells along x whose shared x-faces are ambiguous near-ties: interior faces must pair up"""
    ties = _near_ties(48)
    for v00, v10, v01, v11 in ties:      # the decider itself, on the canonical order, equals the oracle's
        assert lib.mc_host_face_connected(v00, v10, v01, v11, LEVEL) == int(MO._decider(v00, v10, v01, v11, LEVEL))
    vol = np.zeros((len(ties), 2, 2), dtype=np.float32)
    for i, (v00, v10, v01, v11) in enumerate(ties):
        vol[i] = [[v00, v01], [v10, v11]]       # (y, z): y is the face's lower axis u, z its w
    verts, faces = host_marching_cubes(lib, vol, LEVEL)
    bnd = boundary_edges(faces)
    p, q = verts[bnd[:, 0]], verts[bnd[:, 1]]
    hi = np.array(vol.shape, dtype=np.float32) - 1
    on = ((p == 0) & (q == 0)) | ((p == hi) & (q == hi))
    assert on.any(axis=1).all(), "an interior face's segments do not pair up"
    ov, of = MO.marching_cubes(vol, LEVEL)
    assert np.array_equal(faces, of)


def test_level_out_of_range_and_empty(lib):
    vol = random_volume((5, 6, 7), 1)
    for level in (-0.1, 1.5, float(vol.max()) + 1e-3):
        with pytest.raises(ValueError, match="Surface level must be within volume data range."):
            host_marching_cubes(lib, vol, level)
    verts, faces = host_marching_cubes(lib, vol, float(vol.max()))     # no point above the level
    assert verts.shape == (0, 3) and faces.shape == (0, 3) and faces.dtype == np.int32
    with pytest.raises(ValueError):
        host_marching_cubes(lib, vol[:1], 0.5)


def test_abi_argument_checks(lib):
    n = C.c_int64(0)
    assert lib.tir_marching_cubes_work_size(1, 5, 5, C.byref(n)) == -2
    assert lib.tir_marching_cubes_work_size(5, 5, 5, None) == -1
    assert lib.tir_marching_cubes_work_size(2048, 2048, 1024, C.byref(n)) == -2     # > INT32_MAX points
    assert lib.tir_marching_cubes_work_size(4, 5, 6, C.byref(n)) == 0
    vol = torch.zeros(4, 5, 6)
    work = torch.zeros(n.value, dtype=torch.uint8)
    tot = torch.zeros(2, dtype=torch.int64)
    p = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731
    assert lib.tir_marching_cubes_count(p(vol), 4, 5, 6, 0.5, p(work), n.value - 1, p(tot), None) == -4
    assert lib.tir_marching_cubes_emit(p(vol), 4, 5, 6, 0.5, 1., 1., 1., p(work), n.value, 2 ** 31, 0, None, None,
                                       None) == -2
    assert lib.tir_marching_cubes_emit(p(vol), 4, 5, 6, 0.5, 1., 1., 1., p(work), n.value, 3, 0, None, None,
                                       None) == -1


# ---- the reference's post-processing and PLY file (tests/golden/mesh_reference.pt) --------------------------------

@pytest.fixture(scope="module")
def golden_mesh():
    from gpu_helpers import load_fixture
    return load_fixture("mesh_reference.pt")


@pytest.mark.parametrize("model", ["rotated", "A", "B"])
def test_reference_post_processing(golden_mesh, model, tmp_path, monkeypatch, capsys):
    fx, rec = golden_mesh, golden_mesh["models"][model]
    seen = {}

    def standin(volume, level, spacing=(1., 1., 1.)):
        seen.update(shape=tuple(volume.shape), level=level, spacing=list(spacing))
        return fx["standin_verts"].clone(), fx["standin_faces"].clone()
    monkeypatch.setattr(mesh, "marching_cubes", standin)
    path = tmp_path / "mesh.ply"
    mesh.convert_sdf_samples_to_ply(rec["volume"], str(path), bbox=rec["aabb"], level=fx["level"])
    assert capsys.readouterr().out == f"saving mesh to {path}\n"
    assert seen["shape"] == rec["mc_shape"] and seen["level"] == rec["mc_level"]
    assert seen["spacing"] == rec["mc_spacing"]                    # (bbox[1]-bbox[0]) / N, bit for bit
    data = path.read_bytes()
    V, F = rec["vertex_records"].shape[0], rec["face_records"].shape[0]
    head = HEADER.replace(b"{V}", str(V).encode()).replace(b"{F}", str(F).encode())
    assert data[:len(head)] == head
    verts, faces = mesh.read_ply(str(path))
    assert np.array_equal(verts.view(np.uint32), rec["vertex_records"].numpy().view(np.uint32))
    assert np.array_equal(faces, rec["face_records"].numpy())       # the reference's faces[..., ::-1]
    body = np.frombuffer(data[len(head):], dtype=np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4")]), count=V)
    assert np.array_equal(np.stack([body["x"], body["y"], body["z"]], -1), verts)


def test_ply_scale_and_offset_follow_numpy():
    verts = torch.tensor([[0.1, 0.2, 0.3], [1.7, 2.9, 0.004]])
    faces = torch.tensor([[0, 1, 1]], dtype=torch.int32)
    bbox = torch.tensor([[-1.5, -1.25, -0.75], [1.5, 1.0, 0.5]])
    for scale, offset in ((2.5, None), (None, np.array([0.1, 0.2, 0.3])), (np.float64(3.0), 0.7)):
        got, _ = _parse(mesh.ply_bytes(verts, faces, bbox, offset=offset, scale=scale))
        mp = np.zeros((2, 3), np.float32)
        for c in range(3):
            mp[:, c] = bbox[0, c] + verts.numpy()[:, c]
        if scale is not None:
            mp = mp / scale
        if offset is not None:
            mp = mp - offset
        assert np.array_equal(got, mp.astype(np.float32))


def _parse(data):
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode().split("\n")
    V = int(head[2].split()[-1])
    return np.frombuffer(data, "<f4", 3 * V, end).reshape(V, 3), data[end + 12 * V:]
