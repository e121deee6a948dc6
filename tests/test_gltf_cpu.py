"""Textured glTF export on the CPU, through the host twin of csrc/tir_atlas.cu (tests/host_atlas.cpp, the same body
header): the atlas layout and its no-bleed guarantee, the texel enumeration, the probe points against float64, the
encoding and tangent frames against glTF's decoding rules, the winding, and the .glb writer and reader."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

from helpers import build_host_lib, on_host
from mesh_helpers import host_marching_cubes, sphere_volume
from tensoir_b200 import _lib, gltf


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = build_host_lib(tmp_path_factory.mktemp("host_atlas"), "host_atlas.cpp")
    lib.at_host_frame.restype = C.c_int
    lib.at_host_frame.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    return lib


def random_mesh(F, V=None, seed=0):
    """faces [F,3] int32 (marching_cubes winding) on random positions v [V,3] float32"""
    g = np.random.default_rng(seed)
    V = V or max(3, F // 2 + 3)
    v = g.normal(size=(V, 3)).astype(np.float32)
    faces = np.stack([g.choice(V, 3, replace=False) for _ in range(F)]).astype(np.int32)
    return torch.from_numpy(faces), torch.from_numpy(v)


def owned(s, side):
    """the (i, j) a face owns in its cell, as the layout states it"""
    i, j = np.meshgrid(np.arange(s), np.arange(s), indexing="ij")
    m = i + j <= s - 2 if side == 0 else i + j >= s
    return set(zip(i[m].tolist(), j[m].tolist()))


def srgb64(c):
    c = np.clip(np.nan_to_num(c.astype(np.float64), nan=0.0), 0, 1)
    return np.where(c <= 0.0031308, 12.92 * c, 1.055 * c ** (1 / 2.4) - 0.055)


# ---- 1. the no-bleed guarantee ----------------------------------------------------------------------------------------

def test_no_bleed_guarantee_for_every_cell_size(lib):
    T = 256
    faces, v = random_mesh(2, seed=1)
    for s in range(6, 65):
        q = s * (s - 1) // 2
        with on_host(lib):
            pix, _ = gltf.atlas_texels(faces, v, T, s, 0, 2 * q)
            uv = gltf.atlas_corners(faces, v, T, s)["TEXCOORD_0"].double().numpy()
        sets = []
        for side in (0, 1):
            p = pix[side * q:(side + 1) * q].numpy()
            got = set(zip((p % T).tolist(), (p // T).tolist()))
            assert got == owned(s, side), s
            sets.append(got)
        assert not sets[0] & sets[1]
        assert not any(i + j == s - 1 for i, j in sets[0] | sets[1])
        xy = uv * T - 0.5                                   # texel-centre coordinates of the corners
        assert np.array_equal(xy, np.round(xy))
        m = 256                     # a power of two: the grid points, edges and corners included, are exact
        a, b = np.meshgrid(np.arange(m + 1), np.arange(m + 1), indexing="ij")
        keep = a + b <= m
        a, b = a[keep][:, None], b[keep][:, None]
        rnd = np.random.default_rng(s).dirichlet((1, 1, 1), 2000)
        for side in (0, 1):
            c = xy[3 * side:3 * side + 3]
            pts = np.concatenate([(c[0] * m + a * (c[1] - c[0]) + b * (c[2] - c[0])) / m, rnd @ c])
            x0, y0 = np.floor(pts[:, 0]), np.floor(pts[:, 1])
            fx, fy = pts[:, 0] - x0, pts[:, 1] - y0
            for dx in (0, 1):
                for dy in (0, 1):
                    w = (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
                    tx, ty = (x0 + dx)[w > 0].astype(int), (y0 + dy)[w > 0].astype(int)
                    assert set(zip(tx.tolist(), ty.tolist())) <= sets[side], (s, side)


# ---- 2. enumeration and cell size -------------------------------------------------------------------------------------

@pytest.mark.parametrize("F,T", [(7, 256), (2000, 256), (5001, 512)])
def test_enumeration_is_a_bijection_onto_the_owned_texels(lib, F, T):
    faces, v = random_mesh(F, seed=F)
    s = gltf.atlas_cell_size(F, T)
    q, P = s * (s - 1) // 2, T // s
    with on_host(lib):
        pix, _ = gltf.atlas_texels(faces, v, T, s, 0, gltf.texel_count(F, s))
    pix = pix.numpy().astype(np.int64)
    assert len(np.unique(pix)) == len(pix) == F * q
    f = np.arange(F * q) // q
    c = f // 2
    x, y = pix % T - s * (c % P), pix // T - s * (c // P)
    assert ((x >= 0) & (x < s) & (y >= 0) & (y < s)).all()
    want = set()
    for face in range(F):
        cx, cy = s * (face // 2 % P), s * (face // 2 // P)
        want |= {(cy + j) * T + cx + i for i, j in owned(s, face & 1)}
    assert set(pix.tolist()) == want
    # a range in the middle gives the same texels
    with on_host(lib):
        part, _ = gltf.atlas_texels(faces, v, T, s, q + 3, 50)
    assert np.array_equal(part.numpy(), pix[q + 3:q + 53])


def test_cell_size_choice():
    assert gltf.atlas_cell_size(476680, 4096) == 8
    assert gltf.texel_count(476680, 8) == 13347040
    for F, T in [(1, 256), (2, 256), (17, 256), (1000, 256), (5001, 512), (476680, 8192), (900000, 4096)]:
        s = gltf.atlas_cell_size(F, T)
        assert 6 <= s <= 64 and (T // s) ** 2 >= (F + 1) // 2
        assert s == 64 or (T // (s + 1)) ** 2 < (F + 1) // 2
    with pytest.raises(ValueError, match="smallest texture size that fits is 4096"):
        gltf.atlas_cell_size(476680, 2048)
    with pytest.raises(ValueError, match="no texture size up to 8192 fits"):
        gltf.atlas_cell_size(2 * 1366 ** 2 + 2, 8192)
    for T in (128, 300, 16384):
        with pytest.raises(ValueError, match="power of two"):
            gltf.atlas_cell_size(10, T)


# ---- 3. probe points ----------------------------------------------------------------------------------------------------

def closest_bary(p, c):
    """float64 barycentrics of the point of triangle c [3,2] nearest to each p [n,2]"""
    def bary(q):
        m = np.stack([c[1] - c[0], c[2] - c[0]], 1)
        b12 = np.linalg.solve(m, (q - c[0]).T).T
        return np.concatenate([1 - b12.sum(1, keepdims=True), b12], 1)
    b = bary(p)
    out = b.copy()
    outside = (b < 0).any(1)
    best = np.full(len(p), np.inf)
    for i, j in ((0, 1), (1, 2), (2, 0)):
        e = c[j] - c[i]
        t = np.clip(((p - c[i]) @ e) / (e @ e), 0, 1)
        q = c[i] + t[:, None] * e
        d = np.linalg.norm(p - q, axis=1)
        nb = np.zeros((len(p), 3))
        nb[:, i], nb[:, j] = 1 - t, t
        take = outside & (d < best)
        out[take], best[take] = nb[take], d[take]
    return out


def test_positions_against_float64_and_corner_texels_exact(lib):
    F, T = 300, 256
    faces, v = random_mesh(F, seed=5)
    s = gltf.atlas_cell_size(F, T)
    q = s * (s - 1) // 2
    with on_host(lib):
        pix, pos = gltf.atlas_texels(faces, v, T, s, 0, F * q)
        uv = gltf.atlas_corners(faces, v, T, s)["TEXCOORD_0"].double().numpy().reshape(F, 3, 2)
    pix, pos = pix.numpy(), pos.numpy()
    v64 = v.double().numpy()
    corner_hits = 0
    for f in range(F):
        c = uv[f] * T - 0.5
        rows = slice(f * q, (f + 1) * q)
        p = np.stack([pix[rows] % T, pix[rows] // T], 1).astype(np.float64)
        b = closest_bary(p, c)
        ids = faces[f].numpy()[::-1]
        want = b @ v64[ids]
        err = np.abs(pos[rows] - want)
        assert (err <= 4 * np.finfo(np.float32).eps * np.abs(v64[ids]).max()).all(), f
        for k in range(3):
            hit = (p == c[k]).all(1)
            assert hit.sum() == 1
            assert np.array_equal(pos[rows][hit][0].view(np.uint32), v.numpy()[ids[k]].view(np.uint32))
            corner_hits += 1
    assert corner_hits == 3 * F


# ---- 4. encoding and tangent frames ----------------------------------------------------------------------------------

def _encode(lib, faces, v, T, s, albedo, rough, normal, probed):
    img = gltf.new_images(T, "cpu")
    with on_host(lib):
        gltf.atlas_encode(faces, v, T, s, 0, albedo, rough, normal, probed, img)
        pix, _ = gltf.atlas_texels(faces, v, T, s, 0, albedo.shape[0])
    return img.numpy().reshape(3, T * T, 4), pix.numpy()


def test_base_color_and_roughness_bytes(lib):
    F, T = 2000, 256
    faces, v = random_mesh(F, seed=7)
    s = gltf.atlas_cell_size(F, T)
    n = gltf.texel_count(F, s)
    g = np.random.default_rng(0)
    alb = g.uniform(-0.1, 1.1, (n, 3)).astype(np.float32)
    alb[:300] = g.uniform(0, 0.01, (300, 3))                          # the linear segment and its joint
    alb[300, 0], alb[301, 1], alb[302, 2] = np.nan, np.inf, -np.inf
    rough = g.uniform(-0.1, 1.1, n).astype(np.float32)
    probed = g.random(n) < 0.9
    normal = torch.nn.functional.normalize(torch.randn(n, 3, generator=torch.Generator().manual_seed(1)), dim=-1)
    img, pix = _encode(lib, faces, v, T, s, torch.from_numpy(alb), torch.from_numpy(rough), normal,
                       torch.from_numpy(probed))
    base, mr, nm = img[0][pix], img[1][pix], img[2][pix]
    want = np.where(probed[:, None], np.clip(np.round(srgb64(alb) * 255), 0, 255), 0)
    assert np.abs(base[:, :3].astype(int) - want).max() <= 1
    assert (base[:, 3] == 255).all()
    r32 = np.where(probed, np.clip(rough, 0, 1), np.float32(1)).astype(np.float32)
    assert np.array_equal(mr[:, 1], np.floor(r32 * np.float32(255) + np.float32(0.5)).astype(np.uint8))
    assert (mr[:, 0] == 255).all() and (mr[:, 2] == 0).all() and (mr[:, 3] == 255).all()
    assert (nm[:, 3] == 255).all()
    # every other texel keeps its default
    rest = np.ones(T * T, bool)
    rest[pix] = False
    for k, rgba in enumerate(gltf.IMAGE_DEFAULTS):
        assert (img[k][rest] == np.array(rgba, np.uint8)).all()


def _frames(lib, faces, v):
    out = np.zeros((faces.shape[0], 7), np.float32)
    deg = np.zeros(faces.shape[0], bool)
    for f in range(faces.shape[0]):
        deg[f] = lib.at_host_frame(faces.numpy().ctypes.data, f, v.numpy().ctypes.data, out[f].ctypes.data) == 1
    return out, deg


def test_normal_map_decodes_through_the_file_frames(lib, tmp_path):
    F, T = 400, 256
    faces, v = random_mesh(F, seed=11)
    s = gltf.atlas_cell_size(F, T)
    n = gltf.texel_count(F, s)
    g = torch.Generator().manual_seed(2)
    normal = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    img, pix = _encode(lib, faces, v, T, s, torch.rand(n, 3, generator=g), torch.rand(n, generator=g), normal,
                       torch.ones(n, dtype=torch.bool))
    with on_host(lib):
        corners = {k: t.numpy() for k, t in gltf.atlas_corners(faces, v, T, s).items()}
    path = tmp_path / "m.glb"
    path.write_bytes(gltf.glb_bytes(corners, [gltf.png_bytes(i.reshape(T, T, 4)) for i in img]))
    got = gltf.read_glb(str(path))
    N = got["accessors"][1][0::3].astype(np.float64)
    Tw = got["accessors"][2][0::3].astype(np.float64)
    face = np.arange(n) // (s * (s - 1) // 2)
    x = got["images"][2].reshape(-1, 4)[pix, :3].astype(np.float64) / 255 * 2 - 1
    Nf, Tf = N[face], Tw[face, :3]
    B = np.cross(Nf, Tf) * Tw[face, 3:]
    dec = Tf * x[:, :1] + B * x[:, 1:2] + Nf * x[:, 2:]
    dec /= np.linalg.norm(dec, axis=1, keepdims=True)
    err = np.linalg.norm(dec - normal.double().numpy(), axis=1)
    assert err.max() <= 2 * np.sqrt(3) / 255, err.max()


def test_tangent_frames(lib):
    F, T = 200, 256
    faces, v = random_mesh(F, seed=13)
    faces[5] = torch.tensor([1, 1, 2])                             # two corners on one vertex
    v[7:10] = torch.tensor([[0.0, 0, 0], [1, 1, 1], [2, 2, 2]])    # collinear corners
    faces[6] = torch.tensor([7, 8, 9])
    s = gltf.atlas_cell_size(F, T)
    with on_host(lib):
        c = {k: t.double().numpy() for k, t in gltf.atlas_corners(faces, v, T, s).items()}
    fr, deg = _frames(lib, faces, v)
    assert deg[5] and deg[6] and deg.sum() == 2
    N, Tw = c["NORMAL"][0::3], c["TANGENT"][0::3]
    assert np.array_equal(np.concatenate([N, Tw], 1).astype(np.float32), fr)
    assert np.array_equal(c["NORMAL"][1::3], N) and np.array_equal(c["TANGENT"][2::3], Tw)
    assert (N[deg] == [0, 0, 1]).all() and (Tw[deg] == [1, 0, 0, 1]).all()
    ok = ~deg
    assert np.abs(np.linalg.norm(Tw[ok, :3], axis=1) - 1).max() < 1e-6
    assert np.abs(np.linalg.norm(N[ok], axis=1) - 1).max() < 1e-6
    assert np.abs((N[ok] * Tw[ok, :3]).sum(1)).max() < 1e-6
    assert set(np.unique(Tw[:, 3])) <= {-1.0, 1.0}
    # dP/du and dP/dv by finite differences of the affine UV -> P map of each face
    P = c["POSITION"].reshape(F, 3, 3)
    UV = c["TEXCOORD_0"].reshape(F, 3, 2)
    h = 1e-3
    for f in np.nonzero(ok)[0]:
        m = np.stack([UV[f, 1] - UV[f, 0], UV[f, 2] - UV[f, 0]], 1)

        def at(uv):
            b = np.linalg.solve(m, uv - UV[f, 0])
            return P[f, 0] + b[0] * (P[f, 1] - P[f, 0]) + b[1] * (P[f, 2] - P[f, 0])
        mid = UV[f].mean(0)
        du = (at(mid + [h, 0]) - at(mid - [h, 0])) / (2 * h)
        dv = (at(mid + [0, h]) - at(mid - [0, h])) / (2 * h)
        t = Tw[f, :3]
        assert np.dot(t, du / np.linalg.norm(du)) > 1 - 1e-5, f
        up = -dv - np.dot(-dv, t) * t
        bt = np.cross(N[f], t) * Tw[f, 3]
        assert np.dot(bt, up / np.linalg.norm(up)) > 1 - 1e-5, f


# ---- 5. winding ----------------------------------------------------------------------------------------------------------

def test_triangles_face_outward_on_the_sphere(lib, tmp_path):
    shape = (41, 37, 45)
    mesh_lib = build_host_lib(tmp_path, "host_mesh.cpp")
    verts, faces = host_marching_cubes(mesh_lib, sphere_volume(shape), 0.5)
    F = faces.shape[0]
    T = 256 if (256 // 6) ** 2 >= (F + 1) // 2 else 512
    s = gltf.atlas_cell_size(F, T)
    with on_host(lib):
        c = gltf.atlas_corners(torch.from_numpy(faces), torch.from_numpy(verts), T, s)
    P = c["POSITION"].double().numpy().reshape(F, 3, 3)
    nrm = np.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0])
    ok = np.linalg.norm(nrm, axis=1) > 1e-9
    centre = np.array([(n - 1) / 2 for n in shape])
    assert ok.sum() > 0.99 * F
    assert ((nrm[ok] * (P[ok].mean(1) - centre)).sum(1) > 0).all()
    N = c["NORMAL"].double().numpy()[0::3]
    assert ((N[ok] * (P[ok].mean(1) - centre)).sum(1) > 0).all()


# ---- 6. the .glb file --------------------------------------------------------------------------------------------------

def _hand_glb(lib, F=9, T=256):
    faces, v = random_mesh(F, seed=17)
    s = gltf.atlas_cell_size(F, T)
    n = gltf.texel_count(F, s)
    g = torch.Generator().manual_seed(3)
    img, _ = _encode(lib, faces, v, T, s, torch.rand(n, 3, generator=g), torch.rand(n, generator=g),
                     torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1),
                     torch.rand(n, generator=g) < 0.8)
    img = img.reshape(3, T, T, 4)
    with on_host(lib):
        corners = {k: t.numpy() for k, t in gltf.atlas_corners(faces, v, T, s).items()}
    return gltf.glb_bytes(corners, [gltf.png_bytes(i) for i in img]), corners, img


def test_glb_structure(lib, tmp_path):
    import json
    data, corners, img = _hand_glb(lib)
    magic, version, length = struct.unpack_from("<III", data)
    assert (magic, version, length) == (0x46546C67, 2, len(data))
    jlen, jtype = struct.unpack_from("<II", data, 12)
    assert jtype == 0x4E4F534A and jlen % 4 == 0
    js = data[20:20 + jlen]
    assert js == js.rstrip(b" ") + b" " * (len(js) - len(js.rstrip(b" ")))
    doc = json.loads(js)
    blen, btype = struct.unpack_from("<II", data, 20 + jlen)
    assert btype == 0x004E4942 and blen % 4 == 0 and 28 + jlen + blen == len(data)
    body = data[28 + jlen:]
    assert doc["asset"]["version"] == "2.0"
    assert doc["buffers"] == [{"byteLength": blen}]
    for bv in doc["bufferViews"]:
        assert bv["byteOffset"] % 4 == 0 and bv["byteOffset"] + bv["byteLength"] <= blen
        assert body[bv["byteOffset"] + bv["byteLength"]:(bv["byteOffset"] + bv["byteLength"] + 3) // 4 * 4] \
            == b"\0" * ((4 - bv["byteLength"] % 4) % 4)
    prim = doc["meshes"][0]["primitives"][0]
    assert prim["mode"] == 4 and "indices" not in prim
    assert set(prim["attributes"]) == {"POSITION", "NORMAL", "TANGENT", "TEXCOORD_0"}
    for name, typ, k in gltf.ATTRIBUTES:
        acc = doc["accessors"][prim["attributes"][name]]
        assert (acc["count"], acc["type"], acc["componentType"]) == (27, typ, 5126)
        bv = doc["bufferViews"][acc["bufferView"]]
        assert bv["target"] == 34962
        raw = np.frombuffer(body, "<f4", 27 * k, bv["byteOffset"]).reshape(27, k)
        assert np.array_equal(raw, corners[name])
    pos = doc["accessors"][prim["attributes"]["POSITION"]]
    assert pos["min"] == corners["POSITION"].min(0).tolist() and pos["max"] == corners["POSITION"].max(0).tolist()
    assert doc["samplers"] == [{"magFilter": 9729, "minFilter": 9729, "wrapS": 33071, "wrapT": 33071}]
    assert doc["nodes"] == [{"mesh": 0, "matrix": [1, 0, 0, 0, 0, 0, -1, 0, 0, 1, 0, 0, 0, 0, 0, 1]}]
    M = np.array(doc["nodes"][0]["matrix"], float).reshape(4, 4).T          # column-major
    assert np.array_equal(M[:3, :3] @ [1.0, 2.0, 3.0], [1.0, 3.0, -2.0])
    mat = doc["materials"][0]
    assert mat["doubleSided"] is False and mat["normalTexture"] == {"index": 2}
    pbr = mat["pbrMetallicRoughness"]
    assert pbr["baseColorTexture"] == {"index": 0} and pbr["metallicRoughnessTexture"] == {"index": 1}
    assert pbr["metallicFactor"] == 1 and pbr["roughnessFactor"] == 1
    assert all(im["mimeType"] == "image/png" for im in doc["images"]) and len(doc["images"]) == 3
    path = tmp_path / "hand.glb"
    path.write_bytes(data)
    got = gltf.read_glb(str(path))
    assert got["json"] == doc
    for k in range(3):
        assert np.array_equal(got["images"][k], img[k])
    for i, (name, _, _) in enumerate(gltf.ATTRIBUTES):
        assert np.array_equal(got["accessors"][i], corners[name])


def test_read_glb_rejects_malformed_files(lib, tmp_path):
    data, _, _ = _hand_glb(lib)
    cases = {"truncated": data[:-8], "header": data[:10], "magic": b"gltf" + data[4:],
             "version": data[:4] + struct.pack("<I", 1) + data[8:],
             "json tag": data[:16] + struct.pack("<I", 0x4E4F534B) + data[20:]}
    jlen = struct.unpack_from("<I", data, 12)[0]
    cases["bin tag"] = data[:24 + jlen] + struct.pack("<I", 0x004E4943) + data[28 + jlen:]
    for name, bad in cases.items():
        p = tmp_path / f"{name}.glb"
        p.write_bytes(bad)
        with pytest.raises(ValueError):
            gltf.read_glb(str(p))
    with pytest.raises(ValueError, match="positive multiple of 3"):
        gltf.glb_bytes({name: np.zeros((0, k), np.float32) for name, _, k in gltf.ATTRIBUTES}, [])


# ---- 7. argument checks ---------------------------------------------------------------------------------------------------

def _abi_checks(lib):
    p = C.c_void_p(16)
    assert lib.tir_atlas_texels(None, 10, None, 256, 8, 0, 5, None, None, None) == -1
    assert lib.tir_atlas_encode(None, 10, None, 256, 8, 0, 5, *[None] * 8) == -1
    assert lib.tir_atlas_corners(None, 10, None, 256, 8, *[None] * 5) == -1
    assert lib.tir_atlas_texels(p, 10, p, 256, 8, 0, 5, p, None, None) == -1
    # empty: no-ops
    assert lib.tir_atlas_texels(None, 10, None, 256, 8, 0, 0, None, None, None) == 0
    assert lib.tir_atlas_encode(None, 10, None, 256, 8, 0, 0, *[None] * 8) == 0
    assert lib.tir_atlas_corners(None, 0, None, 256, 8, *[None] * 5) == 0
    # negative sizes, a bad layout, a range past the last texel
    for F, T, s, first, n in [(10, 256, 8, 0, -1), (-1, 256, 8, 0, 5), (10, 256, 8, -1, 5), (10, 300, 8, 0, 5),
                              (10, 128, 8, 0, 5), (10, 256, 5, 0, 5), (10, 256, 65, 0, 5),
                              (2 * 43 ** 2 + 1, 256, 6, 0, 5), (10, 256, 8, 270, 11)]:
        assert lib.tir_atlas_texels(p, F, p, T, s, first, n, p, p, None) == -2, (F, T, s, first, n)
        assert lib.tir_atlas_encode(p, F, p, T, s, first, n, *[p] * 7, None) == -2
    assert lib.tir_atlas_corners(p, -1, p, 256, 8, *[p] * 4, None) == -2
    assert lib.tir_atlas_corners(p, 10, p, 256, 70, *[p] * 4, None) == -2


def test_argument_checks_host_twin(lib):
    _abi_checks(lib)


def test_argument_checks_library():
    import __graft_entry__ as g
    g.build()
    _abi_checks(_lib.load())
