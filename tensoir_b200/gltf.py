"""Textured glTF export of the relightable asset: ``export_asset``'s surface, materials and predicted normals as one
binary glTF 2.0 file (.glb) that standard renderers read, with the learned lighting as .hdr files beside it.

glTF's metallic-roughness material holds this model's BRDF: tir_ggx.h uses alpha = roughness^2 as glTF does, the
Fresnel term's F0 is ``fixed_fresnel`` (0.04 by default, glTF's dielectric value) and the diffuse term is Lambertian
albedo.  glTF has no per-vertex material, so albedo, roughness and the predicted normal are baked into three textures
of one UV atlas on the GPU (csrc/tir_atlas.cu; the layout, its no-bleed guarantee, the probe point of every texel and
the encoding are documented in csrc/tir_atlas_body.h):

  * every texel is one probe point on its face, probed as ``mesh.probe`` probes a vertex (derived normal, one
    eval-mode primary ray), in chunks, so that peak memory does not grow with the texture size;
  * base colour is the sRGB-encoded albedo, metallic-roughness holds roughness in G and metallic 0, and the normal
    texture holds the predicted normal in each face's tangent frame (glTF's +Y-up convention);
  * the mesh is unwelded: 3F vertices with POSITION, flat NORMAL, TANGENT and TEXCOORD_0.  POSITION holds the field
    positions, where the field's surface lies (``mesh.field_positions``), not the PLY's ``x y z``, which the reference
    scales by (N-1)/N toward bbox[0];
  * one node maps TensoIR's Z-up world to glTF's Y-up, (x, y, z) -> (x, z, -y); the vertex data stay in world units;
  * the sampler is LINEAR / LINEAR with CLAMP_TO_EDGE and no mipmaps: the layout keeps neighbouring faces apart only
    for bilinear lookups, and a mipmapped lookup would mix faces.

An external renderer shows the same materials, not the same image as ``relight()``: glTF's diffuse / Fresnel coupling
and its Smith term differ from TensoIR's, and image-based lighting is not part of core glTF (the .hdr files stay
beside the .glb).
"""
from __future__ import annotations

import json
import math
import struct

import numpy as np
import torch

from . import _lib, mesh

T_MIN, T_MAX = 256, 8192       # AT_T_MIN, AT_T_MAX
S_MIN, S_MAX = 6, 64           # AT_S_MIN, AT_S_MAX
TEXEL_CHUNK = 1 << 20          # texels probed per chunk
GLTF_F0 = 0.04                 # glTF's dielectric F0
GLB_MAGIC, GLB_VERSION = 0x46546C67, 2
CHUNK_JSON, CHUNK_BIN = 0x4E4F534A, 0x004E4942
FLOAT, ARRAY_BUFFER, TRIANGLES = 5126, 34962, 4
LINEAR, CLAMP_TO_EDGE = 9729, 33071
Y_UP = [1, 0, 0, 0, 0, 0, -1, 0, 0, 1, 0, 0, 0, 0, 0, 1]   # column-major: (x, y, z) -> (x, z, -y)
ATTRIBUTES = (("POSITION", "VEC3", 3), ("NORMAL", "VEC3", 3), ("TANGENT", "VEC4", 4), ("TEXCOORD_0", "VEC2", 2))
IMAGE_DEFAULTS = ((0, 0, 0, 255), (255, 255, 0, 255), (128, 128, 255, 255))   # unowned texels: base, MR, normal
N_COMPONENTS = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4}


def atlas_cell_size(F, T):
    """s, the largest cell size <= 64 with floor(T/s)^2 >= ceil(F/2), for F faces in a T x T atlas.  Raises
    ValueError when T is not a power of two in [256, 8192], or when s would be below 6, naming the smallest T that
    fits."""
    if T < T_MIN or T > T_MAX or T & (T - 1):
        raise ValueError(f"texture size {T} is not a power of two in [{T_MIN}, {T_MAX}]")
    cells = (F + 1) // 2
    for s in range(S_MAX, S_MIN - 1, -1):
        if (T // s) ** 2 >= cells:
            return s
    fits = [t for t in (1 << k for k in range(8, 14)) if (t // S_MIN) ** 2 >= cells]
    hint = f"the smallest texture size that fits is {fits[0]}" if fits else f"no texture size up to {T_MAX} fits"
    raise ValueError(f"{F} faces do not fit a {T}x{T} atlas with cells of at least {S_MIN} texels: {hint}")


def texel_count(F, s):
    """F * s(s-1)/2: the texels the faces own (face-major order)."""
    return F * (s * (s - 1) // 2)


def atlas_texels(faces, v, T, s, first, n):
    """tir_atlas_texels: texels [first, first+n) -> (pix [n] int32 = row * T + column, pos [n,3] their probe points)."""
    lib = _lib.load()
    pix = torch.empty(n, dtype=torch.int32, device=v.device)
    pos = torch.empty(n, 3, dtype=torch.float32, device=v.device)
    _lib.check(lib.tir_atlas_texels(_lib.dptr(faces, torch.int32), faces.shape[0], _lib.dptr(v), T, s, first, n,
                                    _lib.dptr(pix, torch.int32), _lib.dptr(pos), _lib.stream_ptr()),
               "tir_atlas_texels")
    return pix, pos


def new_images(T, device):
    """The three RGBA8 images [3,T,T,4] (base colour, metallic-roughness, normal) with the unowned-texel defaults."""
    img = torch.empty(3, T, T, 4, dtype=torch.uint8, device=device)
    for k, rgba in enumerate(IMAGE_DEFAULTS):
        img[k] = torch.tensor(rgba, dtype=torch.uint8, device=device)
    return img


def atlas_encode(faces, v, T, s, first, albedo, rough, normal, probed, images):
    """tir_atlas_encode: the bytes of texels [first, first+n) (n = albedo rows) into ``images`` [3,T,T,4] uint8."""
    lib = _lib.load()
    n = albedo.shape[0]
    # the inputs stay referenced until the call returns (dptr keeps no reference)
    ins = (albedo.contiguous(), rough.reshape(n).contiguous(), normal.contiguous(),
           probed.reshape(n).to(torch.uint8).contiguous())
    args = [_lib.dptr(t) for t in ins[:3]] + [_lib.dptr(ins[3], torch.uint8)]
    _lib.check(lib.tir_atlas_encode(_lib.dptr(faces, torch.int32), faces.shape[0], _lib.dptr(v), T, s, first, n, *args,
                                    *[_lib.dptr(images[k], torch.uint8) for k in range(3)], _lib.stream_ptr()),
               "tir_atlas_encode")


def atlas_corners(faces, v, T, s):
    """tir_atlas_corners -> {POSITION [3F,3], NORMAL [3F,3], TANGENT [3F,4], TEXCOORD_0 [3F,2]} float32."""
    lib = _lib.load()
    F = faces.shape[0]
    out = {name: torch.empty(3 * F, k, dtype=torch.float32, device=v.device) for name, _, k in ATTRIBUTES}
    _lib.check(lib.tir_atlas_corners(_lib.dptr(faces, torch.int32), F, _lib.dptr(v), T, s,
                                     *[_lib.dptr(out[name]) for name, _, _ in ATTRIBUTES], _lib.stream_ptr()),
               "tir_atlas_corners")
    return out


def probe_texels(tensoIR, pos, edits=None):
    """``mesh.probe`` at texel points ``pos`` [n,3] with their derived normals, then ``mesh.edit_vertices`` when
    ``edits`` is given -> (albedo [n,3], roughness [n], normal [n,3], probed [n] bool)."""
    p = mesh.probe(tensoIR, pos, mesh.vertex_normals(tensoIR, pos))
    albedo, rough = (p["albedo"], p["roughness"]) if edits is None else mesh.edit_vertices(p, pos, edits)
    return albedo, rough, p["normal"], p["probed"]


@torch.no_grad()
def bake(tensoIR, faces, v, T, s, edits=None, chunk=TEXEL_CHUNK):
    """The three textures of the atlas: every owned texel probed (``probe_texels``) and encoded, ``chunk`` texels at a
    time -> (images [3,T,T,4] uint8 on the device, unprobed texel count)."""
    images = new_images(T, v.device)
    total, unprobed = texel_count(faces.shape[0], s), 0
    for first in range(0, total, chunk):
        n = min(chunk, total - first)
        _, pos = atlas_texels(faces, v, T, s, first, n)
        albedo, rough, normal, probed = probe_texels(tensoIR, pos, edits)
        atlas_encode(faces, v, T, s, first, albedo, rough, normal, probed, images)
        unprobed += n - int(probed.sum())
    return images, unprobed


def png_bytes(rgba):
    """A PNG of an RGBA8 [H,W,4] array (cv2, which takes BGRA)."""
    import cv2
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(np.asarray(rgba)[..., [2, 1, 0, 3]]))
    if not ok:
        raise RuntimeError("cv2.imencode failed to encode a PNG")
    return buf.tobytes()


def _pad4(n):
    return (4 - n % 4) % 4


def glb_bytes(corners, pngs):
    """The .glb file of one unwelded, non-indexed triangle mesh: ``corners`` {POSITION, NORMAL, TANGENT, TEXCOORD_0}
    float32 host arrays of 3F rows and ``pngs`` the base-colour, metallic-roughness and normal PNGs."""
    arrays = [np.ascontiguousarray(corners[name], dtype="<f4").reshape(-1, k) for name, _, k in ATTRIBUTES]
    count = arrays[0].shape[0]
    if count == 0 or count % 3:
        raise ValueError(f"a glb mesh needs a positive multiple of 3 vertices, got {count}")
    blobs = [a.tobytes() for a in arrays] + list(pngs)
    views, offset = [], 0
    for i, b in enumerate(blobs):
        view = {"buffer": 0, "byteOffset": offset, "byteLength": len(b)}
        if i < len(arrays):
            view["target"] = ARRAY_BUFFER
        views.append(view)
        offset += len(b) + _pad4(len(b))
    accessors = [{"bufferView": i, "componentType": FLOAT, "count": count, "type": typ}
                 for i, (_, typ, _) in enumerate(ATTRIBUTES)]
    accessors[0]["min"] = [float(x) for x in arrays[0].min(0)]
    accessors[0]["max"] = [float(x) for x in arrays[0].max(0)]
    n_attr = len(arrays)
    doc = {
        "asset": {"version": "2.0", "generator": "tensoir_b200"},
        "scene": 0,
        "scenes": [{"nodes": [0]}],
        "nodes": [{"mesh": 0, "matrix": Y_UP}],
        "meshes": [{"primitives": [{"attributes": {name: i for i, (name, _, _) in enumerate(ATTRIBUTES)},
                                    "material": 0, "mode": TRIANGLES}]}],
        "materials": [{"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}, "baseColorFactor": [1, 1, 1, 1],
                                                "metallicRoughnessTexture": {"index": 1}, "metallicFactor": 1,
                                                "roughnessFactor": 1},
                       "normalTexture": {"index": 2}, "doubleSided": False}],
        "samplers": [{"magFilter": LINEAR, "minFilter": LINEAR, "wrapS": CLAMP_TO_EDGE, "wrapT": CLAMP_TO_EDGE}],
        "textures": [{"sampler": 0, "source": k} for k in range(len(pngs))],
        "images": [{"bufferView": n_attr + k, "mimeType": "image/png"} for k in range(len(pngs))],
        "accessors": accessors,
        "bufferViews": views,
        "buffers": [{"byteLength": offset}],
    }
    js = json.dumps(doc, separators=(",", ":")).encode("utf-8")
    js += b" " * _pad4(len(js))
    body = b"".join(b + b"\0" * _pad4(len(b)) for b in blobs)
    total = 12 + 8 + len(js) + 8 + len(body)
    return (struct.pack("<III", GLB_MAGIC, GLB_VERSION, total) + struct.pack("<II", len(js), CHUNK_JSON) + js
            + struct.pack("<II", len(body), CHUNK_BIN) + body)


def read_glb(path):
    """Parse a .glb written by ``export_asset_glb`` (or any glTF 2.0 binary with float accessors and PNG images in its
    BIN chunk) -> {"json": the glTF JSON, "accessors": [array per accessor, float32 [count, components]], "images":
    [RGBA8 [H,W,4] uint8 per image]}.  Raises ValueError for a malformed file: a wrong magic, version or length,
    missing or mistyped chunks, or a view, accessor or image outside the BIN chunk."""
    import cv2
    with open(path, "rb") as f:
        data = f.read()

    def bad(msg):
        return ValueError(f"{path}: {msg}")
    if len(data) < 20:
        raise bad(f"{len(data)} bytes is shorter than a glb header")
    magic, version, length = struct.unpack_from("<III", data, 0)
    if magic != GLB_MAGIC:
        raise bad("not a glb file (wrong magic)")
    if version != GLB_VERSION:
        raise bad(f"glb version {version}, expected {GLB_VERSION}")
    if length != len(data):
        raise bad(f"header length {length} but the file has {len(data)} bytes")
    chunks, off = [], 12
    while off < len(data):
        if off + 8 > len(data):
            raise bad("truncated chunk header")
        n, typ = struct.unpack_from("<II", data, off)
        if n % 4 or off + 8 + n > len(data):
            raise bad(f"chunk at byte {off} of {n} bytes is misaligned or runs past the end")
        chunks.append((typ, data[off + 8:off + 8 + n]))
        off += 8 + n
    if not chunks or chunks[0][0] != CHUNK_JSON:
        raise bad("the first chunk is not JSON")
    try:
        doc = json.loads(chunks[0][1].decode("utf-8"))
    except (UnicodeDecodeError, json.JSONDecodeError) as e:
        raise bad(f"the JSON chunk does not parse: {e}") from None
    bin_ = chunks[1][1] if len(chunks) > 1 else b""
    if len(chunks) > 1 and chunks[1][0] != CHUNK_BIN:
        raise bad("the second chunk is not BIN")
    if doc.get("asset", {}).get("version") != "2.0":
        raise bad("asset.version is not 2.0")

    def view(i):
        try:
            bv = doc["bufferViews"][i]
            lo, n = bv.get("byteOffset", 0), bv["byteLength"]
        except (KeyError, IndexError, TypeError):
            raise bad(f"bufferView {i} is missing or incomplete") from None
        if bv.get("buffer", 0) != 0 or lo < 0 or lo + n > len(bin_):
            raise bad(f"bufferView {i} lies outside the BIN chunk")
        return bin_[lo:lo + n]
    accessors = []
    for i, acc in enumerate(doc.get("accessors", [])):
        if acc.get("componentType") != FLOAT or acc.get("type") not in N_COMPONENTS:
            raise bad(f"accessor {i} is not a float scalar or vector")
        k, count = N_COMPONENTS[acc["type"]], acc["count"]
        raw = view(acc["bufferView"])
        start = acc.get("byteOffset", 0)
        if start + 4 * k * count > len(raw):
            raise bad(f"accessor {i} runs past its bufferView")
        accessors.append(np.frombuffer(raw, "<f4", k * count, start).reshape(count, k).copy())
    images = []
    for i, im in enumerate(doc.get("images", [])):
        if im.get("mimeType") != "image/png" or "bufferView" not in im:
            raise bad(f"image {i} is not a PNG in the BIN chunk")
        img = cv2.imdecode(np.frombuffer(view(im["bufferView"]), np.uint8), cv2.IMREAD_UNCHANGED)
        if img is None or img.ndim != 3 or img.shape[2] != 4:
            raise bad(f"image {i} does not decode to an RGBA image")
        images.append(np.ascontiguousarray(img[..., [2, 1, 0, 3]]))
    return {"json": doc, "accessors": accessors, "images": images}


@torch.no_grad()
def export_asset_glb(tensoIR, glb_path, level=0.005, texture_size=4096, envmaps=True, edits=None):
    """The relightable asset as a textured glTF: ``glb_path`` holds export_asset's surface (at the field positions) with
    the albedo, roughness and predicted normal baked into a texture_size^2 atlas (``bake``), and, with ``envmaps``,
    ``envmap_paths(glb_path, ...)`` the radiance of each light (for ``{ckpt[:-3]}_asset.glb`` the .hdr names of the
    PLY asset).  ``edits`` (MaterialEdit rules without fresnel ops) edit the probed texels as ``export_asset`` edits
    vertices.  Pass envmaps=False when the lights were not learned.  Nothing on the model changes.
    Returns (unprobed texel count, degenerate face count)."""
    from .relight import write_hdr
    if edits is not None:
        mesh._check_asset_edits(edits)
    _, faces, v = mesh.asset_surface(tensoIR, level)
    F = int(faces.shape[0])
    if F == 0:
        raise ValueError("the model has no surface at this level: nothing to export")
    s = atlas_cell_size(F, texture_size)
    if not math.isclose(float(tensoIR.fixed_fresnel), GLTF_F0):
        print(f"the model's fixed_fresnel is {float(tensoIR.fixed_fresnel)}, but glTF's dielectric F0 is {GLTF_F0}: "
              "the glb's specular reflectance uses 0.04")
    images, unprobed = bake(tensoIR, faces, v, texture_size, s, edits)
    corners = atlas_corners(faces, v, texture_size, s)
    fallback = torch.tensor([0, 0, 1, 1, 0, 0, 1], dtype=torch.float32, device=v.device)
    degenerate = int((torch.cat([corners["NORMAL"], corners["TANGENT"]], 1)[0::3] == fallback).all(1).sum())
    host = {k: t.cpu().numpy() for k, t in corners.items()}
    data = glb_bytes(host, [png_bytes(img) for img in images.cpu().numpy()])
    print(f"saving asset to {glb_path}: {F} faces, {texel_count(F, s)} texels ({texture_size}^2 atlas, cells of {s}), "
          f"{unprobed} unprobed texels, {degenerate} degenerate faces")
    with open(glb_path, "wb") as f:
        f.write(data)
    if envmaps:
        for path, rgb in zip(mesh.envmap_paths(glb_path, tensoIR.light_num), mesh.light_envmaps(tensoIR).cpu().numpy()):
            write_hdr(path, rgb)
    return unprobed, degenerate
