"""Mesh export: the reference's `scripts/export_mesh.py` / `--export_mesh 1` path (utils.py:165-225) on the GPU.

``marching_cubes`` runs the tir_marching_cubes_* kernels (csrc/tir_mesh.cu; topology, vertex placement and winding in
csrc/tir_mc_body.h) on a dense volume; ``convert_sdf_samples_to_ply`` keeps the reference's signature and
post-processing and writes the file plyfile writes for the reference's structured arrays; ``export_mesh`` is the
reference's export_mesh on a model.  There is no CPU fallback: a CPU volume is moved to the current CUDA device.

``export_asset`` writes a relightable asset: export_mesh's geometry with the recovered BRDF parameters and predicted
normal per vertex (from one eval-mode primary ray per vertex through the model's own forward), plus every learned
environment map as a Radiance .hdr.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib

PLY_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex {V}\nproperty float x\nproperty float y\n"
              "property float z\nelement face {F}\nproperty list uchar int vertex_indices\nend_header\n")
ASSET_PLY_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex {V}\nproperty float x\nproperty float y\n"
                    "property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
                    "property uchar green\nproperty uchar blue\nproperty float roughness\nproperty float albedo_r\n"
                    "property float albedo_g\nproperty float albedo_b\nproperty uchar probed\nelement face {F}\n"
                    "property list uchar int vertex_indices\nend_header\n")
ASSET_VERTEX = np.dtype([("xyz", "<f4", (3,)), ("normal", "<f4", (3,)), ("rgb", "u1", (3,)), ("roughness", "<f4"),
                         ("albedo", "<f4", (3,)), ("probed", "u1")])          # 44 bytes, no padding
FACE = np.dtype([("n", "u1"), ("v", "<i4", (3,))])
INT32_MAX = 2 ** 31 - 1
# probe rays start this many voxels outside their vertex (export_asset, DESIGN.md §3.3)
PROBE_OFFSET_VOXELS = 2.0
PROBE_ACC_THRESHOLD = 0.5          # acc_mask_threshold of relight_importance.py
PROBE_CHUNK = 65536
ENVMAP_HW = (256, 512)             # the evaluation's environment-map grid (renderer.py:183)


def marching_cubes(volume, level, spacing=(1., 1., 1.)):
    """Surface of {v > level} of a [X,Y,Z] volume -> (verts [V,3] float32, faces [F,3] int32) on the device.

    Vertex coordinates are (axis0, axis1, axis2) index coordinates times ``spacing``.  The winding is skimage's default
    (gradient_direction='descent'): a triangle's right-hand normal points toward higher values, into the dense region;
    convert_sdf_samples_to_ply reverses it, as the reference does, so the PLY faces outward.  Raises ValueError like
    skimage.measure.marching_cubes when ``level`` lies outside the volume's [min, max]; returns an empty mesh when no
    point is above ``level``."""
    if volume.dim() != 3:
        raise ValueError("Input volume should be a 3D numpy array.")
    if min(volume.shape) < 2:
        raise ValueError("Input array must be at least 2x2x2.")
    device = volume.device if volume.is_cuda else torch.device("cuda", torch.cuda.current_device())
    vol = volume.detach().to(device=device, dtype=torch.float32).contiguous()
    with torch.cuda.device(device):
        return extract(vol, level, spacing)


def extract(vol, level, spacing=(1., 1., 1.)):
    """marching_cubes on a contiguous float32 [X,Y,Z] tensor that already lives where the library runs."""
    lo, hi = torch.aminmax(vol)
    level = float(np.float32(level))
    if not (float(lo) <= level <= float(hi)):
        raise ValueError("Surface level must be within volume data range.")
    X, Y, Z = (int(s) for s in vol.shape)
    sp = [float(s) for s in spacing]
    if len(sp) != 3:
        raise ValueError("spacing must have three entries")
    lib = _lib.load()
    nbytes = C.c_int64(0)
    _lib.check(lib.tir_marching_cubes_work_size(X, Y, Z, C.byref(nbytes)), "tir_marching_cubes_work_size")
    work = torch.empty(nbytes.value, dtype=torch.uint8, device=vol.device)
    totals = torch.empty(2, dtype=torch.int64, device=vol.device)
    _lib.check(lib.tir_marching_cubes_count(_lib.dptr(vol), X, Y, Z, level, _lib.dptr(work, torch.uint8), nbytes.value,
                                            _lib.dptr(totals, torch.int64), _lib.stream_ptr()),
               "tir_marching_cubes_count")
    V, F = (int(t) for t in totals.tolist())
    if V > INT32_MAX or F > INT32_MAX:
        raise _lib.TirError(f"marching_cubes: {V} vertices / {F} faces do not fit int32 indices")
    verts = torch.empty(V, 3, dtype=torch.float32, device=vol.device)
    faces = torch.empty(F, 3, dtype=torch.int32, device=vol.device)
    if V or F:
        _lib.check(lib.tir_marching_cubes_emit(_lib.dptr(vol), X, Y, Z, level, sp[0], sp[1], sp[2],
                                               _lib.dptr(work, torch.uint8), nbytes.value, V, F, _lib.dptr(verts),
                                               _lib.dptr(faces, torch.int32), _lib.stream_ptr()),
                   "tir_marching_cubes_emit")
    return verts, faces


def ply_spacing(shape, bbox):
    """voxel_size of utils.py:184, ``(bbox[1] - bbox[0]) / np.array(shape)``, with its dtype: the divisor is N, not
    N-1, so the mesh is scaled by (N-1)/N toward bbox[0] compared with the sample grid (kept as in the reference)."""
    if torch.is_tensor(bbox):
        bbox = bbox.detach().cpu()
    return list((bbox[1] - bbox[0]) / np.array(shape))


def ply_positions(verts, bbox, offset=None, scale=None):
    """utils.py:189-208 after marching_cubes: bbox[0] + verts, then / scale and - offset with the reference's dtypes
    -> the float32 [V,3] ``x y z`` the PLY carries, where verts lives."""
    if torch.is_tensor(bbox):
        bbox = bbox.detach().cpu()
    b0 = torch.as_tensor(np.asarray(bbox[0]), dtype=torch.float32, device=verts.device)
    pts = verts + b0                       # bbox[0, c] + verts[:, c] on float32 (a 0-d tensor plus a float32 array)
    for op, arg in (("div", scale), ("sub", offset)):
        if arg is None:
            continue
        cur = np.empty(0, torch.empty(0, dtype=pts.dtype).numpy().dtype)
        dt = torch.from_numpy(np.empty(0, np.result_type(cur, arg))).dtype
        a = torch.as_tensor(np.asarray(arg), dtype=dt, device=pts.device)
        pts = pts.to(dt) / a if op == "div" else pts.to(dt) - a
    return pts.to(torch.float32).contiguous()


def face_records(faces):
    """The PLY face element of utils.py:210-222: faces[..., ::-1] (inverse face orientation), one 13-byte record
    (uchar 3, int32 x3) per face -> uint8 [F*13], where faces lives."""
    fl = faces.to(torch.int32).flip(-1).contiguous()
    F = fl.shape[0]
    rec = torch.empty(F, 13, dtype=torch.uint8, device=fl.device)
    rec[:, 0] = 3
    rec[:, 1:] = fl.view(torch.uint8).view(F, 12)
    return rec.reshape(-1)


def ply_bytes(verts, faces, bbox, offset=None, scale=None):
    """utils.py:189-222 after marching_cubes: faces[..., ::-1], bbox[0] + verts, then / scale and - offset with the
    reference's dtypes, packed into the PLY file plyfile writes for the reference's structured arrays.  The records
    are built on the device (or wherever verts lives) and copied to the host once."""
    pts = ply_positions(verts, bbox, offset=offset, scale=scale)
    body = torch.cat([pts.view(torch.uint8).reshape(-1), face_records(faces)]).cpu().numpy()
    return PLY_HEADER.format(V=pts.shape[0], F=faces.shape[0]).encode("ascii") + body.tobytes()


def convert_sdf_samples_to_ply(pytorch_3d_sdf_tensor, ply_filename_out, bbox, level=0.5, offset=None, scale=None):
    """utils.py:165-225: marching cubes at ``level`` with spacing (bbox[1]-bbox[0]) / shape, reversed faces, the mesh
    moved to bbox[0] (then / scale, - offset) and written to ``ply_filename_out`` as binary little-endian PLY.  The
    reversed faces point out of the dense region."""
    voxel_size = ply_spacing(tuple(pytorch_3d_sdf_tensor.shape), bbox)
    verts, faces = marching_cubes(pytorch_3d_sdf_tensor, level=level, spacing=[float(v) for v in voxel_size])
    data = ply_bytes(verts, faces, bbox, offset=offset, scale=scale)
    print("saving mesh to %s" % (ply_filename_out))
    with open(ply_filename_out, "wb") as f:
        f.write(data)


def read_ply(path):
    """(verts [V,3] float32, faces [F,3] int32) of a file written by convert_sdf_samples_to_ply."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    V = int(next(s for s in head if s.startswith("element vertex")).split()[-1])
    F = int(next(s for s in head if s.startswith("element face")).split()[-1])
    verts = np.frombuffer(data, dtype="<f4", count=3 * V, offset=end).reshape(V, 3)
    rec = np.frombuffer(data, dtype=FACE, count=F, offset=end + 12 * V)
    if F and not (rec["n"] == 3).all():
        raise ValueError(f"{path}: a face is not a triangle")
    if end + 12 * V + 13 * F != len(data):
        raise ValueError(f"{path}: {len(data) - end} body bytes for {V} vertices and {F} faces")
    return verts.copy(), rec["v"].astype(np.int32)


def read_asset_ply(path):
    """The arrays of a file written by export_asset: {xyz [V,3] float32, normal [V,3] float32, rgb [V,3] uint8,
    roughness [V] float32, albedo [V,3] float32, probed [V] uint8, faces [F,3] int32}.  Raises ValueError unless the
    header is export_asset's layout and the body holds exactly V vertex and F face records."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    V = int(next(s for s in head if s.startswith("element vertex")).split()[-1])
    F = int(next(s for s in head if s.startswith("element face")).split()[-1])
    if data[:end] != ASSET_PLY_HEADER.format(V=V, F=F).encode("ascii"):
        raise ValueError(f"{path}: not the vertex / face layout of export_asset")
    if end + ASSET_VERTEX.itemsize * V + FACE.itemsize * F != len(data):
        raise ValueError(f"{path}: {len(data) - end} body bytes for {V} vertices and {F} faces")
    vert = np.frombuffer(data, dtype=ASSET_VERTEX, count=V, offset=end)
    rec = np.frombuffer(data, dtype=FACE, count=F, offset=end + ASSET_VERTEX.itemsize * V)
    if F and not (rec["n"] == 3).all():
        raise ValueError(f"{path}: a face is not a triangle")
    out = {k: vert[k].copy() for k in ASSET_VERTEX.names}
    out["faces"] = rec["v"].astype(np.int32)
    return out


@torch.no_grad()
def export_mesh(tensoIR, ply_path, level=0.005):
    """export_mesh of scripts/export_mesh.py / train_tensoIR.py:53-62: the dense alpha at the model's gridSize, then
    convert_sdf_samples_to_ply with bbox = tensoIR.aabb."""
    alpha, _ = tensoIR.getDenseAlpha()
    convert_sdf_samples_to_ply(alpha, ply_path, bbox=tensoIR.aabb, level=level)


# ---- relightable asset --------------------------------------------------------------------------------------------

def field_positions(idx, bbox, shape):
    """Where marching-cubes index coordinates ``idx`` [V,3] lie in the field: getDenseAlpha's own expression
    bbox[0] (1 - s) + bbox[1] s with s = idx / (N - 1), since it samples axis i at linspace(0, 1, N_i).  The PLY puts the
    same vertex at bbox[0] + idx (bbox[1] - bbox[0]) / N (ply_spacing), up to one voxel toward bbox[0]."""
    b = torch.as_tensor(bbox).detach().to(device=idx.device, dtype=torch.float32)
    s = idx / torch.tensor([n - 1 for n in shape], dtype=torch.float32, device=idx.device)
    return b[0] * (1 - s) + b[1] * s


def asset_surface(tensoIR, level=0.005):
    """export_mesh's surface of the model -> (x y z [V,3] as the PLY carries them, faces [F,3] in marching_cubes'
    winding, the vertices where the surface lies in the field [V,3]), on the device.  The two marching-cubes calls
    differ only in their spacing, so they emit the same vertices in the same order."""
    alpha, _ = tensoIR.getDenseAlpha()
    shape = tuple(alpha.shape)
    verts, faces = marching_cubes(alpha, level, [float(s) for s in ply_spacing(shape, tensoIR.aabb)])
    idx, _ = marching_cubes(alpha, level, (1., 1., 1.))
    assert idx.shape == verts.shape
    return ply_positions(verts, tensoIR.aabb), faces, field_positions(idx, tensoIR.aabb, shape)


def vertex_normals(tensoIR, v):
    """The model's derived normal at field positions ``v`` [V,3] (compute_derived_normals, tensorBase:839-856, on the
    tir_vm_density_grad kernel): the normalised density gradient w.r.t. the normalised coordinates, negated, so it
    points out of the dense region.  Unit length where |gradient| >= 1e-6 (the normalisation's eps), shorter below."""
    from .primary import _derived_normals
    if v.shape[0] == 0:
        return torch.zeros_like(v)
    return _derived_normals(tensoIR, tensoIR.normalize_coord(v))


def probe_offset(tensoIR):
    """r: the distance outside its vertex at which a probe ray's samples start, PROBE_OFFSET_VOXELS of the largest
    voxel edge of the model's grid.  Marching cubes places a vertex by linear interpolation on a grid edge whose ends
    straddle the level, so the field's own level set can lie up to a voxel away along the normal; two voxels put the
    first sample outside it, while geometry more than two voxels out along the normal is not in front of the vertex."""
    return PROBE_OFFSET_VOXELS * float(tensoIR.units.max())


def has_normal(n):
    """Whether derived normals n [V,3] give a direction: |n| is 1 where the density gradient is at least the
    normalisation's eps (1e-6) and falls from there to 0 with the gradient, so |n| < 0.5 means no direction."""
    return n.norm(dim=-1) >= 0.5


def probe_rays(v, n, near, r):
    """One primary ray per vertex, [V,6]: d = -n, o = v + (near + r) n.  The sampler starts at max(box entry, near),
    so the samples start at v + r n, or at the box entry if that comes later."""
    return torch.cat([v + (near + r) * n, -n], dim=-1)


@torch.no_grad()
def probe(tensoIR, v, n, chunk=PROBE_CHUNK):
    """Render the probe rays of field positions ``v`` with derived normals ``n`` through the model's forward (eval mode,
    light 0, white background: relight()'s call) in chunks.  Only vertices whose n gives a direction (``has_normal``)
    are rendered; a vertex is probed when it is rendered and its ray's acc is at least PROBE_ACC_THRESHOLD.  An unprobed
    vertex gets albedo 0, roughness 1 and normal n ((0,0,1) when n gives no direction).
    -> dict of rays [V,6], acc [V] (0 where not rendered), albedo [V,3], roughness [V], normal [V,3], probed [V] bool."""
    V, dev = v.shape[0], v.device
    rays = probe_rays(v, n, float(tensoIR.near_far[0]), probe_offset(tensoIR))
    has_n = has_normal(n)
    sel = torch.nonzero(has_n).reshape(-1)
    # the forward's acc, albedo, roughness and normal of the rendered rays; rows without a normal stay 0
    maps = [torch.zeros(V, k, device=dev) for k in (1, 3, 1, 3)]
    if sel.numel():
        sub = rays.index_select(0, sel)
        li = torch.zeros((min(chunk, sub.shape[0]), 1), dtype=torch.int32, device=dev)
        for s in range(0, sub.shape[0], chunk):
            e = min(s + chunk, sub.shape[0])
            _, _, nrm, alb, rgh, _, a, *_ = tensoIR(sub[s:e], li[:e - s], is_train=False, white_bg=True, ndc_ray=False,
                                                    N_samples=-1)
            for dst, t in zip(maps, (a, alb, rgh, nrm)):
                dst[sel[s:e]] = t.detach().reshape(e - s, -1)
    acc, albedo, rough, normal = maps
    acc, rough = acc[:, 0], rough[:, 0]
    probed = has_n & (acc >= PROBE_ACC_THRESHOLD)
    fallback_n = torch.where(has_n[:, None], n, torch.tensor([0., 0., 1.], device=dev))
    return dict(rays=rays, acc=acc, albedo=torch.where(probed[:, None], albedo, 0.),
                roughness=torch.where(probed, rough, 1.), normal=torch.where(probed[:, None], normal, fallback_n),
                probed=probed)


def vertex_colors(albedo):
    """uint8 vertex colours of linear albedo [V,3]: the evaluation's albedo_gamma_corrected.png expression."""
    return (albedo ** (1 / 2.2) * 255).to(torch.uint8)


def asset_ply_bytes(pts, faces, normal, albedo, roughness, probed):
    """The PLY file of export_asset: ASSET_PLY_HEADER, one 44-byte ASSET_VERTEX record per vertex (x y z, predicted
    normal, gamma-corrected uint8 colour, roughness, linear albedo, probed) and ply_bytes' face records.  The records are
    built where pts lives and copied to the host once."""
    V = pts.shape[0]

    def f32(t, k):
        return t.detach().to(torch.float32).reshape(V, k).contiguous().view(torch.uint8)
    rec = torch.empty(V, ASSET_VERTEX.itemsize, dtype=torch.uint8, device=pts.device)
    rec[:, 0:12] = f32(pts, 3)
    rec[:, 12:24] = f32(normal, 3)
    rec[:, 24:27] = vertex_colors(albedo.reshape(V, 3))
    rec[:, 27:31] = f32(roughness, 1)
    rec[:, 31:43] = f32(albedo, 3)
    rec[:, 43] = probed.reshape(V).to(torch.uint8)
    body = torch.cat([rec.reshape(-1), face_records(faces)]).cpu().numpy()
    return ASSET_PLY_HEADER.format(V=V, F=faces.shape[0]).encode("ascii") + body.tobytes()


def envmap_paths(ply_path, n_lights):
    """``{ply stem}_envmap_{k}.hdr`` for every light index k."""
    stem = os.path.splitext(ply_path)[0]
    return [f"{stem}_envmap_{k}.hdr" for k in range(n_lights)]


@torch.no_grad()
def light_envmaps(tensoIR):
    """The radiance of every light of the model on the evaluation's 256x512 generate_envir_map_dir grid, clipped at 0
    as the evaluation's environment map is, not tone-mapped -> float32 [light_num, 256, 512, 3] on the device."""
    H, W = ENVMAP_HW
    dev = tensoIR.aabb.device
    _, dirs = tensoIR.generate_envir_map_dir(H, W)
    rgbs = tensoIR.get_light_rgbs(dirs.reshape(-1, 3).to(dev), device=dev)
    return rgbs.detach().float().clamp(min=0).reshape(tensoIR.light_num, H, W, 3)


def _check_asset_edits(edits):
    if any(e.fresnel_set is not None or e.fresnel_mul is not None for e in edits):
        raise ValueError("the asset has no fresnel column: fresnel edits cannot be exported")


def edit_vertices(p, v, edits):
    """The probe outputs ``p`` (``probe``) at field positions ``v`` with the material rules ``edits`` (a list of
    tensoir_b200.editing.MaterialEdit) applied by tir_material_edit: scale 1, only probed vertices edited.
    -> (albedo [V,3], roughness [V]).  Raises ValueError for a fresnel op: the asset has no fresnel column."""
    from .editing import edit_materials
    _check_asset_edits(edits)
    V = v.shape[0]
    maps = (None, None, p["albedo"], p["roughness"].reshape(V, 1), torch.zeros(V, 3, device=v.device),
            p["probed"].float())
    albedo, rough, _, _ = edit_materials(maps, edits, 1.0, 0.5, points=v)
    return albedo, rough[:, 0]


@torch.no_grad()
def export_asset(tensoIR, ply_path, level=0.005, envmaps=True, edits=None):
    """A relightable asset of the model: ``ply_path`` holds export_mesh's geometry (byte-identical x y z and faces) with
    the probed albedo, roughness and predicted normal per vertex (``probe``), and, with ``envmaps``,
    ``{ply stem}_envmap_{k}.hdr`` the radiance of light k.  Pass envmaps=False when the model's lights were not
    learned, as for a general multi-light model loaded from a checkpoint (its lgtSGs_list is not in the state_dict).
    With ``edits`` (a list of tensoir_b200.editing.MaterialEdit without fresnel ops) the albedo, colour and roughness
    columns hold the edited materials of the probed vertices (``edit_vertices``).  Nothing on the model changes.
    Returns the number of unprobed vertices."""
    from .relight import write_hdr
    if edits is not None:
        _check_asset_edits(edits)
    pts, faces, v = asset_surface(tensoIR, level)
    p = probe(tensoIR, v, vertex_normals(tensoIR, v))
    albedo, rough = (p["albedo"], p["roughness"]) if edits is None else edit_vertices(p, v, edits)
    data = asset_ply_bytes(pts, faces, p["normal"], albedo, rough, p["probed"])
    unprobed = int(pts.shape[0] - int(p["probed"].sum()))
    print(f"saving asset to {ply_path}: {pts.shape[0]} vertices, {faces.shape[0]} faces, {unprobed} unprobed")
    with open(ply_path, "wb") as f:
        f.write(data)
    if not envmaps:
        return unprobed
    for path, rgb in zip(envmap_paths(ply_path, tensoIR.light_num), light_envmaps(tensoIR).cpu().numpy()):
        write_hdr(path, rgb)
    return unprobed
