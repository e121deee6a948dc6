"""Mesh export: the reference's `scripts/export_mesh.py` / `--export_mesh 1` path (utils.py:165-225) on the GPU.

``marching_cubes`` runs the tir_marching_cubes_* kernels (csrc/tir_mesh.cu; topology, vertex placement and winding in
csrc/tir_mc_body.h) on a dense volume; ``convert_sdf_samples_to_ply`` keeps the reference's signature and
post-processing and writes the file plyfile writes for the reference's structured arrays; ``export_mesh`` is the
reference's export_mesh on a model.  There is no CPU fallback: a CPU volume is moved to the current CUDA device.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

PLY_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex {V}\nproperty float x\nproperty float y\n"
              "property float z\nelement face {F}\nproperty list uchar int vertex_indices\nend_header\n")
INT32_MAX = 2 ** 31 - 1


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


def ply_bytes(verts, faces, bbox, offset=None, scale=None):
    """utils.py:189-222 after marching_cubes: faces[..., ::-1], bbox[0] + verts, then / scale and - offset with the
    reference's dtypes, packed into the PLY file plyfile writes for the reference's structured arrays.  The records
    are built on the device (or wherever verts lives) and copied to the host once."""
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
    pts = pts.to(torch.float32).contiguous()
    fl = faces.to(torch.int32).flip(-1).contiguous()          # faces[..., ::-1]: inverse face orientation
    V, F = pts.shape[0], fl.shape[0]
    rec = torch.empty(F, 13, dtype=torch.uint8, device=pts.device)
    rec[:, 0] = 3
    rec[:, 1:] = fl.view(torch.uint8).view(F, 12)
    body = torch.cat([pts.view(torch.uint8).reshape(-1), rec.reshape(-1)]).cpu().numpy()
    return PLY_HEADER.format(V=V, F=F).encode("ascii") + body.tobytes()


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
    rec = np.frombuffer(data, dtype=np.dtype([("n", "u1"), ("v", "<i4", (3,))]), count=F, offset=end + 12 * V)
    if F and not (rec["n"] == 3).all():
        raise ValueError(f"{path}: a face is not a triangle")
    if end + 12 * V + 13 * F != len(data):
        raise ValueError(f"{path}: {len(data) - end} body bytes for {V} vertices and {F} faces")
    return verts.copy(), rec["v"].astype(np.int32)


@torch.no_grad()
def export_mesh(tensoIR, ply_path, level=0.005):
    """export_mesh of scripts/export_mesh.py / train_tensoIR.py:53-62: the dense alpha at the model's gridSize, then
    convert_sdf_samples_to_ply with bbox = tensoIR.aabb."""
    alpha, _ = tensoIR.getDenseAlpha()
    convert_sdf_samples_to_ply(alpha, ply_path, bbox=tensoIR.aabb, level=level)
