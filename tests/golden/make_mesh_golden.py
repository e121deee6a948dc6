"""Generate tests/golden/mesh_reference.pt by running the REAL reference (imported from a checkout of TensoIR) on the
CPU.  The reference import and the model builders are make_golden.py's and make_shrunk_golden.py's.

    python tests/golden/make_mesh_golden.py <path to the TensoIR checkout>

For the rotated G=24 fixture model and the shrunk states A and B (30x31x29 grid, asymmetric box) it records
  * getDenseAlpha(): the raw dense alpha volume at the model's gridSize (no clamp, no pooling) and the model's aabb;
  * the reference's own utils.convert_sdf_samples_to_ply run on that volume with level 0.005, under capturing
    stand-ins for skimage.measure.marching_cubes and plyfile: the stand-in marching_cubes returns a fixed, hand-made
    (verts, faces) and records the spacing and level the reference passes; the plyfile stand-in records the `vertex`
    and `face` structured arrays the reference describes and the path it writes.
skimage and plyfile are not needed: the fixture pins the reference's post-processing (spacing, face flip, vertex
records) around marching cubes.  tests/test_mesh_cpu.py replays it, tests/test_mesh_gpu.py checks getDenseAlpha.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, build_rotated, import_reference  # noqa: E402
from make_shrunk_golden import SHRINK_BOX, UPSAMPLE  # noqa: E402

LEVEL = 0.005
# the stand-in's mesh: float32 vertices with fractional coordinates, int32 faces in no particular order
STANDIN_VERTS = (np.arange(21, dtype=np.float32).reshape(7, 3) * np.float32(0.37) - np.float32(1.1)) ** 2 / 3
STANDIN_FACES = np.array([[0, 1, 2], [2, 1, 3], [4, 3, 5], [6, 5, 0], [1, 6, 4]], dtype=np.int32)


def install_standins():
    """Capturing skimage.measure.marching_cubes and plyfile.PlyElement / PlyData; returns the capture dict."""
    cap = {}
    measure = types.ModuleType("skimage.measure")

    def marching_cubes(volume, level=None, spacing=(1.0, 1.0, 1.0), **kw):
        cap["mc_shape"] = tuple(volume.shape)
        cap["mc_level"] = level
        cap["mc_spacing"] = [float(s) for s in spacing]
        cap["mc_spacing_types"] = [type(s).__name__ for s in spacing]
        cap["mc_kwargs"] = sorted(kw)
        return STANDIN_VERTS.copy(), STANDIN_FACES.copy(), np.zeros_like(STANDIN_VERTS), np.zeros(7, np.float32)

    measure.marching_cubes = marching_cubes
    skimage = types.ModuleType("skimage")
    skimage.measure = measure
    sys.modules["skimage"], sys.modules["skimage.measure"] = skimage, measure
    plyfile = types.ModuleType("plyfile")

    class PlyElement:
        @staticmethod
        def describe(arr, name):
            cap[f"element_{name}"] = arr.copy()
            return name

    class PlyData:
        def __init__(self, elements):
            cap["elements"] = list(elements)

        def write(self, path):
            cap["written"] = path

    plyfile.PlyElement, plyfile.PlyData = PlyElement, PlyData
    sys.modules["plyfile"] = plyfile
    return cap


def record(utils, cap, m):
    alpha, _ = m.getDenseAlpha()
    cap.clear()
    utils.convert_sdf_samples_to_ply(alpha.cpu(), "mesh.ply", bbox=m.aabb.cpu(), level=LEVEL)
    v, f = cap["element_vertex"], cap["element_face"]
    return dict(volume=alpha.detach().clone(), aabb=m.aabb.clone(), grid_size=m.gridSize.tolist(),
                mc_shape=cap["mc_shape"], mc_level=cap["mc_level"], mc_spacing=cap["mc_spacing"],
                mc_spacing_types=cap["mc_spacing_types"], elements=cap["elements"], written=cap["written"],
                vertex_dtype=str(v.dtype), face_dtype=str(f.dtype),
                vertex_records=torch.from_numpy(np.stack([v["x"], v["y"], v["z"]], -1).copy()),
                face_records=torch.from_numpy(np.ascontiguousarray(f["vertex_indices"])))


def main():
    cap = install_standins()
    _, rot, _, _ = import_reference()
    import utils
    out = dict(level=LEVEL, standin_verts=torch.from_numpy(STANDIN_VERTS.copy()),
               standin_faces=torch.from_numpy(STANDIN_FACES.copy()), models={})
    m = build_rotated(rot)
    m.updateAlphaMask((24, 24, 24))
    out["models"]["rotated"] = record(utils, cap, m)
    m.shrink(torch.tensor(SHRINK_BOX))
    m.upsample_volume_grid(UPSAMPLE)
    out["models"]["A"] = record(utils, cap, m)
    m.updateAlphaMask(tuple(m.gridSize.tolist()))
    out["models"]["B"] = record(utils, cap, m)
    path = os.path.join(HERE, "mesh_reference.pt")
    torch.save(out, path)
    size = os.path.getsize(path)
    print("mesh_reference.pt", size // 1024, "KiB")
    assert size < 1 << 20


if __name__ == "__main__":
    if REF is None or not os.path.isdir(REF):
        raise SystemExit(__doc__)
    main()
