"""Shared pieces of the mesh-export tests: tensoir_b200.mesh.extract on the host build of the tir_marching_cubes_* C ABI
(tests/host_mesh.cpp), mesh checks, and the random / analytic test volumes."""
import numpy as np
import torch

from helpers import on_host

LEVEL = 0.5


def host_marching_cubes(lib, vol, level, spacing=(1.0, 1.0, 1.0)):
    """tensoir_b200.mesh.extract through the real ctypes wrapper, on the host build."""
    from tensoir_b200 import mesh
    with on_host(lib):
        v, f = mesh.extract(torch.from_numpy(np.ascontiguousarray(vol, dtype=np.float32)), level, spacing)
    return v.numpy(), f.numpy()


def directed_edges(faces):
    return np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])


def boundary_edges(faces):
    """directed edges whose reverse is missing; raises if a directed edge appears twice"""
    e = directed_edges(faces)
    key = e[:, 0].astype(np.int64) * (1 << 32) + e[:, 1]
    assert len(np.unique(key)) == len(key), "a directed edge appears twice"
    rev = e[:, 1].astype(np.int64) * (1 << 32) + e[:, 0]
    return e[~np.isin(key, rev)]


def assert_closed(faces):
    assert len(boundary_edges(faces)) == 0, "open mesh"
    assert not ((faces[:, 0] == faces[:, 1]) | (faces[:, 1] == faces[:, 2]) | (faces[:, 0] == faces[:, 2])).any()


def euler(verts, faces):
    e = np.sort(directed_edges(faces), axis=1)
    return len(verts) - len(np.unique(e, axis=0)) + len(faces)


def signed_volume(verts, faces):
    v = verts.astype(np.float64)[faces]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6)


def random_volume(shape, seed, border=True, at_level=0.1):
    """uniform values in [0,1) with a share set to exactly LEVEL, and (border=True) a zero border"""
    g = np.random.default_rng(seed)
    v = g.random(shape).astype(np.float32)
    v[g.random(shape) < at_level] = np.float32(LEVEL)
    if border:
        v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = 0, 0, 0, 0, 0, 0
    return v


def sphere_volume(shape=(41, 37, 45), r=13.0, spacing=(1.0, 1.0, 1.0)):
    """1 - |x - c| / r on a non-cubic grid: the 0.5 level is a sphere of radius r/2 (in index units times spacing)"""
    idx = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) * s for n, s in zip(shape, spacing)], indexing="ij"),
                   -1)
    c = np.array([(n - 1) * s / 2 for n, s in zip(shape, spacing)])
    return (1 - np.linalg.norm(idx - c, axis=-1) / r).astype(np.float32)


def torus_volume(shape=(48, 44, 24), R=12.0, r=4.5):
    x, y, z = np.meshgrid(*[np.arange(n, dtype=np.float64) - (n - 1) / 2 for n in shape], indexing="ij")
    d = np.sqrt((np.sqrt(x ** 2 + y ** 2) - R) ** 2 + z ** 2)
    return (1 - d / (2 * r)).astype(np.float32)            # 0.5 level: tube radius r


def saddle_volume(shape=(26, 23, 29)):
    """a product of sines with a half-cell period mismatch: most cells hold saddles, both decider outcomes occur"""
    x, y, z = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    v = 0.5 + 0.5 * np.sin(1.9 * x + 0.3) * np.sin(2.3 * y + 0.7) * np.sin(1.7 * z + 1.1)
    v = v.astype(np.float32)
    v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = 0, 0, 0, 0, 0, 0
    return v


def shared_volumes():
    """(name, volume, spacing) of the random and analytic volumes the CPU and GPU tests share"""
    out = []
    for n, shape in enumerate([(6, 7, 5), (17, 9, 23), (31, 28, 19)]):
        out.append((f"random{shape}", random_volume(shape, 100 + n), (0.5, 1.25, 2.0)))
    out.append(("sphere", sphere_volume(), (1.0, 1.0, 1.0)))
    out.append(("torus", torus_volume(), (1.0, 1.0, 1.0)))
    out.append(("saddle", saddle_volume(), (0.3, 0.7, 1.1)))
    return out
