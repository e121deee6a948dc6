"""Shared test helpers: build oracle fields from golden fixtures, and run the ctypes wrappers on a host build of their
C entries (tests/host_*.cpp) with CPU tensors."""
import contextlib
import ctypes as C
import os
import subprocess

import torch

from oracle import tensoir_oracle as O
from tensoir_b200 import _lib, ops

HERE = os.path.dirname(os.path.abspath(__file__))


def oracle_field(fx, with_mask=True, requires_grad=False):
    kw = {}
    if fx["kind"] == "rotated":
        kw["light_rotation"] = fx["light_rotation"]
    if fx["kind"] == "general":
        kw["lgt_sgs_list"] = fx["lgt_sgs_list"]
    f = O.field_from_state_dict(fx["state_dict"], fx["aabb"], fx["grid_size"], kind=fx["kind"],
                                alpha_volume=fx["alpha_volume"] if with_mask else None,
                                alpha_aabb=fx["alpha_aabb"] if with_mask else None, **kw)
    if requires_grad:
        for p in f.parameters():
            p.requires_grad_(True)
    return f


def named_oracle_params(f):
    """reference state_dict key -> oracle tensor."""
    out = {}
    for i in range(3):
        out[f"density_plane.{i}"] = f.density_plane[i]
        out[f"density_line.{i}"] = f.density_line[i]
        out[f"app_plane.{i}"] = f.app_plane[i]
        out[f"app_line.{i}"] = f.app_line[i]
    out["basis_mat.weight"] = f.basis_w
    if f.light_line_w is not None:
        out["light_line.weight"] = f.light_line_w
    for name, m in (("renderModule", f.mlp_rgb), ("renderModule_brdf", f.mlp_brdf),
                    ("renderModule_normal", f.mlp_normal)):
        if m is None:
            continue
        for j, (w, b) in zip((0, 2, 4), ((m.w0, m.b0), (m.w1, m.b1), (m.w2, m.b2))):
            out[f"{name}.mlp.{j}.weight"] = w
            out[f"{name}.mlp.{j}.bias"] = b
    if f.lgt_sgs is not None and f.light_rotation is not None:
        out["lgtSGs"] = f.lgt_sgs[0]
    return out


def build_host_lib(tmpdir, *cpp_files):
    """Compile the host builds ``cpp_files`` (names under tests/) into one shared library in tmpdir and load it, with
    the restype and argtypes of _lib.EXPORTS bound for every tir_* entry it exports."""
    so = os.path.join(str(tmpdir), "lib" + "_".join(os.path.splitext(f)[0] for f in cpp_files) + ".so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so]
                   + [os.path.join(HERE, f) for f in cpp_files], check=True)
    lib = C.CDLL(so)
    for name, (res, args) in _lib.EXPORTS.items():
        if hasattr(lib, name):
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def host_dptr(t, dtype=torch.float32, allow_none=False):
    """_lib.dptr for a host build: exactly as strict about None, dtype and contiguity, but for a CPU tensor."""
    if t is None:
        if allow_none:
            return None
        raise _lib.TirError("required tensor is None")
    if t.device.type != "cpu":
        raise _lib.TirError("the host build needs CPU tensors")
    if dtype is not None and t.dtype != dtype:
        raise _lib.TirError(f"expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise _lib.TirError("tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


def use_host(monkeypatch, lib, march=None):
    """Point the ctypes wrappers at the host build ``lib``; ``march``, if given, replaces ops.march_density, the
    density march every relighting module calls."""
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    monkeypatch.setattr(_lib, "dptr", host_dptr)
    if march is not None:
        monkeypatch.setattr(ops, "march_density", march)


@contextlib.contextmanager
def on_host(lib):
    """use_host for the length of a with block."""
    import pytest
    with pytest.MonkeyPatch.context() as mp:
        use_host(mp, lib)
        yield
