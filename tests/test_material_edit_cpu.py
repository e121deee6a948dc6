"""Material editing on the CPU.

tir_material_edit is built for the host (tests/host_edit.cpp: the same C ABI, argument checks and per-point math of
csrc/tir_edit_body.h, a loop instead of a kernel) and driven through the real ctypes wrapper tensoir_b200.editing; it
must agree bit for bit with the numpy restatement of the rules below.  relight_edited runs on the host relighting build
(tests/host_relight.cpp) with the oracle's density march, as in test_relighting_cpu.py."""
import ctypes as C
import json
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from helpers import build_host_lib, oracle_field, use_host
from oracle import tensoir_oracle as O
from tensoir_b200 import _lib, editing, relighting
from tensoir_b200.editing import MaterialEdit

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
f32 = np.float32


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_edit"), "host_edit.cpp", "host_relight.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


def np_edit(rules, pts, albedo, rough, fresnel, acc, thr, scale):
    """The semantics of tir_material_edit (include/tensoir_b200.h), restated on float32 numpy arrays."""
    a0 = albedo * np.asarray(scale, f32).reshape(-1)
    a, r, f = a0.copy(), rough.copy(), fresnel.copy()
    sel = np.zeros(len(acc), np.int32)
    hit = acc > f32(thr)
    for k, e in enumerate(rules):
        m = hit.copy()
        if e.aabb is not None:
            lo, hi = np.asarray(e.aabb, f32)
            m &= ((lo <= pts) & (pts <= hi)).all(1)
        if e.key is not None:
            m &= (np.abs(a0 - np.asarray(e.key, f32)) <= f32(e.key_tol)).all(1)
        sel[m] |= 1 << k

        def op(x, v_set, v_mul, lo, hi):
            if v_set is not None:
                y = np.broadcast_to(np.asarray(v_set, f32), x.shape)
            elif v_mul is not None:
                y = x * np.asarray(v_mul, f32)
            else:
                return x
            return np.where(m[:, None], np.clip(y, f32(lo), f32(hi)), x)
        a = op(a, e.albedo_set, e.albedo_mul, 0, 1)
        r = op(r, e.roughness_set, e.roughness_mul, 0.09, 0.99)
        f = op(f, e.fresnel_set, e.fresnel_mul, 0, 1)
    return a, r, f, sel


def random_rules(g, count):
    rules = []
    for k in range(count):
        kw = {}
        if k % 3 != 2:
            c = g.uniform(-1, 1, 3)
            h = g.uniform(0.2, 1.0, 3)
            kw["aabb"] = [list(c - h), list(c + h)]
        if k % 4 == 1:
            kw["key"], kw["key_tol"] = list(g.uniform(0, 1, 3)), float(g.uniform(0.2, 0.6))
        for q, n in (("albedo", 3), ("roughness", 1), ("fresnel", 3)):
            op = ("set", "mul", None)[(k + len(q)) % 3]
            if op is not None:
                v = g.uniform(0, 1.5, n) if op == "set" else g.uniform(0.3, 2.5, n)
                kw[f"{q}_{op}"] = float(v[0]) if n == 1 else list(v)
        rules.append(MaterialEdit(**kw))
    return rules


def _run(rules, pts, albedo, rough, fresnel, acc, thr, scale, rays=None, depth=None):
    t = torch.from_numpy
    maps = (None if depth is None else t(depth), None, t(albedo), t(rough), t(fresnel), t(acc))
    out = editing.edit_materials(maps, rules, t(np.asarray(scale, f32)), thr,
                                 points=None if pts is None else t(pts), rays=None if rays is None else t(rays))
    return [o.numpy() for o in out]


def _assert_same(got, want):
    for g_, w_ in zip(got, want):
        assert g_.dtype == w_.dtype and np.array_equal(g_, w_, equal_nan=True)


@pytest.mark.parametrize("stride", [1, 3])
def test_sixteen_overlapping_rules(host_lib, stride):
    g = np.random.default_rng(stride)
    n = 20000
    pts = g.uniform(-1.5, 1.5, (n, 3)).astype(f32)
    albedo = g.uniform(0, 1.2, (n, 3)).astype(f32)
    rough = g.uniform(0.09, 0.99, (n, stride)).astype(f32)
    fresnel = g.uniform(0, 1, (n, 3)).astype(f32)
    acc = g.uniform(0, 1, n).astype(f32)
    rules = random_rules(g, _lib.EDIT_MAX_RULES)
    scale = [0.8, 1.1, 0.95]
    got = _run(rules, pts, albedo, rough, fresnel, acc, 0.5, scale)
    want = np_edit(rules, pts, albedo, rough, fresnel, acc, 0.5, scale)
    _assert_same(got, want)
    sel = got[3]
    assert (sel != 0).mean() > 0.3 and (np.bitwise_count(sel.astype(np.uint32)) > 1).any()  # rules do overlap
    miss = acc <= 0.5                           # non-hit rows: albedo*scale, the rest unchanged, no selection
    assert np.array_equal(got[0][miss], albedo[miss] * np.asarray(scale, f32))
    assert np.array_equal(got[1][miss], rough[miss]) and np.array_equal(got[2][miss], fresnel[miss])
    assert not sel[miss].any()


def test_points_from_rays_are_the_sampler_points(host_lib):
    g = np.random.default_rng(3)
    n = 5000
    rays = np.concatenate([g.uniform(-3, 3, (n, 3)), g.normal(size=(n, 3))], 1).astype(f32)
    depth = g.uniform(0, 5, n).astype(f32)
    pts = rays[:, :3] + depth[:, None] * rays[:, 3:]              # rl_surface: one fp32 multiply, one add
    albedo, fresnel = g.uniform(0, 1, (n, 3)).astype(f32), g.uniform(0, 1, (n, 3)).astype(f32)
    rough, acc = g.uniform(0.1, 0.9, (n, 1)).astype(f32), np.ones(n, f32)
    rules = [MaterialEdit(aabb=[[-1, -1, -1], [1, 2, 1]], albedo_set=0.3), MaterialEdit(aabb=[[0, 0, 0], [3, 3, 3]],
                                                                                       roughness_mul=2.0)]
    got = _run(rules, None, albedo, rough, fresnel, acc, 0.5, [1, 1, 1], rays=rays, depth=depth)
    _assert_same(got, np_edit(rules, pts, albedo, rough, fresnel, acc, 0.5, [1, 1, 1]))
    assert got[3].any()


def test_box_faces_key_tolerance_and_clamps(host_lib):
    lo, hi = f32(-0.25), f32(0.5)
    up, down = np.nextafter(hi, f32(1)), np.nextafter(lo, f32(-1))
    pts = np.array([[lo, lo, lo], [hi, hi, hi], [lo, hi, 0], [up, 0, 0], [0, down, 0], [0, 0, up], [0, 0, 0]], f32)
    n = len(pts)
    acc = np.ones(n, f32)
    albedo = np.full((n, 3), 0.5, f32)
    albedo[3] = [0.75, 0.5, 0.5]                                 # |0.75 - 0.5| = 0.25: exactly at the tolerance
    albedo[4] = [0.5, np.nextafter(f32(0.75), f32(1)), 0.5]       # one ulp past it
    rough, fresnel = np.full((n, 1), 0.5, f32), np.full((n, 3), 0.5, f32)
    box = MaterialEdit(aabb=[[float(lo)] * 3, [float(hi)] * 3], albedo_set=[2.0, -1.0, 0.5])        # clamps to 1, 0
    key = MaterialEdit(key=[0.5, 0.5, 0.5], key_tol=0.25, roughness_set=0.01, fresnel_mul=[3.0, -1.0, 1.0])
    big = MaterialEdit(roughness_mul=100.0, fresnel_set=[-5, 5, 0.25])
    got = _run([box, key, big], pts, albedo, rough, fresnel, acc, 0.5, [1, 1, 1])
    _assert_same(got, np_edit([box, key, big], pts, albedo, rough, fresnel, acc, 0.5, [1, 1, 1]))
    a, r, f, sel = got
    assert list(sel & 1) == [1, 1, 1, 0, 0, 0, 1]                # faces are inside, one ulp beyond is not
    assert list((sel >> 1) & 1) == [1, 1, 1, 1, 0, 1, 1]
    assert np.array_equal(a[0], np.array([1, 0, 0.5], f32))
    assert np.all(r == f32(0.99))                                 # 0.01 -> 0.09, then * 100 -> 0.99 (or 50 -> 0.99)
    assert np.array_equal(f[0], np.array([0, 1, 0.25], f32))
    none_selected = _run([box], pts, albedo, rough, fresnel, np.zeros(n, f32), 0.5, [1, 1, 1])
    assert not none_selected[3].any() and np.array_equal(none_selected[0], albedo)


def test_empty_and_no_rules(host_lib):
    z3, z1 = np.zeros((0, 3), f32), np.zeros((0, 1), f32)
    got = _run([MaterialEdit(albedo_set=0.5)], z3, z3, z1, z3, np.zeros(0, f32), 0.5, [1, 1, 1])
    assert [o.shape for o in got] == [(0, 3), (0, 1), (0, 3), (0,)]
    g = np.random.default_rng(5)
    pts, alb, fr = (g.uniform(0, 1, (9, 3)).astype(f32) for _ in range(3))
    rough = g.uniform(0, 1, (9, 3)).astype(f32)
    a, r, f, sel = _run([], pts, alb, rough, fr, np.ones(9, f32), 0.5, [0.5, 2, 1])
    assert np.array_equal(a, alb * np.array([0.5, 2, 1], f32)) and np.array_equal(r, rough)
    assert np.array_equal(f, fr) and not sel.any()


def test_edit_arguments(host_so):
    lib = host_so
    rules = (_lib.TirEditRule * 17)()
    buf = (C.c_float * 64)()
    sel = (C.c_int32 * 4)()
    call = lambda rl, k, pts, stride, n=4, alb=buf: lib.tir_material_edit(  # noqa: E731
        rl, k, None, None, pts, alb, buf, stride, buf, buf, n, 0.5, buf, buf, buf, buf, sel, None)
    assert call(rules, 17, buf, 1) == -2                  # more than TIR_EDIT_MAX_RULES
    assert call(rules, 1, buf, 2) == -2                   # stride other than 1 or 3
    assert call(rules, 1, buf, 1, n=-1) == -2
    assert call(None, 1, buf, 1) == -1
    assert call(rules, 1, None, 1) == -1                  # neither points nor rays and depth
    assert call(rules, 1, buf, 1, alb=None) == -1
    assert call(None, 0, None, 1, n=0, alb=None) == 0     # nothing to do
    assert call(rules, 1, buf, 3) == 0
    for field, bad in (("albedo_op", 3), ("rough_op", -1), ("fresnel_op", 7), ("flags", 4)):
        rules[0] = _lib.TirEditRule()
        setattr(rules[0], field, bad)
        assert call(rules, 1, buf, 1) == -3, field
        assert call(rules, 1, buf, 1, n=0) == -3, field   # checked before the empty early-out


def test_edit_rule_struct_layout(tmp_path):
    src = tmp_path / "sz.c"
    names = ["flags", "albedo_op", "rough_op", "fresnel_op", "box_lo", "box_hi", "key", "key_tol", "albedo", "rough",
             "fresnel"]
    offs = ",".join(f"offsetof(TirEditRule,{k})" for k in names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tensoir_b200.h"\n'
                   f'int main(void){{printf("%zu{" %zu" * len(names)} %d %d %d %d %d %d %d\\n",sizeof(TirEditRule),'
                   f'{offs},TIR_EDIT_MAX_RULES,TIR_EDIT_NONE,TIR_EDIT_SET,TIR_EDIT_MUL,TIR_EDIT_BOX,TIR_EDIT_KEY,'
                   '(int)(TIR_EDIT_ROUGH_MIN*100+0.5)*100+(int)(TIR_EDIT_ROUGH_MAX*100+0.5));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    T = _lib.TirEditRule
    assert got == ([C.sizeof(T)] + [getattr(T, k).offset for k in names]
                   + [_lib.EDIT_MAX_RULES, _lib.EDIT_NONE, _lib.EDIT_SET, _lib.EDIT_MUL, _lib.EDIT_BOX, _lib.EDIT_KEY,
                      999])


def test_rule_table_encoding():
    t = editing.rule_table([MaterialEdit(aabb=[[0, 1, 2], [3, 4, 5]], albedo_mul=0.5, roughness_set=0.3),
                            MaterialEdit(key=[0.1, 0.2, 0.3], key_tol=0.1, fresnel_set=[0.1, 0.2, 0.3])])
    assert t[0].flags == _lib.EDIT_BOX and list(t[0].box_hi) == [3, 4, 5] and list(t[0].albedo) == [0.5] * 3
    assert (t[0].albedo_op, t[0].rough_op, t[0].fresnel_op) == (_lib.EDIT_MUL, _lib.EDIT_SET, _lib.EDIT_NONE)
    assert t[1].flags == _lib.EDIT_KEY and t[1].fresnel_op == _lib.EDIT_SET
    assert t[1].key_tol == pytest.approx(0.1) and t[1].albedo_op == _lib.EDIT_NONE


@pytest.mark.parametrize("bad", [
    {"v": [{"albedo_sett": 0.5}]},                                   # unknown key
    {"v": [{"albedo_set": 0.5, "albedo_mul": 0.5}]},                 # set and mul on one quantity
    {"v": [{"roughness_set": 0.5, "roughness_mul": 0.5}]},
    {"v": [{"aabb": [[0, 0, 0], [1, 1]]}]},                          # wrong shapes
    {"v": [{"aabb": [[0, 0, 1], [1, 1, 0]]}]},
    {"v": [{"key": [0.5, 0.5]}]},
    {"v": [{"albedo_set": [0.5, 0.5]}]},
    {"v": [{"roughness_set": [0.5]}]},
    {"v": [{"key_tol": -0.1, "key": [0, 0, 0]}]},
    {"v": [{"fresnel_mul": "x"}]},
    {"v": [{"albedo_set": float("nan")}]},
    {"v": [{"albedo_set": 0.5}] * 17},                               # more than 16 rules
    {"v": []},                                                       # empty variant
    {"v": ["albedo_set"]},
    {"../x": [{"albedo_set": 0.5}]},                                 # not a safe directory name
    {"a/b": [{"albedo_set": 0.5}]},
    {"": [{"albedo_set": 0.5}]},
    {"..": [{"albedo_set": 0.5}]},
    {"original": [{"albedo_set": 0.5}]},                             # reserved
    [{"albedo_set": 0.5}],
])
def test_load_edits_rejects(bad):
    with pytest.raises(ValueError):
        editing.load_edits(bad)


def test_load_edits_file(tmp_path):
    spec = {"red": [{"aabb": [[-1, -1, -1], [1, 1, 0]], "albedo_set": [0.8, 0.1, 0.1], "roughness_set": 0.2}],
            "shiny_2": [{"roughness_mul": 0.5, "fresnel_set": 0.5}, {"key": [1, 1, 1], "key_tol": 0.1,
                                                                      "albedo_mul": 0.9}]}
    p = tmp_path / "edits.json"
    p.write_text(json.dumps(spec))
    got = editing.load_edits(str(p))
    assert list(got) == ["red", "shiny_2"] and len(got["shiny_2"]) == 2
    assert got["red"][0].aabb == ((-1.0, -1.0, -1.0), (1.0, 1.0, 0.0)) and got["red"][0].roughness_set == 0.2
    assert got["shiny_2"][0].fresnel_set == (0.5, 0.5, 0.5) and got["shiny_2"][1].albedo_mul == (0.9,) * 3
    assert editing.load_edits(got) == got


# ---- relight_edited on the host relighting build ------------------------------------------------------------------

class StubModel:
    """A model whose primary render is a fixed function of the ray, with the oracle field for the march."""

    def __init__(self, field):
        self.field, self.device = field, torch.device("cpu")

    def __call__(self, rays, light_idx, **kw):
        n = rays.shape[0]
        o, d = rays[:, :3], rays[:, 3:]
        ph = (o * 1.7 + d * 3.1).sum(-1)
        depth = 3.6 + 0.2 * torch.sin(ph)
        normal = -d + 0.3 * torch.stack([torch.sin(ph), torch.cos(ph), torch.sin(2 * ph)], -1)
        albedo = 0.5 + 0.4 * torch.stack([torch.sin(ph), torch.cos(3 * ph), torch.sin(5 * ph)], -1)
        rough = (0.5 + 0.4 * torch.cos(7 * ph))[:, None]
        fresnel = torch.full((n, 3), 0.04)
        acc = (0.5 + 0.5 * torch.sin(11 * ph)).clamp(0, 1)
        rgb = albedo * 0.9
        return rgb, depth, normal, albedo, rough, fresnel, acc


def _host_relight_env(monkeypatch, fx, samples=24):
    field = oracle_field(fx)
    marches = []

    def oracle_march(f, rays_o, rays_d, *, table=None, counters=None, **kw):
        marches.append(rays_o.shape[0])
        nerv, nerfactor = O.compute_transmittance(field, rays_o, rays_d, 96, 0.05, 1.5)
        return nerv, 1 - nerfactor, None
    monkeypatch.setattr(relighting.ops, "march_density", oracle_march)
    monkeypatch.setattr(relighting, "NUM_SAMPLES", samples)
    ratio = (torch.tensor(1.2), torch.tensor([1.1, 0.9, 1.3]))
    monkeypatch.setattr(relighting, "compute_rescale_ratio", lambda *a, **k: ratio)
    import tensoir_b200.evaluation as E
    monkeypatch.setattr(E, "compute_rescale_ratio", lambda *a, **k: ratio)
    return StubModel(field), marches


def _seeded_uniforms(monkeypatch, seed):
    gen = torch.Generator().manual_seed(seed)
    monkeypatch.setattr(relighting, "_uniforms",
                        lambda L, n, S, device: torch.rand(L, n, S, dtype=torch.float64, generator=gen))


def test_relight_edited_original_is_relight(host_lib, golden_rotated, tmp_path, monkeypatch):
    """The 'original' variant's relit PNGs are relight()'s bytes under the same uniforms, the march runs once per
    chunk whatever the number of variants, and a region edit leaves the pixels it does not select unchanged."""
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    import cv2
    model, marches = _host_relight_env(monkeypatch, golden_rotated)
    rgb = golden_rotated["env_rgb"].numpy()
    names = ["sunny", "dim"]
    hdr = {"sunny": rgb, "dim": rgb[:, ::-1].copy() * 0.4}
    H, W, B = 12, 14, 70
    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=names)
    n_chunks = -(-H * W // B)

    _seeded_uniforms(monkeypatch, 1)
    ref = tmp_path / "ref"
    relighting.relight(ds, types.SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(ref), batch_size=B), tensoIR=model)
    assert len(marches) == len(ds) * n_chunks

    marches.clear()
    _seeded_uniforms(monkeypatch, 1)
    out = tmp_path / "edit"
    variants = {"red": [{"aabb": [[-9, -9, -9], [9, 0.0, 9]], "albedo_set": [0.9, 0.1, 0.1]}],
                "rough": [{"roughness_set": 0.95}, {"key": [0.5, 0.5, 0.5], "key_tol": 0.3, "fresnel_mul": 4.0}]}
    psnr = editing.relight_edited(ds, types.SimpleNamespace(hdrdir=hdr, geo_buffer_path=str(out), batch_size=B),
                                  variants, tensoIR=model)
    assert len(marches) == len(ds) * n_chunks                 # one march per chunk for three variants
    assert set(psnr) == {"original", "red", "rough"} and all(len(v) == len(ds) for v in psnr["red"].values())
    files = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs
                   if not f.endswith(".mp4"))
    want = [f"{v}/relight_psnr.txt" for v in psnr]
    for i in range(len(ds)):
        for v in psnr:
            want += [f"test_{i:03d}/{v}/{f}" for f in ("albedo_gamma_corrected.png", "roughness.png", "selection.png",
                                                      "relighting_without_bg/relight_psnr.txt")]
            want += [f"test_{i:03d}/{v}/relighting_{s}/{n}.png" for s in ("with_bg", "without_bg") for n in names]
    assert files == sorted(want)
    for i in range(len(ds)):
        for s in ("with_bg", "without_bg"):
            for n in names:
                a = open(ref / f"test_{i:03d}" / f"relighting_{s}" / f"{n}.png", "rb").read()
                b = open(out / f"test_{i:03d}" / "original" / f"relighting_{s}" / f"{n}.png", "rb").read()
                assert a == b, (i, s, n)
        assert open(ref / f"test_{i:03d}/relighting_without_bg/relight_psnr.txt").read() == \
            open(out / f"test_{i:03d}/original/relighting_without_bg/relight_psnr.txt").read()
        sel = cv2.imread(str(out / f"test_{i:03d}/red/selection.png"), cv2.IMREAD_UNCHANGED)
        assert sel.shape == (H, W) and set(np.unique(sel)) <= {0, 255}
        assert not cv2.imread(str(out / f"test_{i:03d}/original/selection.png"), cv2.IMREAD_UNCHANGED).any()
        for n in names:
            a = cv2.imread(str(out / f"test_{i:03d}/original/relighting_without_bg/{n}.png"))
            b = cv2.imread(str(out / f"test_{i:03d}/red/relighting_without_bg/{n}.png"))
            assert np.array_equal(a[sel == 0], b[sel == 0])
    assert open(ref / "relight_psnr.txt").read() == open(out / "original" / "relight_psnr.txt").read()
