"""Camera-path frames on the CPU.

tir_ground_sample and tir_path_composite are built for the host (tests/host_path.cpp: the same C ABI, argument checks
and per-slot / per-pixel math of csrc/tir_path_body.h, loops instead of kernels) and driven through the real ctypes
wrappers of tensoir_b200.camera_path.  They are compared with a float64 restatement of the definitions in
include/tensoir_b200.h.  The cameras and the command line of tools/render_path.py are checked here too."""
import ctypes as C
import importlib.util
import json
import math
import os
import types

import numpy as np
import pytest
import torch

from helpers import build_host_lib, use_host
from tensoir_b200 import _lib, ops
from tensoir_b200 import camera_path as P
from tensoir_b200 import relighting as R
from tensoir_b200.relight import Environment_Light

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
EPS = float(np.finfo(np.float32).eps)
BOX = ([-0.6, -0.5, -0.7], [0.5, 0.7, 0.6])
GROUND_Z = -0.7


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_path"), "host_relight.cpp", "host_path.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


def env_light(seed=5, H=16, W=32):
    g = np.random.default_rng(seed)
    rgb = g.uniform(0, 1, (H, W, 3)).astype(np.float32) ** 4 * 3
    return Environment_Light({"m": rgb}, device="cpu")


def ground_rays(seed, n):
    """n primary rays from cameras around the box, most of them meeting the ground plane, a few pointing up."""
    g = np.random.default_rng(seed)
    az = g.uniform(0, 2 * np.pi, n)
    el = g.uniform(0.1, 1.2, n)
    cam = 4 * np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)
    tgt = g.uniform(-2.5, 2.5, (n, 3))
    tgt[:, 2] = GROUND_Z + g.uniform(-0.3, 0.05, n)
    d = tgt - cam
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    up = g.uniform(size=n) < 0.1
    d[up, 2] = np.abs(d[up, 2])
    return torch.from_numpy(np.concatenate([cam, d], 1).astype(np.float32))


def slab64(p, w, lo, hi):
    """float64 slab test of p + t w, t >= 0, against [lo, hi] -> (hit, t_enter)."""
    lo, hi = torch.tensor(lo, dtype=torch.float64), torch.tensor(hi, dtype=torch.float64)
    with np.errstate(divide="ignore"):
        t0, t1 = (lo - p) / w, (hi - p) / w
    tn = torch.minimum(t0, t1).amax(1).clamp(min=0)
    tf = torch.maximum(t0, t1).amin(1)
    return tn <= tf, tn


def run_ground(monkeypatch, rays, angle, box, S=48, seed=1):
    """ground_visibility on the host build with a march that records its list and returns seeded visibilities."""
    env = env_light()
    envs, keep = P.rotated_env_tables(env, ["m"], angle)
    n = rays.shape[0]
    u = torch.rand(1, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(seed))
    seen = {}

    def march(model, o, d, **kw):
        seen.update(o=o.clone(), d=d.clone(), table=kw["table"])
        v = torch.rand(o.shape[0], generator=torch.Generator().manual_seed(seed + 1))
        return v, 1 - v, torch.zeros_like(v)

    monkeypatch.setattr(ops, "march_density", march)
    bins, pos, vis = P.ground_visibility(types.SimpleNamespace(), envs, 1, rays, GROUND_Z, box, u, S, "nerv",
                                         torch.linspace(0.05, 1.0, 8))
    return env, u, bins[0], pos[0], vis, seen, keep


@pytest.mark.parametrize("angle", [0.0, 37.0, -120.0])
def test_ground_sample_against_float64(host_lib, monkeypatch, angle):
    rays = ground_rays(3, 700)
    env, u, bins, pos, vis, seen, keep = run_ground(monkeypatch, rays, angle, BOX)
    n, S = bins.shape
    cdf = env._cdf["m"]
    assert torch.equal(bins[pos != -1].long(), torch.searchsorted(cdf, u[0], right=True).clamp(max=cdf.numel() - 1)
                       [pos != -1])
    # the ground point, float64
    o, d = rays[:, :3].double(), rays[:, 3:].double()
    t = (GROUND_Z - o[:, 2]) / d[:, 2]
    ground = (d[:, 2] < 0) & (t > 0)
    assert ground.sum() > 0.8 * n and (~ground).sum() > 10
    assert (pos[~ground] == -1).all()
    table = P.rotated_env_tables(env, ["m"], angle)[1][-1]          # the rotated dir table
    w = table[bins.long()].double()                                  # [n, S, 3]
    below = w[..., 2] <= 1e-6
    gmask = ground[:, None].expand(n, S)
    assert torch.equal(pos[gmask & below], torch.full_like(pos[gmask & below], -1))
    assert (pos[gmask & ~below] != -1).all()
    # the ground point within fp32 rounding of float64's; the shadow rays below start from the fp32 one
    t32 = (torch.tensor(GROUND_Z, dtype=torch.float32) - rays[:, 2]) / rays[:, 5]
    p32 = rays[:, :3] + t32[:, None] * rays[:, 3:]
    p32[:, 2] = GROUND_Z
    p64 = o + t[:, None] * d
    assert ((p32.double() - p64).abs()[ground] <= 4 * EPS * (o.abs() + (t[:, None] * d).abs())[ground] + 1e-7).all()
    # the slab test decides -2, except within 1e-6 of a face
    p = p32.double()[:, None, :].expand(n, S, 3).reshape(-1, 3).clone()
    ww = w.reshape(-1, 3)
    hit, te = slab64(p, ww, *BOX)
    hit_in, _ = slab64(p, ww, [x + 1e-6 for x in BOX[0]], [x - 1e-6 for x in BOX[1]])
    hit_out, _ = slab64(p, ww, [x - 1e-6 for x in BOX[0]], [x + 1e-6 for x in BOX[1]])
    sure = (hit_in == hit_out).reshape(n, S) & gmask & ~below
    flat = pos.reshape(n, S)
    assert sure.sum() > 0.9 * (gmask & ~below).sum()
    assert torch.equal(flat[sure] == -2, ~hit.reshape(n, S)[sure])
    both = (gmask & ~below) & (flat >= 0)
    assert both.sum() > 200 and (flat == -2).sum() > 200
    # the list, in slot order: origins moved to SHADOW_NEAR before the box entry, directions the table's
    rows = flat[both].long()
    assert torch.equal(rows, torch.arange(rows.numel()))
    te = te.reshape(n, S)[both]
    o64 = p.reshape(n, S, 3)[both] + (te - 0.05).clamp(min=0)[:, None] * w[both]
    bound = 8 * EPS * (p.reshape(n, S, 3)[both].abs() + te[:, None] * w[both].abs() + 1)
    assert ((seen["o"].double() - o64).abs() <= bound).all()
    assert torch.equal(seen["d"], w[both].float())
    del keep


def test_ground_sample_empty_box(host_lib, monkeypatch):
    rays = ground_rays(4, 300)
    _, _, _, pos, _, seen, _ = run_ground(monkeypatch, rays, 15.0, ([1.0, 1.0, 1.0], [-1.0, -1.0, -1.0]))
    assert set(pos.unique().tolist()) == {-1, -2} and "o" not in seen


def composite_inputs(seed, n, S, env, angle, p_unocc=0.3, vis_one=False):
    """Seeded bins, pos and vis of n ground rays as tir_ground_sample leaves them: bins of texels above the horizon
    of the map rotated by ``angle``, pos -1, -2 or a list row, visibilities in [0, 1]."""
    g = torch.Generator().manual_seed(seed)
    up = (P.rotated_env_tables(env, ["m"], angle)[1][-1][:, 2] > 1e-6).nonzero().reshape(-1)
    bins = up[torch.randint(0, up.numel(), (1, n, S), generator=g)].to(torch.int32)
    r = torch.rand(1, n, S, generator=g)
    pos = torch.full((1, n, S), -1, dtype=torch.int32)
    pos[r < 1 - 0.1] = -2
    marched = r < 1 - 0.1 - p_unocc
    pos[marched] = torch.arange(int(marched.sum()), dtype=torch.int32)
    vis = torch.ones(max(int(marched.sum()), 1)) if vis_one else torch.rand(max(int(marched.sum()), 1), generator=g)
    return bins, pos, vis


def run_composite(rays, acc, angle, ground_z, vis_in, env, S, wo=None):
    envs, keep = P.rotated_env_tables(env, ["m"], angle)
    n = rays.shape[0]
    without = torch.rand(1, n + 2, 3, generator=torch.Generator().manual_seed(9)) if wo is None else wo
    with_bg = torch.full((1, n + 2, 3), -7.0)
    shadow = torch.full((1, n + 2, 3), -7.0)
    P.path_composite(envs, 1, rays, acc, angle, ground_z, vis_in, S, "nerv", (with_bg, without), 1, shadow)
    return with_bg, without, shadow


def test_composite_ratio_against_float64(host_lib):
    env = env_light(7)
    n, S = 400, 96
    rays = ground_rays(5, n)
    acc = torch.rand(n, generator=torch.Generator().manual_seed(2))
    bins, pos, vis = composite_inputs(11, n, S, env, 30.0)
    with_bg, without, shadow = run_composite(rays, acc, 30.0, GROUND_Z, (bins, pos, vis), env, S)
    assert (with_bg[:, 0] == -7).all() and (with_bg[:, -1] == -7).all()
    tab = P.rotated_env_tables(env, ["m"], 30.0)[1][-1].double()
    rgb = env.hdr_rgbs["m"].reshape(-1, 3).double()
    pdf = env.hdr_pdf_return["m"].reshape(-1).double()
    b, q = bins[0].long(), pos[0].long()
    v = torch.where(q >= 0, vis.double()[q.clamp(min=0)], torch.ones_like(q, dtype=torch.float64))
    keep = (q != -1).double()
    w = (tab[b, 2] / pdf[b] * keep)[..., None] * rgb[b]              # [n, S, 3]
    num, den = (w * v[..., None]).sum(1), w.sum(1)
    r64 = torch.where(den > 0, (num / den).clamp(0, 1), torch.ones_like(den))
    d = rays[:, 5].double()
    ground = (d < 0) & ((GROUND_Z - rays[:, 2].double()) / d > 0)
    r64[~ground] = 1
    # each term: 3 roundings; each sum of positive terms: at most S - 1 additions in the lanes' order and the
    # butterfly; num <= den, so the quotient is off by at most twice the relative error of the sums
    bound = (2 * (S + 4) + 2) * EPS * (r64 + 1)
    assert ((shadow[0, 1:-1].double() - r64).abs() <= bound).all()
    assert (shadow[0, 1:-1][~ground] == 1).all()


def test_composite_unoccluded_is_exactly_one(host_lib):
    env = env_light(8)
    n, S = 200, 64
    rays = ground_rays(6, n)
    bins, pos, vis = composite_inputs(12, n, S, env, 0.0, vis_one=True)
    _, _, shadow = run_composite(rays, torch.zeros(n), 0.0, GROUND_Z, (bins, pos, vis), env, S)
    assert (shadow[0, 1:-1] == 1).all()


def test_composite_without_ground_is_relight_shade(host_lib):
    """Identity rotation and no ground: with_bg has the bits of the host rl_composite path of tir_relight_shade."""
    from test_lighting_cpu import random_chunk
    env = env_light(9)
    n, S = 300, 40
    ch = random_chunk(21, n, 1)
    u = torch.rand(1, n, S, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
    envs, keep = R.env_tables(env, ["m"])
    bins, pos = torch.zeros(1, n, S, dtype=torch.int32), torch.zeros(1, n, S, dtype=torch.int32)
    cnt = torch.zeros(1, dtype=torch.int64)
    lo, ld = torch.empty(n * S, 3), torch.empty(n * S, 3)
    host_lib.tir_relight_sample(envs, 1, C.c_void_p(ch["rays"].data_ptr()), C.c_void_p(ch["depth"].data_ptr()),
                               C.c_void_p(ch["normal"].data_ptr()), C.c_void_p(ch["acc"].data_ptr()), n, S, 0.5,
                               C.c_void_p(u.data_ptr()), C.c_void_p(bins.data_ptr()), C.c_void_p(pos.data_ptr()),
                               C.c_void_p(lo.data_ptr()), C.c_void_p(ld.data_ptr()), n * S,
                               C.c_void_p(cnt.data_ptr()), None)
    vis = torch.rand(max(int(cnt), 1), generator=torch.Generator().manual_seed(5))
    out = (torch.full((1, n, 3), -7.0), torch.full((1, n, 3), -7.0))
    R.relight_shade(envs, 1, ch["rays"], ch["normal"], ch["albedo"], ch["rough"], ch["fresnel"], ch["acc"], S, 0.5,
                    torch.tensor([1.1, 0.9, 1.0]), (bins, pos, vis), "nerv", out, 0)
    with_bg = torch.full((1, n, 3), -7.0)
    P.path_composite(envs, 1, ch["rays"], ch["acc"], 0.0, None, None, S, "nerv", (with_bg, out[1]), 0)
    assert torch.equal(with_bg, out[0])
    # and the rotated table of angle 0 is the map's own, to the bit
    _, keep0 = P.rotated_env_tables(env, ["m"], 0.0)
    assert torch.equal(keep0[-1], env.hdr_dir["m"].reshape(-1, 3))


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def test_argument_checks_launch_nothing(host_lib):
    env = env_light(3)
    envs, keep = R.env_tables(env, ["m"])
    n, S = 8, 4
    rays, acc = ground_rays(1, n), torch.ones(n)
    u = torch.rand(1, n, S, dtype=torch.float64)
    bins, pos = torch.full((1, n, S), 77, dtype=torch.int32), torch.full((1, n, S), 77, dtype=torch.int32)
    lo, ld = torch.full((n * S, 3), 5.0), torch.full((n * S, 3), 5.0)
    cnt = torch.zeros(1, dtype=torch.int64)
    blo, bhi = (C.c_float * 3)(*BOX[0]), (C.c_float * 3)(*BOX[1])

    def sample(envs=envs, L=1, rays=rays, n=n, blo=blo, bhi=bhi, S=S, u=u, bins=bins, pos=pos, lo=lo, ld=ld, cap=n * S,
               cnt=cnt):
        return host_lib.tir_ground_sample(envs, L, _ptr(rays), n, GROUND_Z, blo, bhi, S, _ptr(u), _ptr(bins), _ptr(pos),
                                         _ptr(lo), _ptr(ld), cap, _ptr(cnt), None)

    many = (_lib.TirEnvMap * 17)(*([envs[0]] * 17))
    for rc, kw in ((-1, dict(rays=None)),
                   (-1, dict(u=None)), (-1, dict(bins=None)), (-1, dict(pos=None)), (-1, dict(cnt=None)),
                   (-1, dict(blo=None)), (-1, dict(lo=None)), (-1, dict(envs=None)),
                   (-2, dict(envs=many, L=17)), (-2, dict(n=-1)), (-2, dict(S=-1)), (-2, dict(cap=-1))):
        assert sample(**kw) == rc, kw
        assert (bins == 77).all() and (pos == 77).all() and (lo == 5).all() and int(cnt) == 0
    assert sample() == 0 and int(cnt) >= 0

    vis = torch.rand(n * S)
    wo, wb = torch.rand(1, n, 3), torch.full((1, n, 3), -7.0)
    rot = (C.c_float * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1)

    def comp(envs=envs, L=1, rays=rays, acc=acc, n=n, rot=rot, gz=GROUND_Z, bins=bins, pos=pos, vis=vis, kind=0, S=S,
             wo=wo, wb=wb, rows=n, row0=0):
        return host_lib.tir_path_composite(envs, L, _ptr(rays), _ptr(acc), n, rot, gz, _ptr(bins), _ptr(pos),
                                          _ptr(vis), kind, S, _ptr(wo), _ptr(wb), None, rows, row0, None)

    for rc, kw in ((-1, dict(rays=None)), (-1, dict(acc=None)), (-1, dict(rot=None)), (-1, dict(wo=None)),
                   (-1, dict(wb=None)), (-1, dict(bins=None)), (-1, dict(pos=None)), (-1, dict(vis=None)),
                   (-1, dict(envs=None)), (-2, dict(envs=many, L=17)), (-3, dict(kind=2)), (-2, dict(rows=n - 1)),
                   (-2, dict(row0=1)), (-2, dict(row0=-1)), (-2, dict(S=0)), (-2, dict(n=-1))):
        assert comp(**kw) == rc, kw
        assert (wb == -7).all()
    # without a ground, bin / pos / vis are not read
    assert comp(gz=float("nan"), bins=None, pos=None, vis=None) == 0 and (wb != -7).all()


# ---- cameras and the command line --------------------------------------------------------------------------------

def test_orbit_poses():
    tgt = np.array([0.1, -0.2, 0.3])
    poses = P.orbit_poses(12, 3.5, 25.0, tgt, start_deg=40.0).double()
    assert poses.shape == (12, 4, 4)
    for k, c2w in enumerate(poses):
        Rm, pos = c2w[:3, :3], c2w[:3, 3]
        assert torch.allclose(Rm.T @ Rm, torch.eye(3, dtype=torch.float64), atol=1e-6)
        assert abs(torch.det(Rm) - 1) < 1e-6                                  # right-handed: x right, y down, z fwd
        to = torch.tensor(tgt) - pos
        assert abs(to.norm() - 3.5) < 1e-5
        assert torch.allclose(Rm[:, 2], to / to.norm(), atol=1e-6)             # +z looks at the target
        up_cam = Rm.T @ torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)     # world +z in camera axes
        assert abs(up_cam[0]) < 1e-6 and up_cam[1] < 0                         # straight up in the image
        assert math.degrees(math.asin(-to[2] / to.norm())) == pytest.approx(25.0, abs=1e-4)
        az = math.degrees(math.atan2(-to[1], -to[0]))
        assert (az - (40.0 + 30.0 * k) + 180) % 360 - 180 == pytest.approx(0.0, abs=1e-4)
    r, el, az = P.orbit_of(poses[3], tgt)
    assert (r, el, az) == pytest.approx((3.5, 25.0, 130.0), abs=1e-4)
    with pytest.raises(ValueError):
        P.orbit_poses(4, 2.0, 90.0, tgt)
    with pytest.raises(ValueError):
        P.orbit_poses(0, 2.0, 10.0, tgt)


def test_rotation_matrix_is_the_reference_light_rotation():
    from tensoir_b200.tensorf import TensorVMSplit
    m = TensorVMSplit(torch.tensor([[-1.5] * 3, [1.5] * 3]), [8] * 3, "cpu", light_rotation=["000", "090", "213"],
                      density_n_comp=[4] * 3, appearance_n_comp=[4] * 3, app_dim=6, featureC=8, numLgtSGs=8,
                      shadingMode="MLP_Fea", light_kind="sg")
    for k, a in enumerate((0, 90, 213)):
        assert torch.equal(P.rotation_matrix(a), m.light_rotation_matrix[k].cpu())


def test_path_and_rotation_specs(tmp_path):
    assert P.parse_rotation("0:360") == (0.0, 360.0) and P.parse_rotation("-45.5:10") == (-45.5, 10.0)
    for bad in ("0", "0:1:2", "a:1", "", "nan:1", "0:inf", None):
        with pytest.raises(ValueError):
            P.parse_rotation(bad)
    assert P.frame_angles(4, (0.0, 360.0)) == [0.0, 90.0, 180.0, 270.0]
    assert P.parse_path("orbit") == ("orbit", "orbit") and P.parse_path("test") == ("test", "test")
    f = tmp_path / "poses.json"
    poses = P.orbit_poses(3, 4.0, 30.0, [0, 0, 0])
    f.write_text(json.dumps(poses.tolist()))
    assert P.parse_path(str(f)) == ("file", str(f)) and torch.equal(P.load_poses(str(f)), poses)
    for bad in ("", str(tmp_path / "missing.json")):
        with pytest.raises(ValueError):
            P.parse_path(bad)
    for content in ([[1, 2], [3, 4]], [], [[[0.0] * 4] * 3], [[[float("nan")] * 4] * 4], "x"):
        f.write_text(json.dumps(content))
        with pytest.raises(ValueError):
            P.load_poses(str(f))


def _tool():
    spec = importlib.util.spec_from_file_location("render_path_tool", os.path.join(REPO, "tools", "render_path.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_tool_options(tmp_path):
    tool = _tool()
    argv = ["x", "--config", "c.txt", "--path", "orbit", "--frames", "8", "--ground", "--out", "o", "--ckpt", "k"]
    opts = tool.path_options(argv)
    assert argv == ["x", "--config", "c.txt", "--ckpt", "k"]
    assert opts == dict(path=("orbit", "orbit"), frames=8, rotation=(0.0, 0.0), ground=True, light=None, out="o")
    argv = ["x", "--ground", "-0.9", "--env_rotation", "0:360", "--light", "learned", "--out", "o"]
    opts = tool.path_options(argv)
    assert argv == ["x"] and opts["ground"] == -0.9 and opts["rotation"] == (0.0, 360.0) and opts["light"] == "learned"
    assert opts["path"] == ("orbit", "orbit") and opts["frames"] == 120
    for bad in (["--path", "test", "--frames", "4", "--out", "o"],          # frames belong to an orbit
                ["--path", "nowhere.json", "--out", "o"],
                ["--env_rotation", "90", "--out", "o"],
                ["--light", "sun", "--out", "o"],
                ["--frames", "0", "--out", "o"],
                ["--frames", "many", "--out", "o"],
                ["--ground", "nan", "--out", "o"],
                ["--path", "orbit"]):                                     # no --out
        with pytest.raises(SystemExit):
            tool.path_options(["x"] + bad)


def test_learned_light_of_a_general_model_is_rejected():
    import types
    with pytest.raises(ValueError, match="fit_lights"):
        P.path_maps(types.SimpleNamespace(light="learned"),
                    types.SimpleNamespace(general_lights=True, aabb=torch.zeros(2, 3)), None)
    for args in (types.SimpleNamespace(sampling="mis"), types.SimpleNamespace(indirect_samples=4)):
        with pytest.raises(ValueError):
            P.check_estimator(args)
    P.check_estimator(types.SimpleNamespace())
