"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every symbol
include/tensoir_b200.h declares; the product refuses to run without CUDA (no fallback)."""
import ctypes
import os
import re

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import _lib
    return _lib.load()


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(REPO, "include", "tensoir_b200.h")).read()
    names = sorted(set(re.findall(r"^int\s+(tir_\w+)\s*\(", hdr, flags=re.M)))
    assert len(names) >= 24
    from tensoir_b200 import _lib
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
        assert n in _lib.EXPORTS, f"{n} has no ctypes binding"
    assert lib.tir_abi_version() == 4


def test_struct_sizes_match_header(lib):
    from tensoir_b200 import _lib
    assert (ctypes.sizeof(_lib.TirField), ctypes.sizeof(_lib.TirMlp), ctypes.sizeof(_lib.TirMarchCfg)) == (248, 88, 48)
    assert _lib.APP_SAMPLE_BYTES == 24
    assert ctypes.sizeof(_lib.TirRayMaps) == 64
    assert ctypes.sizeof(_lib.TirAdamTensor) == 64        # p g m v, n, lr_dev, lr + l1, step


def test_primary_struct_sizes_match_the_c_compiler(lib, tmp_path):
    """The ctypes mirrors of the fused-primary structs have the size gcc gives the header's definitions."""
    import subprocess
    from tensoir_b200 import _lib
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "tensoir_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                   'sizeof(TirHeadJob),sizeof(TirPrimaryWork),sizeof(TirPrimaryBwdWork),sizeof(TirPrimaryGrads),'
                   'sizeof(TirField),sizeof(TirMlp),sizeof(TirTvPlane),sizeof(TirAdamTensor));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)], check=True)
    got = tuple(int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    want = tuple(ctypes.sizeof(t) for t in (_lib.TirHeadJob, _lib.TirPrimaryWork, _lib.TirPrimaryBwdWork,
                                            _lib.TirPrimaryGrads, _lib.TirField, _lib.TirMlp, _lib.TirTvPlane,
                                            _lib.TirAdamTensor))
    assert got == want


def test_null_arguments_are_rejected(lib):
    assert lib.tir_tv_loss(None, 1, None, None) == -1
    tab = (__import__("tensoir_b200")._lib.TirTvPlane * 1)()
    assert lib.tir_tv_loss_bwd(tab, 4, None, None) == -1           # no gout
    assert lib.tir_tv_loss(tab, 4, ctypes.c_void_p(16), None) == -2   # more planes than TIR_TV_MAX_PLANES
    assert lib.tir_tv_loss(tab, 1, ctypes.c_void_p(16), None) == -1   # plane without storage
    assert lib.tir_pack_channels_last(None, None, 1, 1, 1, None) == -1
    assert lib.tir_density_points(None, None, 5, None, None, None) == -1
    assert lib.tir_tail_fwd(5, None, None, None, None, None, None, None, None, None, None) == -1
    assert lib.tir_epilogue_fwd(5, None, None, None, None, 0.04, 1, None, None, None, None) == -1
    assert lib.tir_tail_fwd(0, None, None, None, None, None, None, None, None, None, None) == 0      # empty: no-op
    assert lib.tir_density_points(None, None, 0, None, None, None) == 0      # empty input is a no-op, not an error
    # the four shading entry points: NULL inputs, an empty batch, and a direct-light gradient table larger than the
    # 200 KB of shared memory the backward may use (34 lights x 512 directions x 12 B), refused before any launch
    p = ctypes.c_void_p(16)
    for n in (5, 0, -1):
        want = -1 if n > 0 else 0
        assert lib.tir_shade_fwd(*[None] * 6, n, None, None, 512, None, 3, *[None] * 4) == want
        assert lib.tir_shade_bwd(*[None] * 6, n, None, None, 512, None, 3, *[None] * 9) == want
        assert lib.tir_shade_hits_fwd(*[None] * 7, n, None, None, 512, None, 3, None, None, 1, None, None, None) == want
        assert lib.tir_shade_hits_bwd(*[None] * 7, n, None, None, 512, None, 3, None, None, 1, *[None] * 8) == want
    assert lib.tir_shade_bwd(*[p] * 6, 5, p, p, 512, p, 34, *[p] * 8, None) == -2
    assert lib.tir_shade_hits_bwd(*[p] * 7, 5, p, p, 512, p, 34, p, p, 1, *[p] * 7, None) == -2
    assert lib.tir_shade_hits_bwd(*[p] * 7, 5, p, p, 512, p, 33, p, p, 1, *[p] * 6, None, None) == -1
    # the march entry points: NULL inputs, empty inputs, and the shape / capacity / config checks, all before any
    # launch.  The checks that read the structs get a real TirField (dC = 16), TirMarchCfg and TirDensityVolume.
    from tensoir_b200 import _lib
    fld = _lib.TirField()
    fld.dC, fld.aC, fld.grid[:] = 16, 48, [8, 8, 8]
    cfg = _lib.TirMarchCfg()
    cfg.sampling, cfg.n_samples, cfg.z_table = _lib.SAMPLE_TABLE, 96, 16
    vol = _lib.TirDensityVolume()                                   # an empty box: no volume data needed
    mlp = _lib.TirMlp()
    F_, G_, V_, M_ = ctypes.byref(fld), ctypes.byref(cfg), ctypes.byref(vol), ctypes.byref(mlp)

    # every call below is refused, so the stand-in pointers are never dereferenced
    def radiance(n, f=F_, g=G_, cap=64, null=False):
        q = None if null else p
        return lib.tir_march_radiance(f, None if null else M_, q, q, None, n, g, q, q, q, q, q, q, cap, None, None)

    def march(n, f=F_, g=G_, null=False):
        q = None if null else p
        return lib.tir_march_density(f, q, q, n, g, q, q, q, None, None), radiance(n, f, g, null=null)

    def secondary_vol(n_pts, n_dirs=512, f=F_, g=G_, cap=64, null=False, v=V_):
        q, m = (None, None) if null else (p, M_)
        return (lib.tir_secondary_march_vol(f, q, q, n_pts, q, n_dirs, g, v, q, q, q, cap, None, None),
                lib.tir_secondary_radiance_vol(f, m, q, q, None, n_pts, q, n_dirs, g, v, q, q, q, q, cap, None, None))

    def secondary(n_pts, n_dirs=512, f=F_, g=G_, cap=64, null=False):
        q, m = (None, None) if null else (p, M_)
        return (lib.tir_secondary_march(f, q, q, n_pts, q, n_dirs, g, q, q, q, cap, None, None),
                lib.tir_secondary_radiance(f, m, q, q, None, n_pts, q, n_dirs, g, q, q, q, q, cap, None, None)) \
            + secondary_vol(n_pts, n_dirs, f, g, cap, null)
    assert march(5, null=True) == (-1, -1) and march(5, f=None, g=None) == (-1, -1)
    assert secondary(5, null=True) == (-1,) * 4 and secondary(5, f=None, g=None) == (-1,) * 4
    for n in (0, -1):                                               # empty inputs: no-ops, whatever the pointers
        assert march(n, null=True) == (0, 0) and secondary(n, null=True) == (0,) * 4
    assert secondary_vol(5, v=None) == (-1, -1)                   # the volume entry points without a volume
    for n_dirs in (0, -3):
        assert secondary(5, n_dirs=n_dirs) == (-2,) * 4
    for cap in (0, -1):
        assert radiance(5, cap=cap) == -4 and secondary(5, cap=cap) == (-4,) * 4
    for n_samples in (0, -2):
        cfg.n_samples = n_samples
        assert march(5) == (-3, -3) and secondary(5) == (-3,) * 4
    cfg.n_samples = 96
    fld.dC = 8
    assert march(5) == (-2, -2) and secondary(5) == (-2,) * 4
    fld.dC = 16
    cfg.sampling = 7
    assert march(5) == (-3, -3) and secondary(5) == (-3,) * 4
    cfg.sampling = _lib.SAMPLE_TABLE
    cfg.z_table = None
    assert march(5) == (-1, -1) and secondary(5) == (-1,) * 4
    cfg.z_table = 16
    vol.n[:] = [9, 1, 1]                                            # a box that leaves the 8^3 grid
    assert secondary_vol(5) == (-2, -2)
    vol.n[:] = [0, 0, 0]
    # the 3-CTA volume instance keeps 32-bit per-lane counts: n_pts * n_dirs * ceil(n_samples / 32) * 2 must stay
    # below 2^32 (here 2^21 * 512 * 3 * 2 = 6.4e9)
    assert secondary_vol(1 << 21) == (-2, -2)
    # the four fused primary entry points (tir_primary_march / _app_list / _heads / _backward): NULL and empty calls,
    # a capacity of 0, a density field that is not 16 channels, a job table with fewer than 3 jobs or without a role,
    # an indexed light on a job that does not read the ray table, and a backward without the x0 dumps; all before any
    # launch
    w = _lib.TirPrimaryWork()
    for k, _ in w._fields_:
        if k not in ("cap_valid", "cap_app", "x0", "inp", "h1", "h2", "out"):
            setattr(w, k, 16)
    w.cap_valid, w.cap_app = 64, 64
    for j in range(_lib.MAX_HEADS):
        w.out[j] = w.inp[j] = w.h1[j] = w.h2[j] = 16
    w.x0[0] = w.x0[1] = 16
    bw = _lib.TirPrimaryBwdWork()
    for k, _ in bw._fields_:
        if k in ("g_out", "gz1", "gz2", "gfeat", "gx0"):
            getattr(bw, k)[:] = [16] * _lib.MAX_HEADS
        else:
            setattr(bw, k, 16)
    grs = _lib.TirPrimaryGrads()
    maps = _lib.TirRayMaps()
    jobs = (_lib.TirHeadJob * 4)()
    for j, (role, ps, x_in, lm) in enumerate(((0, 0, 0, 1), (1, 0, 1, 2), (2, 1, 1, 2), (3, 0, 1, 2))):
        jobs[j].role, jobs[j].point_set, jobs[j].x_in, jobs[j].light_mode = role, ps, x_in, lm
        jobs[j].mlp.light_line = 16
    W_, B_, J_, R_ = ctypes.byref(w), ctypes.byref(bw), ctypes.byref(grs), ctypes.byref(maps)
    # every call below is refused before any launch (or is empty), so the stand-in pointers are never dereferenced
    def pmarch(n, f=F_, null=False):
        return lib.tir_primary_march(f, None if null else p, n, None if null else G_, None if null else W_, None, None)

    def pheads(n, f=F_, nj=4, kind=0, null=False):
        q = None if null else p
        return lib.tir_primary_heads(f, None if null else jobs, nj, kind, q, q, n, None if null else W_, 0.04, 1,
                                     None if null else R_, q, q, None, None)

    def pbackward(n, f=F_, nj=4, kind=0, null=False):
        q = None if null else p
        return lib.tir_primary_backward(f, None if null else jobs, nj, kind, q, q, n, None if null else W_,
                                        None if null else B_, 0.04, 1, None if null else R_, None, None, None,
                                        None if null else J_, None)

    def primary(n, f=F_, null=False):
        return (pmarch(n, f, null), lib.tir_primary_app_list(f, n, None if null else W_, None),
                pheads(n, f, null=null), pbackward(n, f, null=null))
    assert primary(5, null=True) == (-1,) * 4 and primary(5, f=None) == (-1,) * 4
    for n in (0, -1):
        assert primary(n, null=True) == (0,) * 4
    for cap in ("cap_valid", "cap_app"):
        setattr(w, cap, 0)
        assert pmarch(5) == -4
        setattr(w, cap, 64)
    fld.dC = 8
    assert pmarch(5) == -2
    fld.dC = 16
    assert (pheads(5, nj=2), pbackward(5, nj=2)) == (-3, -3)      # fewer than 3 jobs
    for j, role in ((0, 0), (1, 1), (2, 2)):                         # without the rgb / brdf / brdf-jitter role
        jobs[j].role = 3
        assert (pheads(5, nj=3, kind=2), pbackward(5, nj=3, kind=2)) == (-3, -3)
        jobs[j].role = role
    assert (pheads(5, nj=3, kind=0), pbackward(5, nj=3, kind=0)) == (-3, -3)   # predicted normals, no normal head
    jobs[1].light_mode = 1                                          # an indexed light without the ray table
    assert pheads(5) == -3
    jobs[1].light_mode = 2
    w.x0[1] = None                                                  # the backward needs both x0 dumps
    assert pbackward(5) == -1
    w.x0[1] = 16


def test_no_cpu_fallback():
    from tensoir_b200 import _lib
    with pytest.raises(_lib.TirError):
        _lib.dptr(torch.zeros(3))


def test_model_surface_matches_reference_keys(golden_rotated, golden_general, golden_init):
    """state_dict keys / shapes are the reference's (checkpoint compatibility, SURVEY.md §8b)."""
    from gpu_helpers import model_from_fixture
    for fx in (golden_rotated, golden_general, golden_init):
        m = model_from_fixture(fx, "cpu")
        sd = m.state_dict()
        assert set(sd.keys()) == set(fx["state_dict"].keys())
        for k, v in fx["state_dict"].items():
            assert tuple(sd[k].shape) == tuple(v.shape)
        assert fx["kind"] != "rotated" or m.nSamples == fx["nSamples"]
    m = model_from_fixture(golden_rotated, "cpu")
    groups = m.get_optparam_groups(0.02, 0.001)
    assert len(groups) == 10 and groups[0]["lr"] == 0.02 and groups[5]["lr"] == 0.001
    kw = m.get_kwargs()
    assert kw["light_rotation"] == [0, 120] and kw["gridSize"] == [24, 24, 24]


def test_light_model_matches_oracle(golden_rotated):
    from gpu_helpers import model_from_fixture
    m = model_from_fixture(golden_rotated, "cpu")
    fx = golden_rotated
    assert torch.equal(m.gen_light_incident_dirs(method='fixed_envirmap'), fx["fixed_dirs"])
    assert torch.equal(m.light_area_weight, fx["area_weight"])
    assert torch.equal(m.get_light_rgbs(fx["fixed_dirs"], device='cpu').detach(), fx["light_rgbs"])
    from tensoir_b200.relight_utils import GGX_specular
    nrm, v2c, rough, fres = fx["ggx_in"]
    assert torch.equal(GGX_specular(nrm, v2c, fx["fixed_dirs"][None].repeat(9, 1, 1), rough, fres), fx["ggx"])


def test_regularisers_and_grid_maintenance_match_reference(golden_rotated):
    """vector_comp_diffs / density_L1 / TV losses, shrink and upsample_volume_grid (host-side, parameter-only) against
    the reference's outputs; both maintenance ops rebind Parameters, which must invalidate the kernel-side shadows."""
    from gpu_helpers import model_from_fixture
    fx = golden_rotated
    m = model_from_fixture(fx, "cpu")

    def tv(x):     # utils.TVLoss (utils.py:143-162), restated
        b, _, h, w = x.shape
        ch, cw = x[:, :, 1:, :].numel() // b, x[:, :, :, 1:].numel() // b
        return 2 * (torch.pow(x[:, :, 1:, :] - x[:, :, :h - 1, :], 2).sum() / ch
                    + torch.pow(x[:, :, :, 1:] - x[:, :, :, :w - 1], 2).sum() / cw) / b
    r = fx["reg"]
    assert torch.allclose(m.vector_comp_diffs(), r["ortho"], rtol=1e-6)
    assert torch.allclose(m.density_L1(), r["l1"], rtol=1e-6)
    assert torch.allclose(m.TV_loss_density(tv), r["tv_density"], rtol=1e-6)
    assert torch.allclose(m.TV_loss_app(tv), r["tv_app"], rtol=1e-6)
    old = m.density_plane[0]
    m.shrink(fx["new_aabb"].clone())
    sh = fx["shrink"]
    assert m.density_plane[0] is not old                                  # rebound, like the reference
    assert torch.equal(m.aabb, sh["aabb"]) and m.gridSize.tolist() == sh["grid"] and m.nSamples == sh["nSamples"]
    assert torch.equal(m.density_plane[0], sh["density_plane0"]) and torch.equal(m.app_line[2], sh["app_line2"])
    assert m._host_geom["grid"] == sh["grid"]                             # host geometry cache follows
    m.upsample_volume_grid([30, 31, 29])
    up = fx["upsample"]
    assert m.gridSize.tolist() == up["grid"] and m.nSamples == up["nSamples"]
    assert abs(float(m.stepSize) - up["stepSize"]) < 1e-9
    assert torch.equal(m.density_plane[1], up["density_plane1"]) and torch.equal(m.app_line[0], up["app_line0"])


def test_shrink_and_upsample_reproduce_the_whole_reference_state(golden_rotated):
    """shrink to an asymmetric box + upsample_volume_grid([30,31,29]) reproduce the reference's whole state_dict
    (every factor, bit-exact), aabb, gridSize, nSamples and stepSize (shrunk_g30.pt, state A), and the host geometry
    the kernels read follows all three axes."""
    from gpu_helpers import load_shrunk_state, model_from_fixture
    want = load_shrunk_state("A")
    m = model_from_fixture(golden_rotated, "cpu")
    m.shrink(want["shrink_box"].clone())
    m.upsample_volume_grid(want["upsample"])
    assert torch.equal(m.aabb, want["aabb"]) and m.gridSize.tolist() == want["grid_size"]
    assert m.nSamples == want["nSamples"] and float(m.stepSize) == want["stepSize"]
    sd = m.state_dict()
    assert set(sd) == set(want["state_dict"])
    for k, v in want["state_dict"].items():
        assert sd[k].shape == v.shape and torch.equal(sd[k], v), k
    hg = m._host_geom
    assert hg["grid"] == [30, 31, 29] and hg["lo"] == want["aabb"][0].tolist()
    assert hg["inv"] == (2.0 / (want["aabb"][1] - want["aabb"][0])).tolist()


def test_importance_sampled_light_dirs_match_reference(golden_rotated):
    from gpu_helpers import model_from_fixture
    fx = golden_rotated
    m = model_from_fixture(fx, "cpu")
    torch.manual_seed(41)
    got = m.gen_light_incident_dirs(sample_number=64, method='importance_sample', device='cpu')
    for g, w in zip(got, fx["importance_sample"]):
        assert torch.equal(g.detach(), w)
    torch.manual_seed(5)
    a = m.gen_light_incident_dirs(method='stratifed_sample_equal_areas')
    assert a.shape == (512, 3) and torch.allclose(a.norm(dim=-1), torch.ones(512), atol=1e-5)


def test_shadow_refresh_policy(golden_rotated, monkeypatch):
    """DeviceField must rebuild the channel-last shadows after ANY parameter update: fused optimizers do not bump the
    tensors' version counters, so the policy also listens to optimizer steps and honours force=True (decision logic
    only: the pack kernel itself is replaced by a counting stub, no GPU needed)."""
    from gpu_helpers import model_from_fixture
    from tensoir_b200 import device_field
    m = model_from_fixture(golden_rotated, "cpu")
    m.alphaMask = None
    packs = []

    def fake_pack(self, lib, p):
        packs.append(p.shape)
        return p.detach()[0].permute(1, 2, 0).contiguous()
    monkeypatch.setattr(device_field.DeviceField, "_pack", fake_pack)
    df = device_field.DeviceField()
    df.refresh(m)
    assert len(packs) == 12
    df.refresh(m)
    assert len(packs) == 12                                  # nothing changed: no repack
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    v0 = m.density_plane[0]._version
    torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), fused=True).step()
    assert m.density_plane[0]._version == v0                 # the reason the version key alone is not enough
    df.refresh(m)
    assert len(packs) == 24                                  # optimizer step seen through the post-step hook
    with torch.no_grad():
        m.density_plane[0].mul_(1.0)                         # in-place edit: version bump
    df.refresh(m)
    assert len(packs) == 36
    df.refresh(m, force=True)
    assert len(packs) == 48
    device_field.mark_parameters_updated()
    df.refresh(m)
    assert len(packs) == 60
    df.refresh(m)
    assert len(packs) == 60


def test_static_step_recapture_guard(golden_rotated):
    """The captured step bakes buffer addresses in; its signature must survive optimizer steps and change under the
    grid-maintenance operations that replace parameters or the alpha mask (host logic only)."""
    from gpu_helpers import model_from_fixture
    from tensoir_b200 import AlphaGridMask
    from tensoir_b200.static_step import StaticTrainStep
    m = model_from_fixture(golden_rotated, "cpu")
    st = StaticTrainStep.__new__(StaticTrainStep)
    st.model = m
    sig = st._model_signature()
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), fused=True).step()
    assert st._model_signature() == sig
    old_mask = m.alphaMask
    m.alphaMask = AlphaGridMask("cpu", old_mask.aabb, old_mask.alpha_volume.clone())
    assert st._model_signature() != sig
    m.alphaMask = old_mask
    assert st._model_signature() == sig
    m.upsample_volume_grid([g + 4 for g in golden_rotated["grid_size"]])
    assert st._model_signature() != sig


def test_lr_decay_under_captured_step_host_logic():
    """lr_tensors / scale_lr: tensor learning rates scaled in place are what the next optimizer step uses."""
    from tensoir_b200.static_step import StaticTrainStep, lr_tensors
    p = torch.nn.Parameter(torch.zeros(4))
    groups = lr_tensors([{"params": [p], "lr": 0.1}], "cpu")
    opt = torch.optim.SGD(groups, lr=1.0, foreach=False)
    st = StaticTrainStep.__new__(StaticTrainStep)
    st.opt = opt
    p.grad = torch.ones(4)
    opt.step()
    assert torch.allclose(p.detach(), torch.full((4,), -0.1))
    st.scale_lr(0.5)
    opt.step()
    assert torch.allclose(p.detach(), torch.full((4,), -0.15))
    st.opt = torch.optim.SGD([p], lr=0.1)
    with pytest.raises(TypeError):
        st.scale_lr(0.5)


def test_channel_last_parameters_need_no_shadow(golden_rotated):
    """VM factors are stored channel-last (NCHW-shaped views): DeviceField hands the kernels the parameter's own
    storage, state_dict values / shapes are the reference's, and a DP gradient bucket view has the same strides."""
    from gpu_helpers import model_from_fixture
    from tensoir_b200 import _lib, device_field
    from tensoir_b200.dp import GradBucket
    m = model_from_fixture(golden_rotated, "cpu")
    df = device_field.DeviceField()
    for p in list(m.density_plane) + list(m.app_line):
        assert p.is_contiguous(memory_format=torch.channels_last)
        view = df._pack(_lib.load(), p)
        assert view.data_ptr() == p.data_ptr() and view.is_contiguous() and view.shape == (p.shape[2], p.shape[3], p.shape[1])
        assert torch.equal(view.permute(2, 0, 1)[None], p.detach())
    for k, v in golden_rotated["state_dict"].items():
        assert torch.equal(m.state_dict()[k], v), k
    bucket = GradBucket(m.parameters())
    for p, v in zip(bucket.params, bucket.views):
        assert v.shape == p.shape and v.stride() == p.stride()


def test_tv_planes_host_logic():
    """tv.tv_planes on CPU parameters: the reference's TVLoss module is simply called (the kernel is for CUDA planes),
    and the per-plane scales handed to the kernel are 2 * weight * 1e-2 / count."""
    from tensoir_b200 import tv

    class TVLoss(torch.nn.Module):          # utils.py:143-162, restated
        TVLoss_weight = 3.0

        def forward(self, x):
            b, _, h, w = x.shape
            ch, cw = x[:, :, 1:, :].numel() // b, x[:, :, :, 1:].numel() // b
            return self.TVLoss_weight * 2 * (torch.pow(x[:, :, 1:, :] - x[:, :, :h - 1, :], 2).sum() / ch
                                             + torch.pow(x[:, :, :, 1:] - x[:, :, :, :w - 1], 2).sum() / cw) / b
    ps = [torch.nn.Parameter(torch.randn(1, 8, 5, 7).contiguous(memory_format=torch.channels_last)),
          torch.nn.Parameter(torch.randn(1, 8, 6, 4))]
    reg = TVLoss()
    v = tv.tv_planes(ps, reg, 1e-2)
    assert torch.allclose(v, sum(reg(p) * 1e-2 for p in ps))
    v.backward()
    assert ps[0].grad is not None and ps[1].grad is not None
    tab = tv._table([p.detach() for p in ps], 3.0 * 1e-2, None)
    assert (tab[0].H, tab[0].W, tab[0].C, tab[0].channel_last) == (5, 7, 8, 1)
    assert (tab[1].H, tab[1].W, tab[1].C, tab[1].channel_last) == (6, 4, 8, 0)
    assert abs(tab[0].scale_h - 2 * 3.0e-2 / (8 * 4 * 7)) < 1e-9 and abs(tab[0].scale_w - 2 * 3.0e-2 / (8 * 5 * 6)) < 1e-9
    assert tv._layout(torch.zeros(1, 4, 3, 3)[:, :, ::2]) is None
