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
    assert lib.tir_abi_version() == 3


def test_struct_sizes_match_header(lib):
    from tensoir_b200 import _lib
    assert (ctypes.sizeof(_lib.TirField), ctypes.sizeof(_lib.TirMlp), ctypes.sizeof(_lib.TirMarchCfg)) == (248, 88, 48)
    assert _lib.APP_SAMPLE_BYTES == 24
    assert ctypes.sizeof(_lib.TirRayMaps) == 64


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
