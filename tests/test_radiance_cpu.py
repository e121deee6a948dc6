"""Host-side checks of the radiance-only primary entry points (tir_primary_radiance / _backward): argument validation
happens before anything touches the device, and the training step of the warm-up phase stages no light directions."""
import ctypes

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import _lib
    return _lib.load()


def _job(role=0, point_set=0, x_in=0, light_mode=1):
    from tensoir_b200 import _lib
    j = _lib.TirHeadJob()
    j.role, j.point_set, j.x_in, j.light_mode = role, point_set, x_in, light_mode
    return j


def test_radiance_entry_points_reject_bad_arguments(lib):
    from tensoir_b200 import _lib
    B = ctypes.byref
    f, w, b, gr = _lib.TirField(), _lib.TirPrimaryWork(), _lib.TirPrimaryBwdWork(), _lib.TirPrimaryGrads()
    p = ctypes.c_void_p(256)                  # never dereferenced: every check below returns before a launch
    fwd, bwd = lib.tir_primary_radiance, lib.tir_primary_radiance_backward
    # empty batch: a no-op whatever the arguments
    assert fwd(None, None, None, None, 0, None, 1, None, None, None) == 0
    assert bwd(None, None, None, None, 0, None, None, 1, None, None, None, None, None) == 0
    # missing field / work / outputs
    assert fwd(None, B(_job()), p, p, 5, B(w), 1, p, p, None) == -1
    assert fwd(B(f), B(_job()), p, p, 5, B(w), 1, None, p, None) == -1
    assert fwd(B(f), None, p, p, 5, B(w), 1, p, p, None) == -1
    # only the radiance head (role RGB on the appearance points, fed the view direction) is accepted
    for job in (_job(role=1), _job(role=2), _job(point_set=1), _job(x_in=1), _job(light_mode=3)):
        assert fwd(B(f), B(job), p, p, 5, B(w), 1, p, p, None) == -3
        assert bwd(B(f), B(job), p, p, 5, B(w), B(b), 1, p, None, None, B(gr), None) == -3
    # a valid job on an empty work struct: the list pointers are missing
    assert fwd(B(f), B(_job()), p, p, 5, B(w), 1, p, p, None) == -1
    assert bwd(B(f), B(_job()), p, p, 5, B(w), B(b), 1, p, None, None, B(gr), None) == -1
    assert bwd(B(f), B(_job()), p, p, 5, B(w), None, 1, p, None, None, B(gr), None) == -1


def test_phase1_static_step_stages_no_light_directions(monkeypatch):
    """StaticTrainStep(is_relight=False) draws the per-ray jitter and nothing else, so the CPU random stream of a
    captured warm-up step is the reference's (which draws no light directions before update_AlphaMask_list[0])."""
    from tensoir_b200.static_step import StaticTrainStep

    class _Model:
        envmap_h, envmap_w = 2, 4

        def gen_light_incident_dirs(self, method):
            raise AssertionError("light directions drawn in the radiance-only phase")

    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    st = StaticTrainStep(_Model(), None, 8, 16, None, None, device="cpu", is_relight=False)
    torch.manual_seed(3)
    st._stage_host_randoms(st._slots[0])
    after = torch.rand(3)
    torch.manual_seed(3)
    assert torch.equal(st.static["jitter"], torch.rand(8, 1))
    assert torch.equal(after, torch.rand(3))          # nothing else was drawn from the CPU stream
    st.is_relight = True
    with pytest.raises(AssertionError, match="light directions"):
        st._stage_host_randoms(st._slots[0])
