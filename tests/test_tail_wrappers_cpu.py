"""tensoir_b200/tail.py end to end on the CPU: the library handle is replaced by a host build of the SAME entry points
(tests/host_tail.cpp: identical C-ABI signatures, argument checks and per-item math, loops instead of kernels), so the
real ctypes marshalling (argument order, TirRayMaps packing, NULL handling) and the autograd wrappers run and are
compared with torch autograd of the expressions they replace."""
import pytest
import torch

from helpers import build_host_lib, use_host
from tensoir_b200 import tail


@pytest.fixture(scope="module")
def host_so(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("host_tail"), "host_tail.cpp")


@pytest.fixture
def host_lib(host_so, monkeypatch):
    use_host(monkeypatch, host_so)
    return host_so


def _rel(a, b):
    base = torch.maximum(a, b).clip(min=1e-6)
    return torch.sum(((a - b) / base) ** 2, dim=-1, keepdim=True)


def _torch_tail(w, ray, rgb, brdf, brdfj, vn, dn, viewdirs, n_rays):
    v_alb, v_rough = brdf[..., :3], brdf[..., 3:4] * 0.9 + 0.09
    a_cost, r_cost = _rel(v_alb, brdfj[..., :3]), _rel(v_rough, brdfj[..., 3:4] * 0.9 + 0.09)
    vd = viewdirs.index_select(0, ray)
    if dn is not None:
        nd = torch.sum(torch.pow(vn - dn, 2), dim=-1, keepdim=True)
        no = torch.sum(vd * vn, dim=-1, keepdim=True).clamp(min=0)
    else:
        nd = no = torch.zeros_like(a_cost)
    return torch.zeros(n_rays, 14).index_add_(0, ray, w[:, None] * torch.cat(
        [rgb, vn, v_alb, v_rough, a_cost, r_cost, nd, no], dim=-1))


def _torch_epilogue(packed, acc, depth, rays, fresnel0, bg):
    from tensoir_b200.relight_utils import linear2srgb_torch
    rgb, normal, albedo = packed[:, 0:3], packed[:, 3:6], packed[:, 6:9]
    rough, ac, rc, nd, no = packed[:, 9:10], packed[:, 10:11], packed[:, 11:12], packed[:, 12:13], packed[:, 13:14]
    fres = torch.zeros_like(albedo).fill_(fresnel0)
    if bg:
        depth = depth + (1. - acc) * rays[..., -1]
        rgb = rgb + (1. - acc[..., None])
        normal = normal + (1 - acc[..., None]) * torch.tensor([0., 0., 1.])
        albedo, rough, fres = albedo + (1 - acc[..., None]), rough + (1 - acc[..., None]), fres + (1 - acc[..., None])
    return (linear2srgb_torch(rgb.clamp(0, 1)), depth, torch.nn.functional.normalize(normal, p=2, dim=-1, eps=1e-6),
            albedo.clamp(0, 1), rough.clamp(0, 1), fres.clamp(0, 1), nd, no, acc > 0.5, ac.mean(), rc.mean())


@pytest.mark.parametrize("both", [True, False])
def test_tail_wrapper(host_lib, both):
    torch.manual_seed(3)
    n, n_rays = 400, 50
    ray = torch.sort(torch.randint(0, n_rays, (n,)))[0]
    w = torch.rand(n) * 0.3
    rgb, brdf, brdfj = torch.rand(n, 3), torch.rand(n, 4), torch.rand(n, 4)
    vn = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
    dn = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1) if both else None
    rays = torch.randn(n_rays, 6)
    vd = rays[:, 3:6]                                                   # non-contiguous, as in primary.py
    G = torch.randn(n_rays, 14)
    res = []
    for fn in (tail.fused_tail, _torch_tail):
        leaves = [t.clone().requires_grad_(True) for t in (w, rgb, brdf, brdfj, vn)] + \
                 ([dn.clone().requires_grad_(True)] if both else [])
        out = fn(leaves[0], ray, leaves[1], leaves[2], leaves[3], leaves[4], leaves[5] if both else None, vd, n_rays)
        out.backward(G)
        res.append([out.detach()] + [l.grad for l in leaves])
    for got, want in zip(*res):
        assert torch.allclose(got, want, rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("bg", [True, False])
@pytest.mark.parametrize("partial", [False, True])
def test_epilogue_wrapper(host_lib, bg, partial):
    torch.manual_seed(9)
    n = 300
    packed = torch.rand(n, 14) * 1.3 - 0.1
    acc, depth, rays = torch.rand(n), torch.rand(n) * 4, torch.randn(n, 6)
    res, gs = [], None
    for fn in (tail.epilogue, _torch_epilogue):
        leaves = [t.clone().requires_grad_(True) for t in (packed, acc, depth)]
        outs = fn(leaves[0], leaves[1], leaves[2], rays, 0.04, bg)
        # the fresnel map is a constant when no background is composited: no gradient to compare
        keep = (0, 2, 10) if partial else range(len(outs))   # partial: the other outputs' gradients arrive as None
        diff = [o for k, o in enumerate(outs) if k in keep and o.dtype != torch.bool and (bg or k != 5)]
        if gs is None:
            gs = [torch.randn_like(o) for o in diff]
        torch.autograd.backward(diff, [g.reshape(o.shape) for g, o in zip(gs, diff)])
        res.append((outs, [l.grad if l.grad is not None else torch.zeros_like(l) for l in leaves]))
    for got, want in zip(res[0][0], res[1][0]):
        if got.dtype == torch.bool:
            assert torch.equal(got, want)
        else:
            assert torch.allclose(got, want.reshape(got.shape), rtol=2e-5, atol=2e-6)
    for got, want in zip(res[0][1], res[1][1]):
        assert torch.allclose(got, want, rtol=3e-4, atol=3e-5)


def test_null_and_empty_arguments(host_so):
    """The host build runs the library's own argument checks: NULL inputs fail with TIR_ERR_NULL, an empty batch is a
    no-op (the codes test_abi_cpu.py asserts of the CUDA library)."""
    for n, want in ((5, -1), (0, 0), (-1, 0)):
        assert host_so.tir_tail_fwd(n, *[None] * 10) == want
        assert host_so.tir_tail_bwd(n, *[None] * 16) == want
        assert host_so.tir_epilogue_fwd(n, None, None, None, None, 0.04, 1, None, None, None, None) == want
        assert host_so.tir_epilogue_bwd(n, None, None, None, None, 0.04, 1, *[None] * 7) == want
