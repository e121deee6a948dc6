"""CPU test of the autograd plumbing of heads._FusedHeadsMulti (H heads, own points per head, ONE stacked backward):
the CUDA entry points are replaced by torch emulations of what they compute, and every gradient the node returns is
compared with torch autograd of the same composition.  Exercises slot ordering, zero-padding of 3-output heads, the
three light modes, group-wise summation before the appearance scatter and weight sharing between two heads, and the
single-head wrapper on a model without light_line (the light-free radiance head of TensorVMSplitInit)."""
import types

import pytest
import torch

from tensoir_b200 import heads

F_DIM, AC3, HID, PE = 27, 144, 128, 2
IN_DIM = F_DIM + 3 + 2 * F_DIM * PE + 2 * 3 * PE


def _pe(x):
    freqs = 2.0 ** torch.arange(PE, dtype=x.dtype)
    p = (x[..., None] * freqs).reshape(x.shape[0], -1)
    return torch.sin(p), torch.cos(p)


def _mlp_input(feat, x_in):
    sf, cf = _pe(feat)
    sx, cx = _pe(x_in)
    return torch.cat([feat, x_in, sf, cf, sx, cx], dim=-1)


class _Mod(torch.nn.Module):
    def __init__(self, od):
        super().__init__()
        self.mlp = torch.nn.Sequential(torch.nn.Linear(IN_DIM, HID), torch.nn.ReLU(), torch.nn.Linear(HID, HID),
                                       torch.nn.ReLU(), torch.nn.Linear(HID, od))


def _light_rows(light, light_w, li, n):
    if light == "index":
        return light_w.index_select(0, li.long())
    if light == "mean":
        return light_w.mean(0, keepdim=True).expand(n, -1)
    return None


@pytest.fixture
def world(monkeypatch):
    torch.manual_seed(21)
    model = types.SimpleNamespace(
        renderModule=_Mod(3), renderModule_brdf=_Mod(4), renderModule_normal=_Mod(3),
        basis_mat=torch.nn.Linear(AC3, F_DIM, bias=False), light_line=torch.nn.Embedding(3, AC3),
        app_plane=[torch.nn.Parameter(torch.zeros(1)) for _ in range(3)],
        app_line=[torch.nn.Parameter(torch.zeros(1)) for _ in range(3)])
    proj = torch.randn(3, AC3)                       # stands for the VM gather: raw products x0 = tanh(xn @ proj)
    scattered = []

    def raw_products(_model, xn):
        return torch.tanh(xn @ proj)

    def head_forward(_model, head, light, xn, x_in, li, w0, need, bufs=None):
        mod = getattr(_model, head)
        x0 = raw_products(_model, xn)
        ll = getattr(_model, "light_line", None)
        rows = None if ll is None else _light_rows(light, ll.weight.detach(), li, xn.shape[0])
        xl = x0 if rows is None else x0 * rows
        inp = _mlp_input(xl @ _model.basis_mat.weight.detach().t(), x_in)
        h1 = torch.relu(inp @ mod.mlp[0].weight.detach().t() + mod.mlp[0].bias.detach())
        h2 = torch.relu(h1 @ mod.mlp[2].weight.detach().t() + mod.mlp[2].bias.detach())
        z = h2 @ mod.mlp[4].weight.detach().t() + mod.mlp[4].bias.detach()
        out = torch.tanh(z) if head == "renderModule_normal" else torch.sigmoid(z)
        if need:
            for dst, src in zip(bufs, (xl, inp, h1, h2)):
                dst.copy_(src)
        return out, None, None, None, None

    class FakeLib:
        def tir_vm_app_products_bwd(self, f, xn, n, gx0, gp, gl, stream):
            scattered.append(FakeLib.last_gx0)
            return 0
    monkeypatch.setattr(heads, "_head_forward", head_forward)
    monkeypatch.setattr(heads, "_raw_products", raw_products)
    monkeypatch.setattr(heads._lib, "load", lambda: FakeLib())
    monkeypatch.setattr(heads._lib, "stream_ptr", lambda: None)

    def fake_dptr(t, *a, **k):
        FakeLib.last_gx0 = t                         # the last tensor handed over before the call is gx0's neighbour
        return t
    monkeypatch.setattr(heads._lib, "dptr", fake_dptr)
    monkeypatch.setattr(heads, "_ptr_array", lambda ts: None)
    monkeypatch.setattr(heads, "_grad_shadows", lambda df, kind: ([torch.zeros(1, 1, 1)] * 3, [torch.zeros(1, 1, 1)] * 3))
    field = heads._lib.TirField()
    field.aC = AC3 // 3
    monkeypatch.setattr(heads.ops, "device_field", lambda m: types.SimpleNamespace(refresh=lambda mm: field))
    return model, proj, scattered


def _check_against_autograd(model, proj, scattered, specs, outs):
    """Every gradient of the node against torch autograd of the same composition, and one appearance scatter per point
    set fed with the summed d loss / d x0 of the heads at those points."""
    n = specs[0][1].shape[0]
    ll = getattr(model, "light_line", None)
    mods = [getattr(model, h) for h in dict.fromkeys(s[0] for s in specs)]
    params = [p for m in mods for p in m.parameters()] + [model.basis_mat.weight] + ([] if ll is None else [ll.weight])
    G = [torch.randn_like(o) for o in outs]
    torch.autograd.backward(outs, G)
    got = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None

    # reference: the same composition, differentiated by autograd (x0 of each point set as a leaf to get d/d x0)
    x0s = {}
    for _, xn, _, _, _ in specs:
        x0s.setdefault(id(xn), torch.tanh(xn @ proj).requires_grad_(True))
    ref = []
    for head, xn, x_in, l, light in specs:
        mod = getattr(model, head)
        rows = None if ll is None else _light_rows(light, ll.weight, l if l is not None else torch.empty(0), n)
        xl = x0s[id(xn)] if rows is None else x0s[id(xn)] * rows
        z = mod.mlp(_mlp_input(model.basis_mat(xl), x_in))
        ref.append(torch.tanh(z) if head == "renderModule_normal" else torch.sigmoid(z))
    for o, r in zip(outs, ref):
        assert torch.allclose(o, r.detach(), atol=1e-6)
    torch.autograd.backward(ref, G)
    for p, g in zip(params, got):
        assert torch.allclose(g, p.grad, rtol=2e-4, atol=2e-5), tuple(p.shape)
    assert len(scattered) == len(x0s)
    for sc, x0 in zip(scattered, x0s.values()):
        assert torch.allclose(sc, x0.grad, rtol=2e-4, atol=2e-5)


def test_multi_head_backward_matches_autograd(world):
    model, proj, scattered = world
    n = 300
    x_a, x_j = torch.rand(n, 3) * 2 - 1, torch.rand(n, 3) * 2 - 1
    vd = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
    li = torch.randint(0, 3, (n,), dtype=torch.int32)
    specs = [("renderModule", x_a, vd, li, "index"), ("renderModule_brdf", x_a, x_a, None, "mean"),
             ("renderModule_normal", x_a, x_a, None, "mean"), ("renderModule_brdf", x_j, x_j, None, "mean")]
    _check_against_autograd(model, proj, scattered, specs, heads.fused_heads_multi(model, specs))


def test_single_head_without_light_matches_autograd(world):
    """heads.fused_head on a model without light_line, light "none": one head through the same stacked node."""
    model, proj, scattered = world
    del model.light_line
    n = 300
    x_a = torch.rand(n, 3) * 2 - 1
    vd = torch.nn.functional.normalize(torch.randn(n, 3), dim=-1)
    out = heads.fused_head(model, "renderModule", x_a, vd, None, light="none")
    _check_against_autograd(model, proj, scattered, [("renderModule", x_a, vd, None, "none")], (out,))
