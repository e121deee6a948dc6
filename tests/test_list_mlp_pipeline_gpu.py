"""The list MLP (tir_app_mlp, three warpgroups per CTA) against float64 at the boundaries of its tile schedule: lists
that end just before / after a full wave of 3 x 64-row tiles per SM, lists whose last CTA leaves its third warpgroup
idle or gives it the last tile, light_line tables of 1, 16 and 17 rows, no light_line at all, and a capacity above the
device-side count.  One row per ray at weight 1, checked with the float64 reference and bounds of test_secondary_kernels_fp64."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import test_heads_kernels_fp64 as H                                          # noqa: E402
import test_vm_kernels_fp64 as V                                             # noqa: E402
from test_secondary_kernels_fp64 import DEV, check_mlp, mlp_reference, report, sms  # noqa: E402

NWG = 3                     # warpgroups per CTA of app_mlp_wgmma_kernel
ROWS = 64                   # rows per tile


def _lengths():
    w = NWG * ROWS * sms()                             # rows of one wave: every warpgroup of every SM on one tile
    b = 5                                              # CTAs of the short lists below (capacity equal to the count)
    return {"1": 1, "wave-1": w - 1, "wave+1": w + 1, "3wave+17": 3 * w + 17,
            "last-cta-wg2-idle": ROWS * (NWG * b - 1) - 7,     # the last CTA's third warpgroup gets no tile
            "last-cta-wg2-last": ROWS * NWG * b - 30,          # ... gets the last (partial) tile
            "last-cta-wg0-alone": ROWS * (NWG * b - 2) + 1}    # ... only its first warpgroup has a tile, of one row


@pytest.fixture(scope="module")
def vm_field():
    from tensoir_b200 import _lib
    _lib.load()
    return V.Field(0)


@pytest.mark.parametrize("n_lights", [1, 16, 17, 0])
@pytest.mark.parametrize("cap", ["above", "equal"])
@pytest.mark.parametrize("length", ["1", "wave-1", "wave+1", "3wave+17", "last-cta-wg2-idle", "last-cta-wg2-last",
                                    "last-cta-wg0-alone"])
def test_list_mlp_schedule_and_light_table(vm_field, length, cap, n_lights):
    from tensoir_b200 import _lib
    lib = _lib.load()
    n = _lengths()[length]
    g = torch.Generator().manual_seed(n * 7 + len(cap) + n_lights)
    L = max(n_lights, 1)
    ll = torch.randn(L, H.K0, generator=g).to(DEV)
    basis = (torch.randn(H.NF, H.K0, generator=g) / 12).to(DEV)
    head = H.Head(g, 3, basis, ll if n_lights else None, 1 if n_lights else 0)
    assert head.mlp.n_lights == n_lights
    xn = (torch.rand(n, 3, generator=g) * 2.1 - 1.05).to(DEV)             # some taps just outside +-1
    fl = torch.cat([xn, torch.ones(n, 1, device=DEV)], 1).contiguous()
    it = torch.stack([torch.arange(n), torch.full((n,), 5)], 1).to(DEV, torch.int32).contiguous()
    rows = torch.cat([fl.view(torch.uint8), it.view(torch.uint8)], 1).reshape(-1)
    max_samples = {"above": max(2 * n, 4 * NWG * ROWS * sms()), "equal": n}[cap]
    buf = torch.zeros(max_samples * _lib.APP_SAMPLE_BYTES, dtype=torch.uint8, device=DEV)
    buf[:rows.numel()] = rows
    count = torch.tensor([n], dtype=torch.int32, device=DEV)
    vd = F.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV).contiguous()
    li = torch.randint(0, L, (n,), generator=g, dtype=torch.int32).to(DEV)
    prefill = (torch.rand(n, 3, generator=g) * 2 - 1).to(DEV)
    rgb = prefill.clone()
    _lib.check(lib.tir_app_mlp(C.byref(vm_field.struct), C.byref(head.mlp), _lib.dptr(buf, torch.uint8),
                               _lib.dptr(count, torch.int32), max_samples, _lib.dptr(vd), 0,
                               _lib.dptr(li, torch.int32) if n_lights else None, _lib.dptr(rgb),
                               _lib.stream_ptr()), "tir_app_mlp")
    torch.cuda.synchronize()
    W, B = head.w64()
    ref = mlp_reference([p.to(DEV).double() for p in vm_field.aplane], [p.to(DEV).double() for p in vm_field.aline],
                        V.GRID, W, B, basis.double(), ll.double() if n_lights else None, xn, vd, li,
                        torch.ones(n, device=DEV), torch.arange(n, device=DEV), n)
    stats = {}
    what = f"{n} rows ({length}), max_samples {max_samples}, {n_lights} light rows"
    check_mlp(rgb, prefill, ref, what, stats)
    report(what, stats)
