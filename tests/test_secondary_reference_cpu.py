"""The march reference of test_secondary_kernels_fp64.py, run in float32 on the CPU, reproduces the oracle's
compute_transmittance / compute_radiance on the rotated golden fixture bit for bit: the valid samples (aabb and
alpha-mask test), the weights, the visibility and the appearance mask.  The float64 checks of the secondary kernels
restate the march; this ties the restatement to the reference before any GPU run."""
import types

import torch

from helpers import oracle_field
from oracle import tensoir_oracle as O


def test_march_reference_reproduces_the_oracle(golden_rotated):
    from test_secondary_kernels_fp64 import reference_march
    fx = golden_rotated
    f = oracle_field(fx)
    surf, dirs = fx["surf"], fx["dirs"]
    n, N = surf.shape[0], 96
    sc = types.SimpleNamespace(o32=f, shift=f.density_shift, scale=f.distance_scale)
    t = torch.linspace(0., 1., N)
    z = (0.05 * (1. - t) + 1.5 * t)[None].expand(n, N)
    r = reference_march(sc, surf, dirs, z, dtype=torch.float32, bounds=False)
    nerv, _ = O.compute_transmittance(f, surf, dirs, N, 0.05, 1.5)
    _, _, _, valid, app_mask, weight = O.compute_radiance(f, surf, dirs, fx["li2"], N, 0.05, 1.5, return_aux=True)
    assert torch.equal(r["valid"], valid)
    assert bool(valid.any()) and not bool(valid.all())
    assert torch.equal(r["w"], weight)
    assert torch.equal(r["T_last"], nerv)
    assert torch.equal(r["w"] > f.weight_thres, app_mask)
    assert bool(app_mask.any())
