"""The head kernels' two warp groups per CTA against float64, at list lengths that leave a group without a tile.

app_mlp_kernel and heads_dgrad_kernel run one CTA per SM (up to the list's length) and split each CTA into two warp
groups, each with its own 32-row tile; group g of CTA c takes tiles 2c + g, 2c + g + 2 * CTAs, ...  A one-head launch
(the radiance-only step) uses every SM, so an odd number of 32-row tiles leaves the second group of the last CTA
without its last tile, and longer lists give each group one to three tiles.  The stage checks of
test_heads_kernels_fp64.py run unchanged at those lengths."""
import pytest
import torch

from test_heads_kernels_fp64 import field  # noqa: F401  (module fixture)
from test_heads_kernels_fp64 import test_radiance_head_stages as radiance_head_stages


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (light_mode, lights, act, 32-row tiles as (per SM, extra), extra rows): odd tile counts with one to three tiles per
# CTA (one group short by a tile), a count below one tile per CTA, and partial last tiles
CASES = [(1, 3, 0, (2, -1), -5), (2, 3, 1, (2, 1), 0), (0, 0, 1, (4, -1), 17), (1, 9, 1, (6, -1), -31),
         (2, 13, 0, (0, 67), 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,n_lights,act,tiles,extra", CASES)
def test_group_tiles_match_float64(field, mode, n_lights, act, tiles, extra):  # noqa: F811
    per_sm, more = tiles
    n32 = per_sm * _sms() + more
    assert n32 % 2 == 1
    radiance_head_stages(field, mode, n_lights, act, 32 * n32 + extra if extra <= 0 else 32 * (n32 - 1) + extra)
