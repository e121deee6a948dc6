"""heads_wgrad_kernel's row slices against float64 at list lengths set by the GPU's SM count.

The weight-gradient grid is one CTA per SM, shared by the heads of a launch and split over three roles (gW1, gW0 and
the small gW2 / gb2 / g basis_mat role), each cutting the list into 64-row-aligned slices.  A one-head launch (the
radiance-only step) spreads the roles over every SM, so a list of about as many tiles as SMs leaves some slices empty,
one tile long or partial, and a longer list gives every slice several tiles and thus exercises the prefetch of the next
tile.  The stage checks of test_heads_kernels_fp64.py run unchanged at those lengths."""
import pytest
import torch

from test_heads_kernels_fp64 import field  # noqa: F401  (module fixture)
from test_heads_kernels_fp64 import test_radiance_head_stages as radiance_head_stages


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (light_mode, lights, act, rows as (tiles per SM, extra rows)): rows below, at and above one tile per SM, and past
# two tiles per slice of every role, with partial last tiles
CASES = [(1, 3, 0, (1, -37)), (2, 3, 1, (1, 0)), (0, 0, 1, (1, 1)), (1, 9, 1, (3, 37)), (2, 13, 0, (3, -1))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,n_lights,act,rows", CASES)
def test_wgrad_slices_match_float64(field, mode, n_lights, act, rows):  # noqa: F811
    per_sm, extra = rows
    radiance_head_stages(field, mode, n_lights, act, per_sm * 64 * _sms() + extra)
