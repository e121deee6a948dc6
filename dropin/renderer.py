"""Shadow of the reference's renderer.py for unchanged train scripts: the hot-path boundary, compute_rescale_ratio and
the three evaluation loops all come from tensoir_b200 (same signatures, return values and written files)."""
import os  # noqa: F401
import random  # noqa: F401  (the train scripts take np / random / os / tqdm / torch from `from renderer import *`)

import numpy as np  # noqa: F401
import torch  # noqa: F401
from tqdm.auto import tqdm  # noqa: F401

try:                                   # renderer.py:5 `from utils import *`: the reference's own helpers (N_to_reso,
    from utils import *  # noqa: F401,F403   cal_n_samples, TVLoss, ...), resolved from the reference tree on sys.path
except ImportError:
    pass
try:
    import imageio  # noqa: F401
    import torchvision.utils as vutils  # noqa: F401
except ImportError:
    pass

from tensoir_b200.renderer import Renderer_TensoIR_train, OctreeRender_trilinear_fast  # noqa: F401
from tensoir_b200.relight_utils import render_with_BRDF  # noqa: F401
from tensoir_b200.evaluation import (compute_rescale_ratio, evaluation_iter_TensoIR,  # noqa: F401
                                     evaluation_iter_TensoIR_simple, evaluation_iter_TensoIR_general_multi_lights)

