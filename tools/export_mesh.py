"""The reference's scripts/export_mesh.py entry point on the native mesh export: the same seeds and command line
(opt.config_parser), the checkpoint loaded with tensoir_b200.relighting._load_model, and the mesh written to
``{ckpt[:-3]}.ply`` by tensoir_b200.mesh.export_mesh (level 0.005).  Run it with a TensoIR checkout on PYTHONPATH (for
opt), like tools/relight_importance.py:

    PYTHONPATH=<TensoIR checkout>:. python tools/export_mesh.py --config <config> --ckpt <ckpt>
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)


@torch.no_grad()
def main(args):
    """export_mesh of scripts/export_mesh.py on ``args.ckpt``, on ``cuda:{args.local_rank}`` like the reference (device
    0 when args has no local_rank); returns the path written (None without a checkpoint)."""
    from tensoir_b200.mesh import export_mesh
    from tensoir_b200.relighting import _load_model
    tensoIR = _load_model(args, torch.device(f"cuda:{getattr(args, 'local_rank', 0)}"))   # the reference's device
    if tensoIR is None:
        return None
    path = f'{args.ckpt[:-3]}.ply'
    export_mesh(tensoIR, path, level=0.005)
    return path


if __name__ == "__main__":
    from opt import config_parser

    args = config_parser()
    print(args)
    torch.set_default_dtype(torch.float32)
    torch.manual_seed(20211202)
    torch.cuda.manual_seed_all(20211202)
    np.random.seed(20211202)
    main(args)
