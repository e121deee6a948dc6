"""Estimate the lighting of photographs of a reconstructed object: fit one environment map per light of the test set to
its photographs, with the checkpoint's geometry and materials held fixed (tensoir_b200.light_fit.fit_lights).  The
command line is tools/relight_importance.py's (opt.config_parser; --hdrdir is only needed by datasets that load it),
plus

    --fit_views <spec>       views to fit on: 'i,j,...', 'a:b:step' or 'none'        (default 0::10)
    --eval_views <spec>      views relight() renders under the fitted maps             (default 5::10; 'none' skips)
    --fit_res HxW            resolution of the fitted maps, W = 2H, 4 <= H <= 32       (default 16x32)
    --pixels_per_view N      masked pixels drawn per fit view                          (default 65536)
    --smooth s, --ridge r    regularisers relative to trace(G) / K                     (defaults in light_fit)
    --out <dir>              where {light}.hdr and fit_report.json go                   (required)

relight()'s files for the evaluation views go to --geo_buffer_path.  Run it with a TensoIR checkout on PYTHONPATH (for
opt and dataLoader):

    PYTHONPATH=<TensoIR checkout>:. python tools/fit_lights.py --config <config> --ckpt <ckpt> \\
        --geo_buffer_path <eval dir> --out <fit dir> [--fit_views 0::10] [--fit_res 16x32]
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

# names of the relighting test set's photographs (relight_importance.py's light_name_list)
LIGHT_NAMES = ['bridge', 'city', 'fireplace', 'forest', 'night']
OPTIONS = {"--fit_views": str, "--eval_views": str, "--fit_res": str, "--pixels_per_view": int, "--smooth": float,
           "--ridge": float, "--out": str}


def parse_fit_args(argv):
    """Remove this tool's options from ``argv`` (a list, edited in place) and check them -> dict of the given ones
    (fit_res as (H, W)).  Raises SystemExit with a message for a missing --out or a malformed value."""
    from tensoir_b200 import light_fit as LF
    got = {}
    for name, cast in OPTIONS.items():
        if name not in argv:
            continue
        i = argv.index(name)
        if i + 1 >= len(argv):
            raise SystemExit(f"{name} needs a value")
        try:
            got[name[2:]] = cast(argv[i + 1])
        except ValueError:
            raise SystemExit(f"{name}: bad value {argv[i + 1]!r}") from None
        del argv[i:i + 2]
    if "out" not in got:
        raise SystemExit("--out <dir> is required")
    try:
        if "fit_res" in got:
            got["fit_res"] = LF.parse_res(got["fit_res"])
        for k in ("fit_views", "eval_views"):          # syntax only; the indices are checked against the dataset
            if k in got:
                LF.parse_views(got[k], 1 << 30)
    except ValueError as e:
        raise SystemExit(str(e)) from None
    if got.get("pixels_per_view", 1) < 1:
        raise SystemExit("--pixels_per_view must be at least 1")
    if got.get("smooth", 0.0) < 0 or got.get("ridge", 0.0) < 0:
        raise SystemExit("--smooth and --ridge must be >= 0")
    return got


def build_dataset(args):
    """The test split of the dataset the config names, with the light names it takes: ``light_name_list`` for the
    general multi-light dataset, relight_importance.py's five maps otherwise."""
    from dataLoader import dataset_dict
    dataset = dataset_dict[args.dataset_name]
    if getattr(args, "light_name_list", None) and "general" in args.dataset_name:
        ds = dataset(args.datadir, args.hdrdir, split='test', downsample=args.downsample_test,
                     light_name=args.light_name, light_rotation=args.light_rotation,
                     light_name_list=args.light_name_list)
        ds.light_names = list(args.light_name_list)      # the order of its rgbs
        return ds
    return dataset(args.datadir, args.hdrdir, split='test', random_test=False, downsample=args.downsample_test,
                   light_names=LIGHT_NAMES, light_rotation=args.light_rotation)


if __name__ == "__main__":
    from tensoir_b200.light_fit import SEED, fit_lights

    fit = parse_fit_args(sys.argv)
    if not torch.cuda.is_available():
        raise SystemExit("fit_lights.py needs a CUDA device: tensoir_b200 has no CPU fallback")
    from opt import config_parser

    args = config_parser()
    print(args)
    for k, v in fit.items():
        setattr(args, k, v)
    print('The fitted maps will be saved in {}'.format(os.path.abspath(args.out)))
    torch.set_default_dtype(torch.float32)
    torch.manual_seed(SEED)
    torch.cuda.manual_seed_all(SEED)
    np.random.seed(SEED)
    args.acc_mask_threshold = 0.5
    args.vis_equation = 'nerv'
    args.seed = SEED
    fit_lights(build_dataset(args), args)
