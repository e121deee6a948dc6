"""Relight a checkpoint under analytic lights with the command line of tools/relight_importance.py (opt.config_parser,
the same seed and dataset; --hdrdir is not needed), calling tensoir_b200.lighting.relight_rig: every view is rendered
once per setup of ``--rig <json>`` (README, "Analytic lights"), or once per light of a one-light-at-a-time sweep of
``--olat N`` hard directional lights on a Fibonacci sphere.  ``--shadow_far <d>`` sets how far shadow rays are marched
(default: the aabb diagonal); ``--save_linear 1`` also writes the un-toned images as .hdr.  Run it with a TensoIR
checkout on PYTHONPATH (for opt and dataLoader):

    PYTHONPATH=<TensoIR checkout>:. python tools/relight_lights.py --config <config> --ckpt <ckpt> \\
        --geo_buffer_path <out dir> --rig rig.json
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)


def pop_option(argv, name, cast=str):
    """Remove ``name <value>`` from argv (opt.config_parser does not know it) -> cast(value) or None."""
    if name not in argv:
        return None
    i = argv.index(name)
    if i + 1 >= len(argv):
        raise SystemExit(f"{name} needs a value")
    try:
        value = cast(argv[i + 1])
    except ValueError:
        raise SystemExit(f"{name}: bad value {argv[i + 1]!r}")
    del argv[i:i + 2]
    return value


if __name__ == "__main__":
    from tensoir_b200.lighting import SEED, load_rig, olat_rig, relight_rig

    rig_path, olat = pop_option(sys.argv, "--rig"), pop_option(sys.argv, "--olat", int)
    shadow_far = pop_option(sys.argv, "--shadow_far", float)
    save_linear = pop_option(sys.argv, "--save_linear", int)
    if (rig_path is None) == (olat is None):
        raise SystemExit("usage: relight_lights.py <relight_importance.py options> (--rig <json> | --olat <N>) "
                         "[--shadow_far <d>] [--save_linear 1]")
    rig = load_rig(rig_path) if olat is None else olat_rig(olat)
    print(f"{len(rig)} setup(s): " + ", ".join(f"{k} ({len(v.lights)} light(s))" for k, v in rig.items()))
    if not torch.cuda.is_available():
        raise SystemExit("relight_lights.py needs a CUDA device: tensoir_b200 has no CPU fallback")

    from dataLoader import dataset_dict
    from opt import config_parser

    args = config_parser()
    print(args)
    print("*" * 80)
    print('The result will be saved in {}'.format(os.path.abspath(args.geo_buffer_path)))

    torch.set_default_dtype(torch.float32)
    torch.manual_seed(SEED)
    torch.cuda.manual_seed_all(SEED)
    np.random.seed(SEED)

    args.acc_mask_threshold = 0.5
    args.vis_equation = 'nerv'
    args.render_video = True
    args.seed = SEED
    args.shadow_far = shadow_far
    args.save_linear = bool(save_linear)

    dataset = dataset_dict[args.dataset_name]
    # the relighting test set needs the names of ground-truth images to load; only its rays and albedo are used
    light_name_list = ['bridge', 'city', 'fireplace', 'forest', 'night']
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', random_test=False,
                           downsample=args.downsample_test, light_names=light_name_list,
                           light_rotation=args.light_rotation)
    relight_rig(test_dataset, args, rig)
