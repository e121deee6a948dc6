"""The reference's scripts/relight_importance.py entry point on the native relighting loop: the same seeds, script flags,
environment-map names, dataset (dataLoader.dataset_dict) and command line (opt.config_parser), calling
tensoir_b200.relighting.relight.  Run it with a TensoIR checkout on PYTHONPATH (for opt and dataLoader), like
tools/dropin_train_check.py:

    PYTHONPATH=<TensoIR checkout>:. python tools/relight_importance.py --config <config> --ckpt <ckpt> \\
        --hdrdir <dir of .hdr maps> --geo_buffer_path <out dir>

``--indirect_samples K`` adds one bounce of indirect light with K directions per surface hit (default 0: direct light
only, the reference's estimator), ``--indirect_light_samples S2`` sets the light samples per secondary hit (default 32)
and ``--save_indirect 1`` also writes the linear indirect-only images.  ``--sampling mis`` shades with multiple
importance sampling (GGX-lobe samples combined with environment-map samples, tensoir_b200/mis.py) instead of the
reference's texel-centre estimator, with ``--brdf_samples N`` of the 512 samples per surface hit drawn from the BRDF
(default 128).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from relight_lights import pop_option  # noqa: E402


def indirect_options(argv):
    """Remove the indirect-light flags from argv (opt.config_parser does not know them) -> dict of the args
    attributes relight() reads: --indirect_samples K (0: direct light only), --indirect_light_samples S2 (32),
    --save_indirect 1 (also write relighting_indirect/{light}.hdr)."""
    k = pop_option(argv, "--indirect_samples", int)
    s2 = pop_option(argv, "--indirect_light_samples", int)
    save = pop_option(argv, "--save_indirect", int)
    return dict(indirect_samples=k or 0, indirect_light_samples=32 if s2 is None else s2,
                save_indirect=bool(save))


def sampling_options(argv):
    """Remove the estimator flags from argv -> dict of the args attributes relight() reads: --sampling light|mis
    (light), --brdf_samples N (128)."""
    sampling = pop_option(argv, "--sampling", str)
    n_brdf = pop_option(argv, "--brdf_samples", int)
    return dict(sampling=sampling or "light", brdf_samples=128 if n_brdf is None else n_brdf)


if __name__ == "__main__":
    indirect = indirect_options(sys.argv)
    indirect.update(sampling_options(sys.argv))

    from dataLoader import dataset_dict
    from opt import config_parser

    from tensoir_b200.relighting import relight

    args = config_parser()
    print(args)
    print("*" * 80)
    print('The result will be saved in {}'.format(os.path.abspath(args.geo_buffer_path)))

    torch.set_default_dtype(torch.float32)
    torch.manual_seed(20211202)
    torch.cuda.manual_seed_all(20211202)
    np.random.seed(20211202)

    # the flags the reference script sets on args (they are not defined in opt.py)
    args.if_save_rgb = False
    args.if_save_depth = False
    args.if_save_acc = True
    args.if_save_rgb_video = False
    args.if_save_relight_rgb = True
    args.if_save_albedo = True
    args.if_save_albedo_gamma_corrected = True
    args.acc_mask_threshold = 0.5
    args.if_render_normal = True
    args.vis_equation = 'nerv'
    args.render_video = True
    for k, v in indirect.items():
        setattr(args, k, v)

    dataset = dataset_dict[args.dataset_name]
    # names of the environment maps used for relighting
    light_name_list = ['bridge', 'city', 'fireplace', 'forest', 'night']
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', random_test=False,
                           downsample=args.downsample_test, light_names=light_name_list,
                           light_rotation=args.light_rotation)
    relight(test_dataset, args)
