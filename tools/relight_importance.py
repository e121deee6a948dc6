"""The reference's scripts/relight_importance.py entry point on the native relighting loop: the same seeds, script flags,
environment-map names, dataset (dataLoader.dataset_dict) and command line (opt.config_parser), calling
tensoir_b200.relighting.relight.  Run it with a TensoIR checkout on PYTHONPATH (for opt and dataLoader), like
tools/dropin_train_check.py:

    PYTHONPATH=<TensoIR checkout>:. python tools/relight_importance.py --config <config> --ckpt <ckpt> \\
        --hdrdir <dir of .hdr maps> --geo_buffer_path <out dir>
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

if __name__ == "__main__":
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

    dataset = dataset_dict[args.dataset_name]
    # names of the environment maps used for relighting
    light_name_list = ['bridge', 'city', 'fireplace', 'forest', 'night']
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', random_test=False,
                           downsample=args.downsample_test, light_names=light_name_list,
                           light_rotation=args.light_rotation)
    relight(test_dataset, args)
