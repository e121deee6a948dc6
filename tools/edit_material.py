"""Material editing of a checkpoint with the command line of tools/relight_importance.py (opt.config_parser, the same
seeds, script flags, environment-map names and dataset), calling tensoir_b200.editing.relight_edited: every view is
relit under each map once with the learned materials (variant ``original``) and once per variant of ``--edits``, all
variants sharing one visibility march per chunk.  ``--edits <json>`` holds {variant: [rule, ...]} with the fields of
tensoir_b200.editing.MaterialEdit (README, "Material editing").  Run it with a TensoIR checkout on PYTHONPATH (for opt
and dataLoader):

    PYTHONPATH=<TensoIR checkout>:. python tools/edit_material.py --config <config> --ckpt <ckpt> \\
        --hdrdir <dir of .hdr maps> --geo_buffer_path <out dir> --edits <json>
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)
TOOLS = os.path.join(ROOT, "tools")
if TOOLS not in sys.path:
    sys.path.append(TOOLS)

if __name__ == "__main__":
    from export_asset import pop_edits

    edits_path = pop_edits(sys.argv)
    if edits_path is None:
        raise SystemExit("usage: edit_material.py <relight_importance.py options> --edits <json>")

    from dataLoader import dataset_dict
    from opt import config_parser

    from tensoir_b200.editing import load_edits, relight_edited

    variants = load_edits(edits_path)
    args = config_parser()
    print(args)
    print("*" * 80)
    print('The result will be saved in {}'.format(os.path.abspath(args.geo_buffer_path)))

    torch.set_default_dtype(torch.float32)
    torch.manual_seed(20211202)
    torch.cuda.manual_seed_all(20211202)
    np.random.seed(20211202)

    # the flags relight_importance.py sets on args (they are not defined in opt.py)
    args.acc_mask_threshold = 0.5
    args.vis_equation = 'nerv'
    args.render_video = True

    dataset = dataset_dict[args.dataset_name]
    light_name_list = ['bridge', 'city', 'fireplace', 'forest', 'night']
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', random_test=False,
                           downsample=args.downsample_test, light_names=light_name_list,
                           light_rotation=args.light_rotation)
    relight_edited(test_dataset, args, variants)
