"""The reference's train_tensoIR.py entry point on the native trainer: the same command line (opt.config_parser),
dataset (dataLoader.dataset_dict), seeds and log folder, calling tensoir_b200.train.reconstruction.  Run it with a
TensoIR checkout on PYTHONPATH (for opt and dataLoader only), like tools/relight_importance.py:

    PYTHONPATH=<TensoIR checkout>:. python tools/train_tensoIR.py --config configs/single_light/armadillo.txt
"""
import datetime
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

if __name__ == "__main__":
    from dataLoader import dataset_dict
    from opt import config_parser

    import __graft_entry__ as g
    g.build()
    from tensoir_b200 import train

    args = config_parser()
    print(args)
    train.check_supported(args)

    torch.set_default_dtype(torch.float32)
    torch.manual_seed(20211202)
    torch.cuda.manual_seed_all(20211202)
    np.random.seed(20211202)
    random.seed(20211202)

    dataset = dataset_dict[args.dataset_name]
    train_dataset = dataset(args.datadir, args.hdrdir, split='train', downsample=args.downsample_train,
                            light_name=args.light_name, light_rotation=args.light_rotation)
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', downsample=args.downsample_test,
                           light_name=args.light_name, light_rotation=args.light_rotation)
    if args.add_timestamp:
        logfolder = f'{args.basedir}/{args.expname}{datetime.datetime.now().strftime("-%Y%m%d-%H%M%S")}'
    else:
        logfolder = f'{args.basedir}/{args.expname}'
    res = train.reconstruction(args, train_dataset, test_dataset, logfolder)
    print(f"steps redone after a list overflow: {res['redone']}, re-captures: {res['recaptures']}")
