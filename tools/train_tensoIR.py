"""The reference's train_tensoIR.py entry point on the native trainer: the same command line (opt.config_parser),
datasets (dataLoader.dataset_dict), seeds and log folders, calling tensoir_b200.train.main.  Run it with a TensoIR
checkout on PYTHONPATH (for opt and dataLoader only), like tools/relight_importance.py:

    PYTHONPATH=<TensoIR checkout>:. python tools/train_tensoIR.py --config configs/single_light/armadillo.txt

The reference's train_tensoIR_rotated_multi_lights.py is the same loop with the same datasets (it differs only in
comments), so this script also runs configs/multi_light_rotated/*.txt.

``--render_only 1 --render_test 1 --ckpt <model.th>`` renders the test views of a checkpoint into
``{basedir}/test_{expname}-{timestamp}/imgs_test_all/`` instead of training; ``--export_mesh 1 --ckpt <model.th>`` first
writes the checkpoint's mesh to ``{ckpt[:-3]}.ply``.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

VARIANT = "full"


def datasets(dataset, args):
    """The train and test sets of reconstruction (train_tensoIR.py:112-128)."""
    train_dataset = dataset(args.datadir, args.hdrdir, split='train', downsample=args.downsample_train,
                            light_name=args.light_name, light_rotation=args.light_rotation)
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', downsample=args.downsample_test,
                           light_name=args.light_name, light_rotation=args.light_rotation)
    return train_dataset, test_dataset


def render_dataset(dataset, args):
    """The test set of render_test (train_tensoIR.py:67-69)."""
    return dataset(args.datadir, args.hdrdir, light_rotation=args.light_rotation, split='test',
                   downsample=args.downsample_train, is_stack=False, sub=args.test_number)


def main(args, dataset, device=None):
    from tensoir_b200 import train
    return train.main(args, VARIANT, lambda: datasets(dataset, args), lambda: render_dataset(dataset, args),
                      device=device)


if __name__ == "__main__":
    from dataLoader import dataset_dict
    from opt import config_parser

    import __graft_entry__ as g
    g.build()

    args = config_parser()
    print(args)
    main(args, dataset_dict[args.dataset_name])
