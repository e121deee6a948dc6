"""The reference's train_tensoIR_general_multi_lights.py entry point on the native trainer: one SG environment per
named light (``light_name_list``), the same command line (opt.config_parser), datasets (dataLoader.dataset_dict), seeds
and log folders, calling tensoir_b200.train.main with the ``general`` variant.  Run it with a TensoIR checkout on
PYTHONPATH (for opt and dataLoader only):

    PYTHONPATH=<TensoIR checkout>:. python tools/train_tensoIR_general_multi_lights.py \
        --config configs/multi_light_general/lego.txt

``--render_only 1 --render_test 1 --ckpt <model.th>`` renders the test views once per light into
``{basedir}/test_{expname}-{timestamp}/imgs_test_all/{light_name}/``; ``--export_mesh 1 --ckpt <model.th>`` first writes
the checkpoint's mesh to ``{ckpt[:-3]}.ply``.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

VARIANT = "general"


def datasets(dataset, args):
    """The train and test sets of reconstruction (train_tensoIR_general_multi_lights.py:137-155)."""
    train_dataset = dataset(args.datadir, args.hdrdir, split='train', downsample=args.downsample_train,
                            light_name=args.light_name, light_rotation=args.light_rotation,
                            light_name_list=args.light_name_list)
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', downsample=args.downsample_test,
                           light_name=args.light_name, light_rotation=args.light_rotation,
                           light_name_list=args.light_name_list)
    return train_dataset, test_dataset


def render_dataset(dataset, args):
    """The test set of render_test (train_tensoIR_general_multi_lights.py:73-75): no light_rotation."""
    return dataset(args.datadir, args.hdrdir, split='test', downsample=args.downsample_train, is_stack=False,
                   sub=args.test_number)


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
