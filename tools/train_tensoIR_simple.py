"""The reference's train_tensoIR_simple.py entry point on the native trainer, for scenes without ground-truth albedo
or normals such as NeRF-synthetic (configs/single_light/blender.txt): the same command line (opt.config_parser),
datasets (dataLoader.dataset_dict), seeds and log folders, calling tensoir_b200.train.main with the ``simple`` variant.
Run it with a TensoIR checkout on PYTHONPATH (for opt and dataLoader only):

    PYTHONPATH=<TensoIR checkout>:. python tools/train_tensoIR_simple.py --config configs/single_light/blender.txt

``--render_only 1 --render_test 1 --ckpt <model.th>`` renders the test views of a checkpoint into
``{basedir}/test_{expname}-{timestamp}/imgs_test_all/``; ``--export_mesh 1 --ckpt <model.th>`` first writes the
checkpoint's mesh to ``{ckpt[:-3]}.ply``.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)

VARIANT = "simple"


def datasets(dataset, args):
    """The train and test sets of reconstruction (train_tensoIR_simple.py:113-131): no hdrdir, the scene_bbox option,
    a stacked test set."""
    train_dataset = dataset(args.datadir, split='train', downsample=args.downsample_train, light_name=args.light_name,
                            light_rotation=args.light_rotation, scene_bbox=args.scene_bbox)
    test_dataset = dataset(args.datadir, split='test', downsample=args.downsample_test, light_name=args.light_name,
                           light_rotation=args.light_rotation, scene_bbox=args.scene_bbox, is_stack=True)
    return train_dataset, test_dataset


def render_dataset(dataset, args):
    """The test set of render_test (train_tensoIR_simple.py:66-69)."""
    return dataset(args.datadir, split='test', downsample=args.downsample_train, is_stack=True, sub=args.test_number)


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
