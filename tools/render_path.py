"""Render a relit camera-path video of a checkpoint with the command line of tools/relight_importance.py
(opt.config_parser, the same seed and dataset), calling tensoir_b200.camera_path.render_path: every frame is rendered
once per environment map of --hdrdir (or per learned light with --light learned, or per setup of an analytic light rig
with --rig), from cameras that need not be dataset views, with the maps or lights rotated per frame and, with --ground,
a ground plane that catches the object's shadow.  Run it with a TensoIR checkout on PYTHONPATH (for opt and
dataLoader):

    PYTHONPATH=<TensoIR checkout>:. python tools/render_path.py --config <config> --ckpt <ckpt> \\
        --hdrdir <dir of .hdr maps> --geo_buffer_path <dir> --out <dir> --path orbit --frames 120 \\
        --env_rotation 0:360 --ground

Options (besides relight_importance.py's):
  --path orbit|test|<poses.json>  orbit: one turn around the aabb centre at the first test camera's radius and
                                  elevation, starting at its azimuth; test: the dataset's test cameras; a JSON list of
                                  4x4 OpenCV camera-to-world matrices (default orbit)
  --frames N                      frames of the orbit (default 120; orbit only)
  --env_rotation a0:a1            map rotation about +z in degrees, linear over the frames (default 0:0)
  --ground [z]                    a shadow-catching ground plane at height z (default: the bottom of the model's
                                  occupied box)
  --light learned                 the model's own learned lights instead of --hdrdir
  --rig <rig.json>                the setups of an analytic light rig (README, "Analytic lights") instead of maps,
                                  each over its background colour; --env_rotation turns the lights about +z as it
                                  turns a map; not with --light
  --shadow_far <d>                with --rig: how far the object's shadow rays are marched (default: the aabb diagonal)
  --out <dir>                     {out}/{map or setup}/with_bg/{frame:04d}.png, without_bg/..., {out}/{map or setup}.mp4

--path orbit --env_rotation 0:360 turns the camera and the map (or the rig) together, so the background and the
lighting stand still while the object turns: a turntable.
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

USAGE = ("usage: render_path.py <relight_importance.py options> --out <dir> [--path orbit|test|<poses.json>] "
         "[--frames N (orbit only)] [--env_rotation a0:a1] [--ground [z]] "
         "[--light learned | --rig <rig.json> [--shadow_far d]]")


def path_options(argv):
    """Remove this tool's options from argv (opt.config_parser does not know them) -> dict(path=(kind, spec),
    frames, rotation=(a0, a1), ground=None | True | z, light=None | 'learned', out).  SystemExit with the usage for a
    bad value or an unknown combination."""
    from tensoir_b200.camera_path import parse_path, parse_rotation
    try:
        path = parse_path(pop_option(argv, "--path") or "orbit")
        frames = pop_option(argv, "--frames", int)
        rotation = parse_rotation(pop_option(argv, "--env_rotation") or "0:0")
    except ValueError as e:
        raise SystemExit(f"{e}\n{USAGE}")
    light = pop_option(argv, "--light")
    out = pop_option(argv, "--out")
    ground = None
    if "--ground" in argv:
        i = argv.index("--ground")
        ground = True
        if i + 1 < len(argv):
            try:
                ground = float(argv[i + 1])
                del argv[i + 1]
            except ValueError:
                pass
        del argv[i]
        if ground is not True and not np.isfinite(ground):
            raise SystemExit(f"--ground: the height must be finite\n{USAGE}")
    if frames is not None and path[0] != "orbit":
        raise SystemExit(f"--frames sets the length of an orbit; a {path[0]} path has its own frames\n{USAGE}")
    if frames is not None and frames < 1:
        raise SystemExit(f"--frames must be at least 1\n{USAGE}")
    if light not in (None, "learned"):
        raise SystemExit(f"--light: only 'learned' is known, got {light!r}\n{USAGE}")
    if not out:
        raise SystemExit(f"--out is required\n{USAGE}")
    return dict(path=path, frames=120 if frames is None else frames, rotation=rotation, ground=ground, light=light,
                out=out)


def rig_options(argv):
    """Remove --rig and --shadow_far from argv -> dict(rig=None | path, shadow_far=None | d).  Run before
    path_options, which removes --light.  SystemExit with the usage for a rig file that does not exist, --rig with
    --light, --shadow_far without --rig, or a shadow_far that is not a finite number above the shadow march's near."""
    from tensoir_b200.lighting import SHADOW_NEAR
    rig = pop_option(argv, "--rig")
    far = pop_option(argv, "--shadow_far", float)
    if rig is not None and not os.path.isfile(rig):
        raise SystemExit(f"--rig: no such file {rig!r}\n{USAGE}")
    if rig is not None and "--light" in argv:
        raise SystemExit(f"--rig lights the frames itself: it does not take --light\n{USAGE}")
    if far is not None and rig is None:
        raise SystemExit(f"--shadow_far sets the march of a rig's shadow rays: it needs --rig\n{USAGE}")
    if far is not None and not (np.isfinite(far) and far > SHADOW_NEAR):
        raise SystemExit(f"--shadow_far must be a finite distance above {SHADOW_NEAR}, got {far}\n{USAGE}")
    return dict(rig=rig, shadow_far=far)


def path_poses(opts, dataset, tensoIR):
    """The cameras of opts['path'] -> float32 [F,4,4]."""
    from tensoir_b200 import camera_path as P
    kind, spec = opts["path"]
    if kind == "file":
        return P.load_poses(spec)
    test = P.dataset_poses(dataset)
    if kind == "test":
        return test
    centre = tensoIR.aabb.detach().double().mean(0).cpu().numpy()
    r, el, az = P.orbit_of(test[0], centre)
    return P.orbit_poses(opts["frames"], r, el, centre, start_deg=az)


if __name__ == "__main__":
    rig_opts = rig_options(sys.argv)
    opts = path_options(sys.argv)
    if not torch.cuda.is_available():
        raise SystemExit("render_path.py needs a CUDA device: tensoir_b200 has no CPU fallback")

    from dataLoader import dataset_dict
    from opt import config_parser

    from tensoir_b200 import camera_path as P
    from tensoir_b200 import relighting as R
    from tensoir_b200.lighting import SEED

    args = config_parser()
    print(args)
    print("*" * 80)
    print('The frames will be saved in {}'.format(os.path.abspath(opts["out"])))

    torch.set_default_dtype(torch.float32)
    torch.manual_seed(SEED)
    torch.cuda.manual_seed_all(SEED)
    np.random.seed(SEED)

    args.acc_mask_threshold = 0.5
    args.vis_equation = 'nerv'
    args.render_video = True
    args.seed = SEED
    args.out = opts["out"]
    args.light = opts["light"]
    args.shadow_far = rig_opts["shadow_far"]

    dataset = dataset_dict[args.dataset_name]
    # the relighting test set needs the names of ground-truth images to load; its cameras, rays and albedo are used
    light_name_list = ['bridge', 'city', 'fireplace', 'forest', 'night']
    test_dataset = dataset(args.datadir, args.hdrdir, split='test', random_test=False,
                           downsample=args.downsample_test, light_names=light_name_list,
                           light_rotation=args.light_rotation)
    model, _ = R._model(args, None)
    if model is None:
        raise SystemExit(1)
    poses = path_poses(opts, test_dataset, model)
    angles = P.frame_angles(poses.shape[0], opts["rotation"])
    print(f"{poses.shape[0]} frames, {'rig' if rig_opts['rig'] else 'map'} rotation {opts['rotation'][0]} -> "
          f"{opts['rotation'][1]} degrees, ground {'off' if opts['ground'] is None else opts['ground']}")
    P.render_path(test_dataset, args, poses, angles, tensoIR=model, ground_z=opts["ground"], rig=rig_opts["rig"])
