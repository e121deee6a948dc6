"""Export a relightable asset of a checkpoint with the command line of tools/export_mesh.py (opt.config_parser, the
same seeds, the checkpoint loaded with tensoir_b200.relighting._load_model): ``{ckpt[:-3]}_asset.ply`` holds the mesh
of tools/export_mesh.py with per-vertex albedo, roughness and predicted normal, and ``{ckpt[:-3]}_asset_envmap_{k}.hdr``
the radiance of light k (tensoir_b200.mesh.export_asset, level 0.005).  A general multi-light checkpoint
(``light_name_list``) gets no .hdr files: its SG lights (lgtSGs_list) are not in the state_dict, so the checkpoint does
not hold them and the loaded model's lights are their random initialisation; the tool says so.  With
``--edits <json>`` (a list of material rules, the fields of tensoir_b200.editing.MaterialEdit, without fresnel ops)
the albedo, colour and roughness columns hold the edited materials.  With ``--glb`` the tool writes
``{ckpt[:-3]}_asset.glb`` instead of the PLY: the same surface as a textured glTF 2.0 mesh, its materials baked into a
``--texture_size`` (default 4096) atlas (tensoir_b200.gltf.export_asset_glb); ``--edits`` applies to it as well.  Run
it with a TensoIR checkout on PYTHONPATH (for opt):

    PYTHONPATH=<TensoIR checkout>:. python tools/export_asset.py --config <config> --ckpt <ckpt> [--edits <json>]
                                                                  [--glb [--texture_size N]]
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.append(ROOT)


def pop_edits(argv):
    """Remove ``--edits <json>`` from argv (opt.config_parser does not know it) -> the JSON path or None."""
    if "--edits" not in argv:
        return None
    i = argv.index("--edits")
    if i + 1 >= len(argv):
        raise SystemExit("--edits needs a JSON file")
    path = argv[i + 1]
    del argv[i:i + 2]
    return path


def pop_glb(argv):
    """Remove ``--glb`` and ``--texture_size <N>`` from argv -> (glb, texture size)."""
    glb = "--glb" in argv
    if glb:
        argv.remove("--glb")
    size = 4096
    if "--texture_size" in argv:
        i = argv.index("--texture_size")
        if i + 1 >= len(argv) or not argv[i + 1].isdigit():
            raise SystemExit("--texture_size needs a power of two in [256, 8192]")
        size = int(argv[i + 1])
        del argv[i:i + 2]
        if not glb:
            raise SystemExit("--texture_size applies to --glb")
    return glb, size


def load_rules(path):
    """The rule list of an --edits JSON file ([rule, ...]) as MaterialEdit, validated as load_edits validates a
    variant."""
    import json
    from tensoir_b200.editing import load_edits
    with open(path) as f:
        return load_edits({"asset": json.load(f)})["asset"]


@torch.no_grad()
def main(args, edits=None, glb=False, texture_size=4096):
    """export_asset (export_asset_glb with ``glb``, on a texture_size^2 atlas) on ``args.ckpt`` with the material rules
    ``edits`` (None: unedited), on ``cuda:{args.local_rank}`` (device 0 when args has no local_rank); returns the path
    written (None without a checkpoint)."""
    from tensoir_b200.gltf import export_asset_glb
    from tensoir_b200.mesh import export_asset
    from tensoir_b200.relighting import _load_model
    tensoIR = _load_model(args, torch.device(f"cuda:{getattr(args, 'local_rank', 0)}"))
    if tensoIR is None:
        return None
    learned_lights = not tensoIR.general_lights
    if glb:
        path = f'{args.ckpt[:-3]}_asset.glb'
        export_asset_glb(tensoIR, path, level=0.005, texture_size=texture_size, envmaps=learned_lights, edits=edits)
    else:
        path = f'{args.ckpt[:-3]}_asset.ply'
        export_asset(tensoIR, path, level=0.005, envmaps=learned_lights, edits=edits)
    if not learned_lights:
        print(f"{args.ckpt} is a general multi-light checkpoint: its lights (lgtSGs_list) are not saved in the "
              "checkpoint, so no environment map is written")
    return path


if __name__ == "__main__":
    from opt import config_parser

    edits_path = pop_edits(sys.argv)
    glb, texture_size = pop_glb(sys.argv)
    edits = load_rules(edits_path) if edits_path else None
    args = config_parser()
    print(args)
    torch.set_default_dtype(torch.float32)
    torch.manual_seed(20211202)
    torch.cuda.manual_seed_all(20211202)
    np.random.seed(20211202)
    main(args, edits, glb, texture_size)
