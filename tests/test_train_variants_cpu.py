"""The trainer's general multi-light and simple variants on the host: the up-front checks on the reference's configs,
the dataset constructor arguments of the entry scripts (tools/train_tensoIR*.py), the order of the scripts' __main__
block (mesh export, then rendering or training) and render_test without a checkpoint."""
import importlib.util
import os
import sys
import types

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from tensoir_b200 import train  # noqa: E402

# configs/multi_light_general/lego.txt and configs/single_light/blender.txt as opt.config_parser parses them (the
# options these files set; every other option keeps its parser default, taken from the recorded armadillo namespace)
GENERAL_LEGO = dict(
    dataset_name="tensoIR_unknown_general_multi_lights", datadir="./data/TensoIR_Synthetic/lego",
    hdrdir="./data/Environment_Maps/high_res_envmaps_2k", expname="lego_ds_1", basedir="./log/log_general_multi_lights",
    add_timestamp=1, downsample_train=1.0, downsample_test=1.0, n_iters=80000, batch_size=4096, lr_decay_iters=80000,
    N_voxel_init=2097152, N_voxel_final=27000000, upsamp_list=[10000, 20000, 30000, 40000],
    update_AlphaMask_list=[10000, 15000, 20000, 25000, 30000, 35000], N_vis=5, vis_every=5000, render_test=1,
    n_lamb_sigma=[16, 16, 16], n_lamb_sh=[48, 48, 48], model_name="TensorVMSplit", shadingMode="MLP_Fea",
    fea2denseAct="softplus", view_pe=2, fea_pe=2, pos_pe=2, light_rotation=["000"],
    light_name_list=["sunset", "snow", "courtyard"], light_kind="sg", numLgtSGs=128,
    normals_kind="derived_plus_predicted", normals_diff_weight=0.002, normals_orientation_weight=0.002,
    rgb_brdf_weight=0.2, batch_size_test=4096, light_name="sunset", albedo_smoothness_loss_weight=0.001,
    roughness_smoothness_loss_weight=0.001, L1_weight_inital=8e-5, L1_weight_rest=4e-5, rm_weight_mask_thre=1e-4,
    TV_weight_density=0.05, TV_weight_app=0.005)
SIMPLE_BLENDER = dict(
    dataset_name="blender", datadir="./data/nerf_synthetic/mic/", hdrdir="./data/Environment_Maps/high_res_envmaps_2k",
    expname="blender_ds_1", basedir="./log/log_original_blender", add_timestamp=1, downsample_train=1.0,
    downsample_test=1.0, n_iters=80000, batch_size=4096, lr_decay_iters=80000, N_voxel_init=2097152,
    N_voxel_final=27000000, upsamp_list=[10000, 20000, 30000, 40000],
    update_AlphaMask_list=[10000, 15000, 20000, 25000, 30000, 35000], N_vis=5, vis_every=5000, render_test=1,
    n_lamb_sigma=[16, 16, 16], n_lamb_sh=[48, 48, 48], model_name="TensorVMSplit", shadingMode="MLP_Fea",
    fea2denseAct="softplus", view_pe=2, fea_pe=2, pos_pe=2, light_rotation=["000"], light_kind="sg", numLgtSGs=128,
    normals_kind="derived_plus_predicted", normals_diff_weight=0.005, normals_orientation_weight=0.005,
    rgb_brdf_weight=0.2, batch_size_test=4096, light_name="None", albedo_smoothness_loss_weight=0.001,
    roughness_smoothness_loss_weight=0.001, L1_weight_inital=8e-5, L1_weight_rest=4e-5, rm_weight_mask_thre=1e-4,
    TV_weight_density=0.1, TV_weight_app=0.01)


# the recorded armadillo namespace has no data paths
PATHS = dict(datadir="./data/TensoIR_Synthetic/armadillo", hdrdir="./data/Environment_Maps/high_res_envmaps_2k")


def _args(values):
    defaults = torch.load(os.path.join(HERE, "golden", "schedule_armadillo.pt"), weights_only=False)["config"]
    return types.SimpleNamespace(**(dict(defaults) | PATHS | values))


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Recorder:
    """A dataset class that records its constructor arguments."""
    calls = []

    def __init__(self, *a, **k):
        Recorder.calls.append((a, k))


def test_check_supported_accepts_the_reference_general_and_simple_configs():
    g = _args(GENERAL_LEGO)
    train.check_supported(g, "general")
    train.check_supported(g, "general", types.SimpleNamespace(light_num=3))
    train.check_supported(_args(SIMPLE_BLENDER), "simple")


@pytest.mark.parametrize("names", [None, []])
def test_check_supported_rejects_a_general_run_without_light_names(names):
    with pytest.raises(ValueError, match="light_name_list"):
        train.check_supported(_args(GENERAL_LEGO | {"light_name_list": names}), "general")


def test_check_supported_rejects_a_light_count_other_than_the_training_sets():
    with pytest.raises(ValueError, match="light_num = 2"):
        train.check_supported(_args(GENERAL_LEGO), "general", types.SimpleNamespace(light_num=2))
    with pytest.raises(ValueError, match="light_num = None"):
        train.check_supported(_args(GENERAL_LEGO), "general", types.SimpleNamespace())


@pytest.mark.parametrize("variant,cfg", [("full", {}), ("general", GENERAL_LEGO), ("simple", SIMPLE_BLENDER)])
def test_check_supported_rejects_render_path(variant, cfg):
    with pytest.raises(ValueError, match="render_path"):
        train.check_supported(_args(cfg | {"render_path": 1, "render_only": 1}), variant)


def test_check_supported_rejects_an_unknown_variant():
    with pytest.raises(ValueError, match="variant"):
        train.check_supported(_args({}), "rotated")


# (the reconstruction train set, its test set, the render_test test set) as each reference script constructs them
def _want(a):
    return {
        "train_tensoIR": [
            ((a.datadir, a.hdrdir), dict(split='train', downsample=a.downsample_train, light_name=a.light_name,
                                         light_rotation=a.light_rotation)),
            ((a.datadir, a.hdrdir), dict(split='test', downsample=a.downsample_test, light_name=a.light_name,
                                         light_rotation=a.light_rotation)),
            ((a.datadir, a.hdrdir), dict(light_rotation=a.light_rotation, split='test',
                                         downsample=a.downsample_train, is_stack=False, sub=a.test_number))],
        "train_tensoIR_general_multi_lights": [
            ((a.datadir, a.hdrdir), dict(split='train', downsample=a.downsample_train, light_name=a.light_name,
                                         light_name_list=a.light_name_list, light_rotation=a.light_rotation)),
            ((a.datadir, a.hdrdir), dict(split='test', downsample=a.downsample_test, light_name=a.light_name,
                                         light_name_list=a.light_name_list, light_rotation=a.light_rotation)),
            ((a.datadir, a.hdrdir), dict(split='test', downsample=a.downsample_train, is_stack=False,
                                         sub=a.test_number))],
        "train_tensoIR_simple": [
            ((a.datadir,), dict(split='train', downsample=a.downsample_train, light_name=a.light_name,
                                light_rotation=a.light_rotation, scene_bbox=a.scene_bbox)),
            ((a.datadir,), dict(split='test', downsample=a.downsample_test, light_name=a.light_name,
                                light_rotation=a.light_rotation, scene_bbox=a.scene_bbox, is_stack=True)),
            ((a.datadir,), dict(split='test', downsample=a.downsample_train, is_stack=True, sub=a.test_number))],
    }


@pytest.mark.parametrize("name", ["train_tensoIR", "train_tensoIR_general_multi_lights", "train_tensoIR_simple"])
def test_entry_scripts_build_the_reference_datasets(name):
    # distinct values, so that an argument passed under the wrong name shows
    a = _args(GENERAL_LEGO | {"downsample_train": 2.0, "downsample_test": 4.0, "test_number": 7,
                              "scene_bbox": ["-1,-1,-1", "1,1,1"], "light_rotation": ["000", "120"]})
    tool = _tool(name)
    Recorder.calls = []
    tool.datasets(Recorder, a)
    tool.render_dataset(Recorder, a)
    assert Recorder.calls == _want(a)[name]


@pytest.mark.parametrize("render_only,render_test,want", [(1, 1, "render_test"), (0, 1, "reconstruction"),
                                                          (1, 0, "reconstruction")])
@pytest.mark.parametrize("name,variant,cfg", [("train_tensoIR", "full", {}),
                                              ("train_tensoIR_general_multi_lights", "general", GENERAL_LEGO),
                                              ("train_tensoIR_simple", "simple", SIMPLE_BLENDER)])
def test_entry_scripts_export_the_mesh_first_then_render_or_train(monkeypatch, tmp_path, name, variant, cfg,
                                                                   render_only, render_test, want):
    a = _args(cfg | {"export_mesh": 1, "ckpt": str(tmp_path / "m.th"), "render_only": render_only,
                     "render_test": render_test, "basedir": str(tmp_path), "add_timestamp": 0})
    seen = []
    monkeypatch.setattr(train, "export_mesh", lambda args, device=None: seen.append(("export_mesh", args.ckpt)))
    monkeypatch.setattr(train, "render_test", lambda args, ds, log, *, variant, device=None:
                        seen.append(("render_test", len(Recorder.calls), log, variant)))
    monkeypatch.setattr(train, "reconstruction", lambda args, tr, te, log, *, variant, device=None:
                        seen.append(("reconstruction", len(Recorder.calls), log, variant)) or
                        {"redone": 0, "recaptures": 0})
    Recorder.calls = []
    _tool(name).main(a, Recorder)
    assert seen[0] == ("export_mesh", a.ckpt)
    assert seen[1][0] == want and seen[1][3] == variant and len(seen) == 2
    if want == "render_test":
        assert seen[1][1] == 1 and seen[1][2].startswith(f"{tmp_path}/test_{a.expname}-")
    else:
        assert seen[1][1] == 2 and seen[1][2] == f"{tmp_path}/{a.expname}"


@pytest.mark.parametrize("variant,cfg", [("full", {}), ("general", GENERAL_LEGO), ("simple", SIMPLE_BLENDER)])
def test_render_test_without_a_checkpoint_prints_the_reference_message_and_writes_nothing(tmp_path, capsys, variant,
                                                                                         cfg):
    a = _args(cfg | {"ckpt": str(tmp_path / "missing.th"), "render_only": 1, "render_test": 1})
    assert train.render_test(a, None, str(tmp_path / "test_x"), variant=variant) is None
    assert capsys.readouterr().out == "the ckpt path does not exists!!\n"
    assert os.listdir(tmp_path) == []
