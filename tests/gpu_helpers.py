"""Build tensoir_b200 models from golden fixtures (GPU tests, smoke, bench)."""
import os
import types

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_fixture(name):
    """A golden fixture; entries listed under "_parts" are stored in files of their own (every file stays < 1 MB)."""
    fx = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    for key, part in fx.pop("_parts", {}).items():
        fx[key] = torch.load(os.path.join(GOLDEN, part), weights_only=False)
    return fx


def load_shrunk_state(state):
    """State "A" or "B" of shrunk_g30.pt (tests/golden/make_shrunk_golden.py) as one flat fixture dict, in the layout
    of rotated_g24.pt: the state's records plus the shared parameters, rays and light indices."""
    fx = load_fixture("shrunk_g30.pt")
    for key in ("state_dict", f"renderer_train_grads_{state}"):
        fx[key] = {**fx.pop(f"{key}:factors"), **fx.pop(f"{key}:rest")}
    out = {k: v for k, v in fx.items() if k != "states" and not k.startswith("renderer_train_grads_")}
    out.update(fx["states"][state])
    out["renderer_train_grads"] = fx[f"renderer_train_grads_{state}"]
    out["state"] = state
    return out


def renderer_args(n=96, near=0.05, far=1.5):
    a = types.SimpleNamespace()
    a.second_nSample, a.second_near, a.second_far = n, near, far
    return a


def model_from_fixture(fx, device, with_mask=True):
    from tensoir_b200 import TensorVMSplit, TensorVMSplitInit, AlphaGridMask
    aabb = fx["aabb"].to(device)
    common = dict(density_n_comp=[16, 16, 16], appearance_n_comp=[48, 48, 48], app_dim=27, near_far=[2.0, 6.0],
                  shadingMode='MLP_Fea', alphaMask_thres=0.001, density_shift=-10, distance_scale=25, pos_pe=2,
                  view_pe=2, fea_pe=2, featureC=128, step_ratio=0.5, fea2denseAct='softplus')
    if fx["kind"] == "init":
        m = TensorVMSplitInit(aabb, fx["grid_size"], device, **common)
    elif fx["kind"] == "rotated":
        m = TensorVMSplit(aabb, fx["grid_size"], device, normals_kind='derived_plus_predicted',
                          light_rotation=[f"{r:03d}" for r in fx["light_rotation"]], light_kind='sg',
                          numLgtSGs=128, **common)
    else:
        m = TensorVMSplit(aabb, fx["grid_size"], device, normals_kind='derived_plus_predicted',
                          light_name_list=['sunset', 'snow', 'courtyard'], light_kind='sg', numLgtSGs=128, **common)
        for p, v in zip(m.lgtSGs_list, fx["lgt_sgs_list"]):
            p.data.copy_(v.to(device))
    m.load_state_dict({k: v.to(device) for k, v in fx["state_dict"].items()})
    if with_mask:
        m.alphaMask = AlphaGridMask(device, fx["alpha_aabb"].to(device), fx["alpha_volume"].to(device))
    return m


def app_sample_list(xn, weight, ray, sample=None):
    """A TirAppSample list (24 B per row: xn[3], weight f32, ray, sample i32) for tir_app_mlp, on xn's device
    -> (uint8 buffer, int32 [1] count).  With one sample per ray at weight 1 and n_dirs = 0, the list kernel writes
    exactly the per-point MLP output into a zeroed rgb_out."""
    n = xn.shape[0]
    if sample is None:
        sample = torch.zeros(n, dtype=torch.int32, device=xn.device)
    f = torch.cat([xn.reshape(n, 3).float(), weight.reshape(n, 1).float()], 1).contiguous()
    i = torch.stack([ray.reshape(n).to(torch.int32), sample.reshape(n).to(torch.int32)], 1).contiguous()
    buf = torch.cat([f.view(torch.uint8), i.view(torch.uint8)], 1).reshape(-1).contiguous()
    return buf, torch.tensor([n], dtype=torch.int32, device=xn.device)


def app_mlp_list(model, mlp, xn, dirs, light_idx, weight=None, ray=None, n_rays=None):
    """The wgmma list kernel (tir_app_mlp) on a hand-built list with n_dirs = 0: sample i at xn[i] on ray ray[i] (default
    i) with weight[i] (default 1), view dir dirs[ray], light light_idx[ray] (or None) -> rgb [n_rays, 3]."""
    import ctypes as C
    from tensoir_b200 import _lib, ops
    n = xn.shape[0]
    dev = xn.device
    ray = torch.arange(n, device=dev) if ray is None else ray
    weight = torch.ones(n, device=dev) if weight is None else weight
    n_rays = n if n_rays is None else n_rays
    buf, count = app_sample_list(xn, weight, ray)
    d = dirs.reshape(-1, 3).float().contiguous()
    li = None if light_idx is None else light_idx.reshape(-1).to(torch.int32).contiguous()
    rgb = torch.zeros(n_rays, 3, device=dev)
    f = ops.device_field(model).refresh(model)
    _lib.check(_lib.load().tir_app_mlp(C.byref(f), C.byref(mlp), _lib.dptr(buf, torch.uint8),
                                       _lib.dptr(count, torch.int32), n, _lib.dptr(d), 0,
                                       None if li is None else _lib.dptr(li, torch.int32), _lib.dptr(rgb),
                                       _lib.stream_ptr()), "tir_app_mlp")
    return rgb
