"""Generate tests/golden/general_g20_train*.pt by running the REAL reference's general multi-light model (imported from
a checkout of TensoIR) through training steps on the CPU.  The reference import, its CPU stubs and the ray builder are
make_golden.py's; general_g20.pt (written by make_golden.py) is read, never rewritten.

    python tests/golden/make_general_train_golden.py <path to the TensoIR checkout>

The model is general_g20.pt's: its state_dict, its three SG sets (``lgtSGs_list``, outside the state_dict) and its
alpha mask are loaded into the reference's ``TensorVMSplit``, so every gradient belongs to the stored state.  Three
training steps are recorded, each with its seed, maps, loss, every ``named_parameters()`` gradient and each SG set's:

  * "relight_mixed": ``Renderer_TensoIR_train(is_train=True, is_relight=True, sample_method='stratified_sampling')`` with
    the loss of make_golden.py's rotated training step, light ids ``arange % 3``;
  * "relight_no1": the same step on a batch that holds lights 0 and 2 only, so light 1's SG set and light_line row get
    exactly zero gradient;
  * "phase1": ``is_relight=False`` with mixed ids and an rgb loss: light_line is the only light-dependent parameter.

Gradients are stored apart from the rest, one file per step, so every file stays below 1 MB.
tests/test_oracle_general_train_cpu.py replays the oracle against it and tests/test_general_train_gpu.py checks the
CUDA path.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, _args, import_reference, rays_for  # noqa: E402

N_RAYS, N_SAMPLES, SECOND_N = 32, 60, 16
LIGHTS = ['sunset', 'snow', 'courtyard']
# name -> (seed, is_relight, light ids)
RUNS = {"relight_mixed": (201, True, torch.arange(N_RAYS) % 3),
        "relight_no1": (202, True, (torch.arange(N_RAYS) % 2) * 2),
        "phase1": (203, False, torch.arange(N_RAYS) % 3)}


def train_loss(ret, is_relight):
    """make_golden.py's rotated training loss for a relight step; the rgb term alone for a phase-1 step (whose
    brdf, normal and smoothness outputs are None)."""
    target = torch.full_like(ret["rgb_map"], 0.5)
    loss = ((ret["rgb_map"] - target) ** 2).mean()
    if is_relight:
        loss = (loss + 0.2 * ((ret["rgb_with_brdf_map"] - target) ** 2).mean()
                + 0.0005 * ret["normals_diff_map"].mean() + 0.001 * ret["normals_orientation_loss_map"].mean()
                + 0.001 * ret["albedo_smoothness_loss"] + 0.001 * ret["roughness_smoothness_loss"])
    return loss


def build_general(gen, fx):
    m = gen.TensorVMSplit(fx["aabb"].clone(), fx["grid_size"], 'cpu', density_n_comp=[16, 16, 16],
                          appearance_n_comp=[48, 48, 48], app_dim=27, near_far=[2.0, 6.0], shadingMode='MLP_Fea',
                          alphaMask_thres=0.001, density_shift=-10, distance_scale=25, pos_pe=2, view_pe=2, fea_pe=2,
                          featureC=128, step_ratio=0.5, fea2denseAct='softplus',
                          normals_kind='derived_plus_predicted', light_name_list=LIGHTS, light_kind='sg',
                          dataset=None, numLgtSGs=128)
    m.load_state_dict(fx["state_dict"])
    for p, v in zip(m.lgtSGs_list, fx["lgt_sgs_list"]):
        p.data.copy_(v)
    m.alphaMask = gen.AlphaGridMask('cpu', fx["alpha_aabb"].clone(), fx["alpha_volume"].clone())
    return m


def main():
    ru, rot, gen, ini = import_reference()
    import renderer as ref_renderer
    fx = torch.load(os.path.join(HERE, "general_g20.pt"), weights_only=False)
    m = build_general(gen, fx)
    rays = rays_for(N_RAYS, seed=9)
    assert torch.equal(rays, fx["rays"])
    out = dict(rays=rays, n_samples=N_SAMPLES, second_nsample=SECOND_N, runs={}, _parts={})
    for name, (seed, is_relight, ids) in RUNS.items():
        light_idx = ids.view(-1, 1).to(torch.int32)
        m.zero_grad()
        for p in m.lgtSGs_list:
            p.grad = None
        torch.manual_seed(seed)
        ret = ref_renderer.Renderer_TensoIR_train(rays, None, light_idx, m, N_samples=N_SAMPLES, ndc_ray=False,
                                                  white_bg=True, is_train=True, is_relight=is_relight,
                                                  sample_method='stratified_sampling', chunk_size=160000,
                                                  device='cpu', args=_args(SECOND_N))
        loss = train_loss(ret, is_relight)
        loss.backward()
        grads = {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in m.named_parameters()}
        for k, p in enumerate(m.lgtSGs_list):
            grads[f"lgtSGs_list.{k}"] = p.grad.detach().clone() if p.grad is not None else None
        out["runs"][name] = dict(seed=seed, is_relight=is_relight, light_idx=light_idx, loss=loss.detach().clone(),
                                 maps={k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in ret.items()})
        part = f"general_g20_train_grads_{name}.pt"
        torch.save(grads, os.path.join(HERE, part))
        out["_parts"][name] = part
    torch.save(out, os.path.join(HERE, "general_g20_train.pt"))
    for n in ["general_g20_train.pt"] + list(out["_parts"].values()):
        print(n, os.path.getsize(os.path.join(HERE, n)) // 1024, "KiB")


if __name__ == "__main__":
    if REF is None or not os.path.isdir(REF):
        raise SystemExit(__doc__)
    main()
