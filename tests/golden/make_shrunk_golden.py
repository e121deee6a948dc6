"""Generate tests/golden/shrunk_g30*.pt by running the REAL reference (imported from a checkout of TensoIR) on the CPU.
The reference import, its CPU stubs and the rotated-model builder are make_golden.py's.

    python tests/golden/make_shrunk_golden.py <path to the TensoIR checkout>

A training run calls updateAlphaMask + shrink and then upsample_volume_grid; from then on the field is no longer cubic,
its aabb differs per axis and the alpha mask has its own resolution and box.  Two such states of the rotated G=24
fixture model are recorded:

  * state "A": updateAlphaMask((24,24,24)), shrink to an asymmetric box inside the mask's bounding box, then
    upsample_volume_grid([30,31,29]).  The alpha mask stays 24^3 on the old +-1.5 box.
  * state "B": state A followed by updateAlphaMask(gridSize): a 29x31x30 (Z,Y,X) mask on the shrunk box.

Both states share the parameters (updateAlphaMask changes none), so the state_dict is stored once.  For each state:
sample_ray (eval / train with a recorded jitter), the unit functions on 257 points, the derived normals on jittered
points that leave [-1,1], compute_transmittance / compute_radiance, the eval boundary and one training step (outputs,
loss, every parameter gradient).  tests/test_oracle_shrunk_golden.py replays the oracle against it and
tests/test_shrunk_field_gpu.py checks the CUDA path.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, _args, build_rotated, import_reference, rays_for, tolist  # noqa: E402

SHRINK_BOX = [[-1.05, -0.9, -0.95], [1.1, 1.0, 0.85]]     # x, y and z all differ; inside the mask's new_aabb
UPSAMPLE = [30, 31, 29]
N_RAYS = 48


def detached(d):
    return {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in d.items()}


def record_state(m, ru, ref_renderer, rays, light_idx):
    """Everything the replay and the GPU tests compare, for the model ``m`` in its current state."""
    n = rays.shape[0]
    fx = dict(aabb=m.aabb.clone(), grid_size=m.gridSize.tolist(), nSamples=m.nSamples, stepSize=float(m.stepSize),
              alpha_volume=m.alphaMask.alpha_volume.clone(), alpha_aabb=m.alphaMask.aabb.clone())
    # a) unit functions on points of the box grown by 5 % (some leave it: zero padding / clamped taps)
    g = torch.Generator().manual_seed(11)
    lo, hi = m.aabb[0], m.aabb[1]
    pts = (lo + hi) / 2 + (hi - lo) / 2 * (torch.rand(257, 3, generator=g) * 2 - 1) * 1.05
    xn = m.normalize_coord(pts)
    fx["pts"] = pts
    fx["sample_alpha"] = m.alphaMask.sample_alpha(pts).clone()
    fx["density_feature"] = m.compute_densityfeature(xn).detach().clone()
    fx["sigma"] = m.feature2density(m.compute_densityfeature(xn)).detach().clone()
    li = (torch.arange(257) % 2).view(-1, 1).to(torch.int32)
    rad, intr = m.compute_bothfeature(xn, li)
    fx["li"], fx["rad_feat"], fx["intr_feat"] = li, rad.detach().clone(), intr.detach().clone()
    fx["app_feat"] = m.compute_appfeature(xn, li).detach().clone()
    fx["intrin_only"] = m.compute_intrinfeature(xn).detach().clone()
    vd = torch.nn.functional.normalize(torch.randn(257, 3, generator=g), dim=-1)
    fx["viewdirs"] = vd
    fx["mlp_rgb"] = m.renderModule(xn, vd, rad).detach().clone()
    fx["mlp_brdf"] = m.renderModule_brdf(xn, intr).detach().clone()
    fx["mlp_normal"] = m.renderModule_normal(xn, intr).detach().clone()
    xj = (xn + 0.05 * torch.randn(257, 3, generator=g)).detach()
    fx["xj"] = xj
    fx["derived_normals"] = m.compute_derived_normals(xj.clone()).detach().clone()
    # b) sample_ray, eval and train with a recorded jitter
    p, z, v = m.sample_ray(rays[:, :3], rays[:, 3:6], is_train=False, N_samples=-1)
    fx["sample_ray_eval"] = (p.clone(), z.clone(), v.clone())
    torch.manual_seed(5)
    p, z, v = m.sample_ray(rays[:, :3], rays[:, 3:6], is_train=True, N_samples=40)
    torch.manual_seed(5)
    fx["jitter40"] = torch.rand(n, 1)
    fx["sample_ray_train"] = (p.clone(), z.clone(), v.clone())
    # c) secondary marches from surface points inside the shrunk box
    surf = (lo + hi) / 2 + (hi - lo) / 2 * (torch.rand(96, 3, generator=g) * 2 - 1) * 0.9
    dirs = torch.nn.functional.normalize(torch.randn(96, 3, generator=g), dim=-1)
    li2 = (torch.arange(96) % 2).view(-1, 1).to(torch.int32)
    fx["surf"], fx["dirs"], fx["li2"] = surf, dirs, li2
    fx["transmittance"] = tolist(ru.compute_transmittance(tensoIR=m, surf_pts=surf, light_in_dir=dirs, nSample=96,
                                                          vis_near=0.05, vis_far=1.5))
    fx["radiance"] = tolist(ru.compute_radiance(tensoIR=m, surf_pts=surf, light_in_dir=dirs, light_idx=li2,
                                                nSample=96, vis_near=0.05, vis_far=1.5))
    # d) the eval boundary, then one training step with its gradients
    args = _args(24)
    torch.manual_seed(102)
    ret = ref_renderer.Renderer_TensoIR_train(rays, None, light_idx, m, N_samples=-1, ndc_ray=False, white_bg=True,
                                              is_train=False, is_relight=True, sample_method='fixed_envirmap',
                                              chunk_size=160000, device='cpu', args=args)
    fx["renderer_eval"] = detached(ret)
    torch.manual_seed(77)
    m.zero_grad()
    ret = ref_renderer.Renderer_TensoIR_train(rays, None, light_idx, m, N_samples=60, ndc_ray=False, white_bg=True,
                                              is_train=True, is_relight=True, sample_method='stratified_sampling',
                                              chunk_size=160000, device='cpu', args=args)
    target = torch.full_like(ret["rgb_map"], 0.5)
    loss = (((ret["rgb_map"] - target) ** 2).mean() + 0.2 * ((ret["rgb_with_brdf_map"] - target) ** 2).mean()
            + 0.0005 * ret["normals_diff_map"].mean() + 0.001 * ret["normals_orientation_loss_map"].mean()
            + 0.001 * ret["albedo_smoothness_loss"] + 0.001 * ret["roughness_smoothness_loss"])
    loss.backward()
    fx["renderer_train"] = detached(ret)
    fx["renderer_train_loss"] = loss.detach().clone()
    fx["train_seed"] = 77
    grads = {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in m.named_parameters()}
    m.zero_grad()
    return fx, grads


def main():
    ru, rot, _, _ = import_reference()
    import renderer as ref_renderer
    m = build_rotated(rot)
    first_aabb = m.updateAlphaMask((24, 24, 24))
    box = torch.tensor(SHRINK_BOX)
    assert bool((box[0] >= first_aabb[0]).all() and (box[1] <= first_aabb[1]).all()), first_aabb
    m.shrink(box.clone())
    m.upsample_volume_grid(UPSAMPLE)
    rays = rays_for(64)[:N_RAYS].contiguous()
    light_idx = (torch.arange(N_RAYS) % 2).view(-1, 1).to(torch.int32)
    out = dict(kind="rotated", light_rotation=list(m.light_rotation), shrink_box=box, upsample=list(UPSAMPLE),
               first_new_aabb=first_aabb.clone(), rays=rays, light_idx=light_idx,
               state_dict={k: v.detach().clone() for k, v in m.state_dict().items()})
    states, parts = {}, {}
    fa, ga = record_state(m, ru, ref_renderer, rays, light_idx)
    states["A"] = fa
    new_aabb = m.updateAlphaMask(tuple(m.gridSize.tolist()))
    fb, gb = record_state(m, ru, ref_renderer, rays, light_idx)
    fb["new_aabb"] = new_aabb.clone()
    states["B"] = fb
    assert all(torch.equal(v, out["state_dict"][k]) for k, v in m.state_dict().items())   # the mask changes no parameter
    out["states"] = states
    # a 30x31x29 state_dict is about 1.1 MB: the VM factors and the rest (MLPs, basis, lights) go to separate files
    for key, d in (("state_dict", out.pop("state_dict")), ("renderer_train_grads_A", ga),
                   ("renderer_train_grads_B", gb)):
        for half, keep in (("factors", True), ("rest", False)):
            out[f"{key}:{half}"] = {k: v for k, v in d.items() if k.startswith(("density_", "app_")) == keep}
            parts[f"{key}:{half}"] = f"shrunk_g30_{key.replace('renderer_train_', '')}_{half}.pt"
    for key, part in parts.items():                  # stored apart: every fixture file stays below 1 MB
        torch.save(out.pop(key), os.path.join(HERE, part))
    torch.save(dict(out, _parts=parts), os.path.join(HERE, "shrunk_g30.pt"))
    for f in ["shrunk_g30.pt"] + list(parts.values()):
        size = os.path.getsize(os.path.join(HERE, f))
        print(f, size // 1024, "KiB")
        assert size < 1 << 20, f


if __name__ == "__main__":
    if REF is None or not os.path.isdir(REF):
        raise SystemExit(__doc__)
    main()
