"""The primary march of TensorBase.forward (models/tensorBase_rotated_lights.py:868-1036) and
TensorBase_Init.forward (models/tensorBase_init.py:406-462), restructured around compacted sample lists.

The reference materialises [N_rays, N_samples, *] tensors and masks them; here the kernels emit the
ray-sorted list of valid samples (2-5 % of N*S), the density gather / compositing / appearance gather run on
that list with custom forward+backward kernels, and the per-ray maps are segment sums.  Row order of the
lists equals the reference's boolean-mask order, so host-side random draws (jitter on the CPU, xyz noise on
the device, background coin on the CPU) consume the generators exactly as the reference does.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch.profiler import record_function

from . import ops, tail
from . import vm_autograd as vm
from .heads import fused_head, fused_heads_multi


def _segment_sum(values, ray_id, n_rays):
    """sum over the samples of each ray: torch.sum(weight[..., None] * x, -2) of the reference."""
    if values.dim() == 1:
        out = torch.zeros(n_rays, device=values.device, dtype=values.dtype)
    else:
        out = torch.zeros((n_rays, values.shape[1]), device=values.device, dtype=values.dtype)
    return out.index_add_(0, ray_id, values)


def note_count(st, slot, count, cap):
    """Shape-static mode bookkeeping, all on the device: remember the real length of list ``slot`` (0 valid samples,
    1 appearance samples, 2 surface hits, 3 secondary appearance scratch) for the host's high-water check and raise the
    step's overflow flag when it exceeds the static capacity (static_step.py: an overflowed step is turned into an
    exact no-op and redone with larger lists)."""
    count = count.to(torch.int64)
    st["stats"][slot].copy_(count)
    st["overflow_step"].add_((count > cap).to(torch.int64))


def any_sample_in_mask(model, rays_o, rays_d, n_samples):
    """(alphaMask.sample_alpha(xyz_sampled) > 0).any(-1) of filtering_rays (tensorBase:803-804)."""
    res = vm.valid_samples(model, rays_o, rays_d, n_samples=n_samples, no_bbox=True, count_only=True)
    return res["counts"] > 0


def _derived_normals(model, xn):
    """compute_derived_normals (tensorBase:839-856): -normalize(d sigma / d x_hat), with
    d sigma = softplus'(f + shift) * d f (analytic, kernel) instead of autograd.grad(create_graph=True)."""
    feat, dfdx = vm.density_feature_and_grad(model, xn)
    if model.fea2denseAct == "softplus":
        x = feat + model.density_shift
        dsig = torch.where(x > 20, torch.ones_like(x), torch.sigmoid(x))
    else:
        dsig = (feat > 0).to(feat.dtype)
    grad = dsig[:, None] * dfdx
    return -F.normalize(grad, p=2, dim=-1, eps=1e-6)


def march(model, rays, is_train, n_samples, counters=None):
    """Shared front half: valid list -> sigma -> weights.  Returns a dict."""
    n_rays = rays.shape[0]
    st = model.__dict__.get("_tir_static")       # shape-static mode (CUDA-graph capture), see static_step.py
    if is_train:
        # a training forward always starts from freshly packed shadows: inside a captured graph this is what makes
        # every replay read the parameters the previous replay's optimizer step wrote (device_field.py)
        ops.device_field(model).refresh(model, force=True)
    jitter = None
    if is_train:
        if st is not None:
            jitter = st["jitter"]                # device buffer refilled by the host before every replay
        else:
            # the reference draws the per-ray jitter on the CPU (rand_like of a CPU tensor, tensorBase:714-718)
            jitter = torch.rand(n_rays, 1).to(rays.device)
    lst = vm.valid_samples(model, rays[:, :3], rays[:, 3:6], n_samples=n_samples, jitter=jitter, counters=counters,
                           capacity=None if st is None else st["cap_valid"])
    if st is not None:
        note_count(st, 0, lst["offsets"][-1], st["cap_valid"])
    ray_id = lst["ray"].long()
    if lst["xn"].shape[0] > 0:
        feat = vm.density_feature(model, lst["xn"])
        sigma = model.feature2density(feat)
    else:
        sigma = torch.zeros(0, device=rays.device)
    weight, t_last, acc, depth = vm.composite(sigma, lst["dist"], lst["offsets"], model.distance_scale, lst["z"])
    lst.update(ray_id=ray_id, sigma=sigma, weight=weight, t_last=t_last, acc=acc, depth=depth)
    return lst


def forward_relight(model, rays_chunk, light_idx, white_bg=True, is_train=False, is_relight=True, N_samples=-1):
    from . import primary_fused
    if primary_fused.supported(model):
        # the whole primary march as one autograd node over the fused C entry points (csrc/tir_primary.cu), with all
        # the heads (is_relight=True) or the radiance head only (is_relight=False, training's warm-up phase); the
        # modular path below (model.__dict__['_tir_modular'] = True) is kept as its cross-check
        if is_relight:
            return primary_fused.forward_relight(model, rays_chunk, light_idx, white_bg, is_train, N_samples)
        return primary_fused.forward_radiance(model, rays_chunk, light_idx, white_bg, is_train, N_samples)
    dev = rays_chunk.device
    rays = rays_chunk.float()
    n_rays = rays.shape[0]
    viewdirs = rays[:, 3:6]
    with record_function("tir::primary_march"):
        m = march(model, rays, is_train, N_samples, counters=model.__dict__.get("_tir_counters"))
    ray_id, weight, xn = m["ray_id"], m["weight"], m["xn"]
    return _forward_relight_tail(model, rays, light_idx, white_bg, is_train, is_relight, m, ray_id, weight, xn, dev,
                                 n_rays, viewdirs)


def _forward_relight_tail(model, rays, light_idx, white_bg, is_train, is_relight, m, ray_id, weight, xn, dev, n_rays,
                          viewdirs):
    st = model.__dict__.get("_tir_static")
    cnt = model.__dict__.get("_tir_counters")
    app_sel = weight > model.rayMarch_weight_thres
    if st is None:
        app_idx = torch.nonzero(app_sel).reshape(-1)
        n_app = app_idx.shape[0]
        if cnt is not None:
            cnt[2] += n_app
        w_a = weight.index_select(0, app_idx)
    else:
        # static capacity: padded index list, padding rows carry weight 0 (and therefore no gradient)
        app_idx = torch.nonzero_static(app_sel, size=st["cap_app"], fill_value=-1).reshape(-1)
        real = app_idx >= 0
        app_idx = app_idx.clamp(min=0)
        n_app = st["cap_app"]
        n_real = app_sel.sum()
        note_count(st, 1, n_real, st["cap_app"])
        if cnt is not None:
            cnt[2] += n_real
        w_a = weight.index_select(0, app_idx) * real.to(weight.dtype)
    r_a = ray_id.index_select(0, app_idx)
    x_a = xn.index_select(0, app_idx)

    acc_map, depth_map = m["acc"], m["depth"]           # per-ray sums straight from the compositing kernel

    def bg():
        # white_bg short-circuits the CPU coin (tensorBase:979 / :1004)
        return white_bg or (is_train and bool(torch.rand((1,)) < 0.5))

    if not is_relight:
        rgb_map = torch.zeros(n_rays, 3, device=dev)
        if n_app > 0:
            with record_function("tir::primary_app_stage"):
                vd = viewdirs.index_select(0, r_a)
                li = light_idx.reshape(-1).index_select(0, r_a)
                rgb = fused_head(model, "renderModule", x_a, vd, li, light="index")
                rgb_map = _segment_sum(w_a[:, None] * rgb, r_a, n_rays)
        if bg():
            depth_map = depth_map + (1. - acc_map) * rays[..., -1]
            rgb_map = rgb_map + (1. - acc_map[..., None])
        return rgb_map, depth_map, None, None, None, None, acc_map, None, None, None, None, None

    packed = None
    if n_app > 0:
        with record_function("tir::primary_app_stage"):
            vd = viewdirs.index_select(0, r_a)
            li = light_idx.reshape(-1).index_select(0, r_a)
            # each head = ONE fused kernel launch (gather -> light factor -> basis -> PE -> MLP); the heads evaluated at
            # the same points share one backward scatter into the appearance factors (heads.py)
            group = [("renderModule", vd, li, "index"), ("renderModule_brdf", x_a, None, "mean")]
            if model.normals_kind != "purely_derived":
                group.append(("renderModule_normal", x_a, None, "mean"))
            # device-side draw, same shape/order as torch.randn_like(xyz_sampled[app_mask]) (tensorBase:937)
            draw = model.__dict__.get("_tir_randn_like")       # test hook: replay the oracle's CPU stream
            x_j = x_a + (draw(x_a) if draw is not None else torch.randn_like(x_a)) * 0.01
            # all heads of the step in one autograd node: one launch each forward, ONE stacked backward chain, one
            # appearance scatter per point set (x_a, x_j)
            res = fused_heads_multi(model, [(h, x_a, xi, l, lt) for h, xi, l, lt in group]
                                    + [("renderModule_brdf", x_j, x_j, None, "mean")])
            rgb, brdf, brdf_j = res[0], res[1], res[-1]
            if model.normals_kind == "purely_predicted":
                v_n, d_n = res[2], None
            elif model.normals_kind == "purely_derived":
                v_n, d_n = _derived_normals(model, x_a), None
            else:  # derived_plus_predicted: the predicted normal shades, the derived one supervises it
                v_n, d_n = res[2], _derived_normals(model, x_a)
            # BRDF split, smoothness / normal costs, weighting and all 14 per-ray sums in one kernel (tail.py)
            packed = tail.fused_tail(w_a, r_a, rgb, brdf, brdf_j, v_n, d_n, viewdirs, n_rays)
    if packed is None:
        packed = torch.zeros(n_rays, tail.TAIL_CHANNELS, device=dev)
    if n_rays == 0:        # torch.mean over zero rays is NaN in the reference; keep that contract on the empty batch
        z3, z1 = torch.zeros(0, 3, device=dev), torch.zeros(0, 1, device=dev)
        nan = torch.full((), float("nan"), device=dev)
        return (z3, depth_map, z3.clone(), z3.clone(), z1, z3.clone(), acc_map, z1.clone(), z1.clone(), acc_map > 0.5,
                nan, nan.clone())
    # background compositing, clamps, sRGB, normal normalisation, acc_mask and the two scalar means: one kernel
    (rgb_map, depth_map, normal_map, albedo_map, roughness_map, fresnel_map, nd_map, no_map, acc_mask,
     albedo_smoothness_loss, roughness_smoothness_loss) = tail.epilogue(packed, acc_map, depth_map, rays,
                                                                        model.fixed_fresnel, bg())
    return (rgb_map, depth_map, normal_map, albedo_map, roughness_map, fresnel_map, acc_map, nd_map, no_map,
            acc_mask, albedo_smoothness_loss, roughness_smoothness_loss)


def forward_init(model, rays_chunk, white_bg=True, is_train=False, N_samples=-1):
    """TensorBase_Init.forward (tensorBase_init.py:406-462) -> (rgb_map, depth_map)."""
    rays = rays_chunk.float()
    n_rays = rays.shape[0]
    m = march(model, rays, is_train, N_samples, counters=model.__dict__.get("_tir_counters"))
    ray_id, weight, xn = m["ray_id"], m["weight"], m["xn"]
    app_idx = torch.nonzero(weight > model.rayMarch_weight_thres).reshape(-1)
    acc_map = m["acc"]
    rgb_map = torch.zeros(n_rays, 3, device=rays.device)
    if app_idx.shape[0] > 0:
        r_a = ray_id.index_select(0, app_idx)
        x_a = xn.index_select(0, app_idx)
        rgb = fused_head(model, "renderModule", x_a, rays[:, 3:6].index_select(0, r_a), None, light="none")
        rgb_map = _segment_sum(weight.index_select(0, app_idx)[:, None] * rgb, r_a, n_rays)
    if white_bg or (is_train and bool(torch.rand((1,)) < 0.5)):
        rgb_map = rgb_map + (1. - acc_map[..., None])
    rgb_map = rgb_map.clamp(0, 1)
    with torch.no_grad():
        depth_map = m["depth"].detach() + (1. - acc_map) * rays[..., -1]
    return rgb_map, depth_map
