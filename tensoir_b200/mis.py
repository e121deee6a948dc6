"""Relighting under environment maps with multiple importance sampling (csrc/tir_relight_mis.cu), opt-in through
relight(args.sampling='mis').

relight()'s default estimator (relight_chunk_fused) is the reference's: every sample sits at a texel centre and is
drawn in proportion to the map's intensity only.  A glossy lobe narrower than the bright region it reflects then gets
a handful of samples and shows as speckle, and a lobe narrower than a texel is evaluated only where it covers a centre.
relight_chunk_mis estimates the continuous integral

    Lo = integral of f(w) V(w) E(w) cos(w) dw,   E piecewise constant over the map's texels,

with S_l light samples per (map, hit), each uniform in the solid angle of a texel drawn from the CDF, and S_b BRDF
samples per hit (half GGX visible normals, half cosine), shared by every map and marched once, combined with the
balance heuristic:

    linear = sum over all S_l + S_b samples of f V E cos / (S_l p_light(w) + S_b p_brdf(w))

(definitions in csrc/tir_mis_body.h).  The visibility list is marched in slot order (relighting.slot_order), so two
calls with the same draws give identical bits.
"""
from __future__ import annotations

import torch

from . import _lib
from .relighting import append_list, chunk_inputs, env_groups, env_tables, march_list, rescale3, vis_kind


def mis_uniforms(L, n, S_l, S_b, device):
    """The draws of one chunk: u_light [L, n, S_l, 3], then u_brdf [n, S_b, 3], fp64 in [0, 1)."""
    u_light = torch.rand(L, n, S_l, 3, device=device, dtype=torch.float64)
    return u_light, torch.rand(n, S_b, 3, device=device, dtype=torch.float64)


def mis_visibility(tensoIR, envs, L, rays, depth, normal, albedo, rough, fresnel, acc, u_light, u_brdf,
                   acc_mask_threshold, vis_equation):
    """tir_relight_mis_sample and the slot-ordered march of its list for up to RELIGHT_MAX_LIGHTS maps (contiguous fp32
    device inputs).  -> (dir [slots,3], pos [slots], vis), what tir_relight_mis_shade reads."""
    lib = _lib.load()
    dev = rays.device
    n, S_l, S_b = int(rays.shape[0]), int(u_light.shape[2]), int(u_brdf.shape[1])
    slots = L * n * S_l + n * S_b
    dirs = torch.empty(slots, 3, device=dev)
    pos = torch.empty(slots, dtype=torch.int32, device=dev)
    list_o, list_d = append_list(
        slots, dev, "relight visibility list", pos,
        lambda *tail: _lib.check(lib.tir_relight_mis_sample(
            envs, L, _lib.dptr(rays), _lib.dptr(depth), _lib.dptr(normal), _lib.dptr(albedo), _lib.dptr(rough),
            int(rough.shape[1]), _lib.dptr(fresnel), _lib.dptr(acc), n, S_l, S_b, float(acc_mask_threshold),
            _lib.dptr(u_light, torch.float64), _lib.dptr(u_brdf, torch.float64), _lib.dptr(dirs),
            _lib.dptr(pos, torch.int32), *tail, _lib.stream_ptr()), "tir_relight_mis_sample"))
    return dirs, pos, march_list(tensoIR, list_o, list_d, vis_equation)


@torch.no_grad()
def relight_chunk_mis(tensoIR, envir_light, light_names, rays, maps, rescale_value, u_light, u_brdf, *,
                      acc_mask_threshold=0.5, vis_equation='nerv', out=None, row0=0, tables=None, linear_out=None):
    """relight_chunk_fused (relighting.py) with the MIS estimator, under the same contract: ``maps`` = (depth, normal,
    albedo, roughness [n,1] or [n,3], fresnel, acc) of the primary render of ``rays``.  ``u_light`` [L, n, S_l, 3] and
    ``u_brdf`` [n, S_b, 3] fp64 uniforms (mis_uniforms; S_l >= 1, S_b >= 0).  ``linear_out`` [L, R, 3] receives the
    un-toned estimate at rows row0.. (0 on non-hit rows).  -> (with_bg, without_bg) [L, n, 3]."""
    kind = vis_kind(vis_equation)
    dev = rays.device
    L, n = len(light_names), int(rays.shape[0])
    rays, (depth, normal, albedo, rough, fresnel, acc) = chunk_inputs(rays, maps)
    if u_light.dim() != 4 or tuple(u_light.shape[:2]) != (L, n) or u_light.shape[3] != 3 or u_light.shape[2] < 1 \
            or u_light.dtype != torch.float64:
        raise ValueError(f"u_light must be float64 [{L}, {n}, S_l >= 1, 3], got {u_light.dtype} {tuple(u_light.shape)}")
    if u_brdf.dim() != 3 or u_brdf.shape[0] != n or u_brdf.shape[2] != 3 or u_brdf.dtype != torch.float64:
        raise ValueError(f"u_brdf must be float64 [{n}, S_b, 3], got {u_brdf.dtype} {tuple(u_brdf.shape)}")
    u_light, u_brdf = u_light.to(dev).contiguous(), u_brdf.to(dev).contiguous()
    if out is None:
        out = (torch.empty(L, n, 3, device=dev), torch.empty(L, n, 3, device=dev))
        row0 = 0
    with_bg, without_bg = out
    if n == 0 or L == 0:
        return with_bg[:, row0:row0 + n], without_bg[:, row0:row0 + n]
    envs, keep = tables if tables is not None else env_tables(envir_light, light_names)
    resc = rescale3(rescale_value, dev)
    thr = float(acc_mask_threshold)
    S_l, S_b = int(u_light.shape[2]), int(u_brdf.shape[1])
    lib = _lib.load()
    for g, Lg, eg in env_groups(envs, L):
        dirs, pos, vis = mis_visibility(tensoIR, eg, Lg, rays, depth, normal, albedo, rough, fresnel, acc,
                                        u_light[g:g + Lg], u_brdf, thr, vis_equation)
        lin = linear_out[g:g + Lg] if linear_out is not None else None
        _lib.check(lib.tir_relight_mis_shade(eg, Lg, _lib.dptr(rays), _lib.dptr(normal), _lib.dptr(albedo),
                                             _lib.dptr(rough), int(rough.shape[1]), _lib.dptr(fresnel), _lib.dptr(acc),
                                             n, S_l, S_b, thr, _lib.dptr(resc), _lib.dptr(dirs),
                                             _lib.dptr(pos, torch.int32), _lib.dptr(vis), kind,
                                             _lib.dptr(with_bg[g:g + Lg]), _lib.dptr(without_bg[g:g + Lg]),
                                             _lib.dptr(lin, allow_none=True), int(with_bg.shape[1]), int(row0),
                                             _lib.stream_ptr()), "tir_relight_mis_shade")
    del keep
    return with_bg[:, row0:row0 + n], without_bg[:, row0:row0 + n]
