"""Relighting with one bounce of indirect light under environment maps (csrc/tir_indirect.cu).

relight() shades every surface hit with direct environment light and marched visibility.  TensoIR fits its materials
with indirect light switched on, so that leaves concave regions darker than the materials imply.
relight_chunk_indirect adds one bounce:

    linear[l,i] = (1/S)  * sum_s direct_s                  (exactly tir_relight_shade's sum, same order, same bits)
                + (1/K)  * sum_k T[i,k] * w[i,k] * Lo[l, h(i,k)]

K cosine-weighted directions per hit are marched with relight()'s visibility table.  The slots whose march is occluded
(w = 1 - vis > 1e-3) become secondary hits x, compacted in slot order.  The model's heads give the material at x, and
Lo is the direct light of every map at x, seen from the primary hit and sampled and marched as relight() does it.  The
secondary hit gets direct light only: one bounce, and cosine sampling only (no GGX-lobe sampling, no MIS), so glossy
interreflection at low roughness is noisy.

Every list the march reads is put in slot order first (relighting.slot_order): the march's result for a ray can
change in its last bits with its neighbours in the list, and the appended lists follow warp scheduling.  So two calls
with the same draws give identical bits.  The direct term is relight_chunk_fused's estimator on the same draws; it
differs from relight_chunk_fused's output only by that list order, in the last bits of the visibility.

Random draws: the direct uniforms are the caller's (relighting._uniforms, as for relight_chunk_fused), and the indirect
draws come from ``gen``: u [n, K, 2], then [L, m, S2] per sub-list of hits.  The direct term does not depend on the
indirect draws, so "with - without" indirect light is exactly the indirect term.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn.functional as F

from . import _lib, ops  # noqa: F401  (indirect.ops.march_density is where callers substitute the march)
from .relighting import (append_list, chunk_inputs, env_groups, env_tables, march_list, relight_visibility,
                         rescale3, vis_kind)


def point_materials(tensoIR, x, xn=None):
    """The material the eval forward returns for a ray whose whole weight is one sample at each world point of ``x``
    [m, 3]: albedo and roughness from the BRDF head (light "mean"), split as tail.fused_tail does and clamped as
    tail.epilogue does; fresnel = fixed_fresnel; the predicted normal, normalised (the derived normal for
    purely_derived models).  ``xn``: the aabb-normalised points, when already known.
    -> (normal [m,3], albedo [m,3], rough [m,1], fresnel [m,3])."""
    from .heads import fused_heads_multi
    from .primary import _derived_normals
    x = x.detach().float().reshape(-1, 3)
    m, dev = x.shape[0], x.device
    xn = (tensoIR.normalize_coord(x) if xn is None else xn).detach().float().reshape(-1, 3).contiguous()
    fresnel = torch.full((m, 3), float(tensoIR.fixed_fresnel), device=dev).clamp(0.0, 1.0)
    if m == 0:
        return torch.zeros(0, 3, device=dev), torch.zeros(0, 3, device=dev), torch.zeros(0, 1, device=dev), fresnel
    specs = [("renderModule_brdf", xn, xn, None, "mean")]
    derived = tensoIR.normals_kind == "purely_derived"
    if not derived:
        specs.append(("renderModule_normal", xn, xn, None, "mean"))
    res = fused_heads_multi(tensoIR, specs)
    brdf = res[0]
    albedo = brdf[:, :3].clamp(0.0, 1.0)
    rough = (brdf[:, 3:4] * 0.9 + 0.09).clamp(0.0, 1.0)
    normal = _derived_normals(tensoIR, xn) if derived else F.normalize(res[1], p=2, dim=-1, eps=1e-6)
    return normal.contiguous(), albedo.contiguous(), rough.contiguous(), fresnel


def secondary_hits(tensoIR, rays, depth, normal, albedo, rough, fresnel, acc, rescale, u, acc_mask_threshold,
                   vis_equation):
    """tir_indirect_sample, the march of the secondary rays and tir_indirect_hits for one chunk (contiguous fp32
    inputs, u [n, K, 2] fp64).  -> dict of T [n,K,3], hit [n,K], and the hit list: rays [m,6] = (x, omega), xn [m,3],
    w [m]."""
    lib = _lib.load()
    dev = rays.device
    n, K = int(rays.shape[0]), int(u.shape[1])
    cap = n * K
    dirs = torch.empty(n, K, 3, device=dev)
    T = torch.empty(n, K, 3, device=dev)
    pos = torch.empty(n, K, dtype=torch.int32, device=dev)
    list_o, list_d = append_list(
        cap, dev, "secondary list", pos,
        lambda *tail: _lib.check(lib.tir_indirect_sample(
            _lib.dptr(rays), _lib.dptr(depth), _lib.dptr(normal), _lib.dptr(albedo), _lib.dptr(rough),
            int(rough.shape[1]), _lib.dptr(fresnel), _lib.dptr(acc), n, K, float(acc_mask_threshold),
            _lib.dptr(rescale), _lib.dptr(u, dtype=torch.float64), _lib.dptr(dirs), _lib.dptr(T),
            _lib.dptr(pos, torch.int32), *tail, _lib.stream_ptr()), "tir_indirect_sample"))
    m = int(list_o.shape[0])
    t_last, acc_s, depth_s = march_list(tensoIR, list_o, list_d)
    hit = torch.empty(n, K, dtype=torch.int32, device=dev)
    hit_rays = torch.empty(cap, 6, device=dev)
    xn = torch.empty(cap, 3, device=dev)
    w = torch.empty(cap, device=dev)
    nbytes = C.c_int64(0)
    _lib.check(lib.tir_indirect_hits_work_size(n, K, C.byref(nbytes)), "tir_indirect_hits_work_size")
    work = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    aabb = (C.c_float * 6)(*tensoIR.aabb[0].tolist(), *tensoIR.invaabbSize.tolist())
    count_h = torch.zeros(1, dtype=torch.int64, device=dev)
    # an empty list has no rows to point at; tir_indirect_hits never reads them but takes non-null pointers
    rows_o, rows_d = (list_o, list_d) if m else (t_last, t_last)
    _lib.check(lib.tir_indirect_hits(n, K, _lib.dptr(pos, torch.int32), _lib.dptr(rows_o), _lib.dptr(rows_d),
                                     _lib.dptr(t_last), _lib.dptr(acc_s), _lib.dptr(depth_s),
                                     vis_kind(vis_equation), aabb, _lib.dptr(hit_rays), _lib.dptr(xn),
                                     _lib.dptr(w), _lib.dptr(hit, torch.int32), cap, _lib.dptr(count_h, torch.int64),
                                     _lib.dptr(work, torch.uint8), nbytes.value, _lib.stream_ptr()),
               "tir_indirect_hits")
    m_h = int(count_h.item())                      # sizes the material query and the secondary light
    return dict(dirs=dirs, T=T, pos=pos, list_o=list_o, list_d=list_d, t_last=t_last[:m], acc=acc_s[:m],
                depth=depth_s[:m], hit=hit, rays=hit_rays[:m_h], xn=xn[:m_h], w=w[:m_h])


def secondary_radiance(tensoIR, envs, L, hits, mats, rescale, Lo, h0, u2, vis_equation):
    """Lo[:, h0:h0+m] ([L, m_h, 3]) of the hits h0.. of ``hits`` for up to RELIGHT_MAX_LIGHTS maps: tir_relight_sample
    and the march from the hits (u2 [L, m, S2] fp64), then tir_indirect_radiance."""
    lib = _lib.load()
    m, S2 = int(u2.shape[1]), int(u2.shape[2])
    dev = Lo.device
    normal, albedo, rough, fresnel = (t[h0:h0 + m] for t in mats)
    rays = hits["rays"][h0:h0 + m]
    bins, pos, vis = relight_visibility(tensoIR, envs, L, rays, torch.zeros(m, device=dev), normal,
                                        torch.ones(m, device=dev), u2, S2, 0.5, vis_equation, ordered=True)
    _lib.check(lib.tir_indirect_radiance(envs, L, _lib.dptr(rays), _lib.dptr(normal), _lib.dptr(albedo),
                                         _lib.dptr(rough), int(rough.shape[1]), _lib.dptr(fresnel), m, S2,
                                         _lib.dptr(rescale), _lib.dptr(bins, torch.int32), _lib.dptr(pos, torch.int32),
                                         _lib.dptr(vis), vis_kind(vis_equation), _lib.dptr(Lo),
                                         int(Lo.shape[1]), int(h0), _lib.stream_ptr()), "tir_indirect_radiance")


@torch.no_grad()
def relight_chunk_indirect(tensoIR, envir_light, light_names, rays, maps, rescale_value, u, gen, *,
                           indirect_samples=16, indirect_light_samples=32, material=None, acc_mask_threshold=0.5,
                           vis_equation='nerv', out=None, row0=0, tables=None, indirect_out=None):
    """relight_chunk_fused (relighting.py) with one bounce of indirect light, under the same contract: ``maps`` =
    (depth, normal, albedo, roughness, fresnel, acc) of the primary render of ``rays``, ``u`` [L, n, S] fp64 direct
    uniforms.  ``gen``: the torch.Generator of the indirect draws, on the rays' device.  K = ``indirect_samples``
    directions per hit, S2 = ``indirect_light_samples`` light samples per secondary hit.  ``material``: a callable
    points [m,3] -> (normal, albedo, rough [m,1], fresnel); None is point_materials.  ``indirect_out`` [L, R, 3]
    receives the un-toned indirect term at rows row0.. (0 on rows without a secondary hit).
    -> (with_bg, without_bg) [L, n, 3], as relight_chunk_fused."""
    kind = vis_kind(vis_equation)
    K, S2 = int(indirect_samples), int(indirect_light_samples)
    if not (1 <= K <= 1024 and 1 <= S2 <= 1024):
        raise ValueError(f"indirect_samples and indirect_light_samples must be in [1, 1024], got {K}, {S2}")
    dev = rays.device
    L, n = len(light_names), int(rays.shape[0])
    rays, (depth, normal, albedo, rough, fresnel, acc) = chunk_inputs(rays, maps)
    if u.dim() != 3 or tuple(u.shape[:2]) != (L, n) or u.dtype != torch.float64:
        raise ValueError(f"u must be float64 [{L}, {n}, S], got {u.dtype} {tuple(u.shape)}")
    S = int(u.shape[2])
    u = u.to(dev).contiguous()
    if out is None:
        out = (torch.empty(L, n, 3, device=dev), torch.empty(L, n, 3, device=dev))
        row0 = 0
    with_bg, without_bg = out
    if n == 0 or L == 0:
        return with_bg[:, row0:row0 + n], without_bg[:, row0:row0 + n]
    envs, keep = tables if tables is not None else env_tables(envir_light, light_names)
    resc = rescale3(rescale_value, dev)
    thr = float(acc_mask_threshold)

    # the map-independent half: one secondary march and one material query for every map
    u_ind = torch.rand(n, K, 2, generator=gen, device=dev, dtype=torch.float64)
    hits = secondary_hits(tensoIR, rays, depth, normal, albedo, rough, fresnel, acc, resc, u_ind, thr, vis_equation)
    m_h = int(hits["rays"].shape[0])
    Lo = torch.zeros(L, max(m_h, 1), 3, device=dev)
    if m_h > 0:
        x = hits["rays"][:, :3]
        mats = material(x) if material is not None else point_materials(tensoIR, x, hits["xn"])
        mats = tuple(t.detach().float().reshape(m_h, -1).contiguous() for t in mats)
        # sub-lists of hits, so that the light samples of a sub-list (L * m * S2) stay within the direct ones (L * n * S)
        step = max(1, (n * S) // S2)
        for h0 in range(0, m_h, step):
            m = min(step, m_h - h0)
            u2 = torch.rand(L, m, S2, generator=gen, device=dev, dtype=torch.float64)
            for g, Lg, eg in env_groups(envs, L):
                secondary_radiance(tensoIR, eg, Lg, hits, mats, resc, Lo[g:g + Lg], h0, u2[g:g + Lg], vis_equation)

    lib = _lib.load()
    for g, Lg, eg in env_groups(envs, L):
        bins, pos, vis = relight_visibility(tensoIR, eg, Lg, rays, depth, normal, acc, u[g:g + Lg], S, thr,
                                            vis_equation, ordered=True)
        ind = indirect_out[g:g + Lg] if indirect_out is not None else None
        _lib.check(lib.tir_indirect_shade(eg, Lg, _lib.dptr(rays), _lib.dptr(normal), _lib.dptr(albedo),
                                          _lib.dptr(rough), int(rough.shape[1]), _lib.dptr(fresnel), _lib.dptr(acc), n,
                                          S, thr, _lib.dptr(resc), _lib.dptr(bins, torch.int32),
                                          _lib.dptr(pos, torch.int32), _lib.dptr(vis), kind, K,
                                          _lib.dptr(hits["T"]), _lib.dptr(hits["hit"], torch.int32),
                                          _lib.dptr(hits["w"]), _lib.dptr(Lo[g:g + Lg]), m_h,
                                          _lib.dptr(with_bg[g:g + Lg]), _lib.dptr(without_bg[g:g + Lg]),
                                          _lib.dptr(ind, allow_none=True),
                                          int(with_bg.shape[1]), int(row0), _lib.stream_ptr()), "tir_indirect_shade")
    del keep
    return with_bg[:, row0:row0 + n], without_bg[:, row0:row0 + n]
