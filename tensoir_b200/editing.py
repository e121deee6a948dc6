"""Material editing: relight a trained model with edited albedo, roughness and fresnel under environment maps.

An edit is a list of rules (``MaterialEdit``).  A rule selects surface points by an axis-aligned box and / or a key
colour of the unedited albedo, and sets or scales albedo, roughness and fresnel there; the tir_material_edit kernel
(csrc/tir_edit.cu, semantics in include/tensoir_b200.h) applies a rule table to a chunk of points.

``relight_edited`` is relight()'s loop (tensoir_b200.relighting) with several material variants per view.  Shading is
the only part of the relighting pass that reads the materials: per chunk, the light samples and the visibility march
run once and every variant is one edit call plus one shade call on the same samples.  So a variant costs a small part
of a view, and the difference between two variants' images holds no Monte-Carlo noise.  The ``original`` variant is
the empty edit; its relit images are the bits relight() writes under the same uniforms.

Edits are read from JSON (``load_edits``) of the form::

    {"red_plate": [{"aabb": [[-1, -1, -1], [1, 1, -0.6]], "albedo_set": [0.8, 0.1, 0.1], "roughness_set": 0.2}],
     "shiny": [{"roughness_mul": 0.5, "fresnel_set": 0.5}]}
"""
from __future__ import annotations

import dataclasses
import json
import math
import os
import re

import numpy as np
import torch

from . import _lib
from . import relighting as R

ORIGINAL = "original"          # the reserved name of the unedited variant
_NAME = re.compile(r"[A-Za-z0-9][A-Za-z0-9_.-]*")


@dataclasses.dataclass(frozen=True)
class MaterialEdit:
    """One rule.  It selects the points inside ``aabb`` ((lo xyz), (hi xyz), inclusive) whose unedited scaled albedo is
    within ``key_tol`` (max over channels) of ``key``; each condition is optional, and a rule with none selects every
    surface point.  On them it sets or multiplies albedo (3 values, or 1 for all channels), roughness (1 value) and
    fresnel (3 values or 1); at most one of set / mul per quantity.  Results are clamped to [0, 1], roughness to the
    model's [0.09, 0.99]."""
    aabb: tuple | None = None
    key: tuple | None = None
    key_tol: float = 0.05
    albedo_set: tuple | None = None
    albedo_mul: tuple | None = None
    roughness_set: float | None = None
    roughness_mul: float | None = None
    fresnel_set: tuple | None = None
    fresnel_mul: tuple | None = None

    def __post_init__(self):
        put = lambda k, v: object.__setattr__(self, k, v)  # noqa: E731
        if self.aabb is not None:
            box = _numbers(self.aabb, "aabb", (2, 3))
            if any(box[0][c] > box[1][c] for c in range(3)):
                raise ValueError(f"aabb: lower corner {box[0]} above upper corner {box[1]}")
            put("aabb", box)
        if self.key is not None:
            put("key", _numbers(self.key, "key", (3,)))
        put("key_tol", _numbers(self.key_tol, "key_tol", ()))
        if self.key_tol < 0:
            raise ValueError(f"key_tol must be >= 0, got {self.key_tol}")
        for q in ("albedo", "fresnel"):
            for op in ("set", "mul"):
                v = getattr(self, f"{q}_{op}")
                if v is not None:
                    three = isinstance(v, (list, tuple))
                    put(f"{q}_{op}", _numbers(v, f"{q}_{op}", (3,)) if three else (_numbers(v, f"{q}_{op}", ()),) * 3)
        for op in ("set", "mul"):
            v = getattr(self, f"roughness_{op}")
            if v is not None:
                put(f"roughness_{op}", _numbers(v, f"roughness_{op}", ()))
        for q in ("albedo", "roughness", "fresnel"):
            if getattr(self, f"{q}_set") is not None and getattr(self, f"{q}_mul") is not None:
                raise ValueError(f"a rule may not both set and multiply {q}")


def _numbers(v, what, shape):
    """v as finite floats of ``shape``: () a float, (3,) a tuple, (2, 3) a tuple of tuples.  Raises ValueError
    otherwise."""
    if shape == ():
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
            raise ValueError(f"{what}: expected a finite number, got {v!r}")
        return float(v)
    if not isinstance(v, (list, tuple)) or len(v) != shape[0]:
        raise ValueError(f"{what}: expected {shape[0]} entries, got {v!r}")
    return tuple(_numbers(x, what + "[]", shape[1:]) for x in v)


def load_edits(src):
    """The material variants of a JSON file (path) or of the mapping such a file holds:
    {variant name: [rule, ...]} with each rule a dict of MaterialEdit's fields (or a MaterialEdit)
    -> {name: [MaterialEdit, ...]} in the given order.  Raises ValueError for an unknown field, set and mul on one
    quantity, a wrong shape, more than TIR_EDIT_MAX_RULES rules or none, or a name that is not a plain directory name or
    is the reserved 'original'."""
    if isinstance(src, (str, os.PathLike)):
        with open(src) as f:
            src = json.load(f)
    if not isinstance(src, dict):
        raise ValueError(f"edits must map variant names to rule lists, got {type(src).__name__}")
    fields = {f.name for f in dataclasses.fields(MaterialEdit)}
    out = {}
    for name, rules in src.items():
        if not isinstance(name, str) or not _NAME.fullmatch(name) or name in (".", ".."):
            raise ValueError(f"variant name {name!r} is not a plain directory name ([A-Za-z0-9][A-Za-z0-9_.-]*)")
        if name == ORIGINAL:
            raise ValueError(f"the variant name {ORIGINAL!r} is reserved for the unedited materials")
        if not isinstance(rules, (list, tuple)) or not rules:
            raise ValueError(f"variant {name!r}: expected a non-empty list of rules")
        if len(rules) > _lib.EDIT_MAX_RULES:
            raise ValueError(f"variant {name!r}: {len(rules)} rules, at most {_lib.EDIT_MAX_RULES}")
        parsed = []
        for r in rules:
            if isinstance(r, MaterialEdit):
                parsed.append(r)
                continue
            if not isinstance(r, dict):
                raise ValueError(f"variant {name!r}: a rule must be an object, got {r!r}")
            unknown = sorted(set(r) - fields)
            if unknown:
                raise ValueError(f"variant {name!r}: unknown rule field(s) {unknown}; known: {sorted(fields)}")
            parsed.append(MaterialEdit(**r))
        out[name] = parsed
    return out


def rule_table(edits):
    """ctypes array of TirEditRule for a list of MaterialEdit."""
    if len(edits) > _lib.EDIT_MAX_RULES:
        raise ValueError(f"{len(edits)} rules, at most {_lib.EDIT_MAX_RULES}")
    arr = (_lib.TirEditRule * max(len(edits), 1))()
    for k, e in enumerate(edits):
        r = arr[k]
        if e.aabb is not None:
            r.flags |= _lib.EDIT_BOX
            r.box_lo[:], r.box_hi[:] = e.aabb
        if e.key is not None:
            r.flags |= _lib.EDIT_KEY
            r.key[:] = e.key
            r.key_tol = e.key_tol
        for q, field in (("albedo", "albedo"), ("roughness", "rough"), ("fresnel", "fresnel")):
            for op, code in (("set", _lib.EDIT_SET), ("mul", _lib.EDIT_MUL)):
                v = getattr(e, f"{q}_{op}")
                if v is None:
                    continue
                setattr(r, f"{field}_op", code)
                if q == "roughness":
                    r.rough = v
                else:
                    getattr(r, field)[:] = v
    return arr


@torch.no_grad()
def edit_materials(maps, edits, scale, thr, points=None, rays=None):
    """One tir_material_edit call.  ``maps`` = (depth, normal, albedo [n,3], roughness [n,1] or [n,3], fresnel [n,3],
    acc [n]) as relight_chunk_fused takes them (depth and normal may be None with ``points``); the points are ``points``
    [n,3], or the surface points of ``rays`` [n,6] at depth.  ``scale``: the albedo scale, one value or three; ``thr``:
    rows with acc > thr are edited.  -> (albedo_out = edited albedo*scale [n,3], roughness [n, stride], fresnel [n,3],
    sel [n] int32 with bit k set where rule k selected the row)."""
    if (points is None) == (rays is None):
        raise ValueError("pass exactly one of points and rays")
    depth, normal, albedo, rough, fresnel, acc = maps
    f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
    albedo, fresnel, acc = f32(albedo), f32(fresnel), f32(acc).reshape(-1)
    n = int(acc.shape[0])
    rough = f32(rough)
    rough = rough[:, None].contiguous() if rough.dim() == 1 else rough
    dev = albedo.device
    if points is not None:
        points, depth_p, rays_p = f32(points), None, None
    else:
        points, depth_p, rays_p = None, f32(depth).reshape(-1), f32(rays)
    scale = R.rescale3(scale, dev)
    table = rule_table(edits)
    a_out, r_out, f_out = torch.empty_like(albedo), torch.empty_like(rough), torch.empty_like(fresnel)
    sel = torch.empty(n, dtype=torch.int32, device=dev)
    lib = _lib.load()
    opt = lambda t: _lib.dptr(t, allow_none=True)  # noqa: E731
    _lib.check(lib.tir_material_edit(table, len(edits), opt(rays_p), opt(depth_p), opt(points), _lib.dptr(albedo),
                                     _lib.dptr(rough), int(rough.shape[1]), _lib.dptr(fresnel), _lib.dptr(acc), n,
                                     float(thr), _lib.dptr(scale), _lib.dptr(a_out), _lib.dptr(r_out),
                                     _lib.dptr(f_out), _lib.dptr(sel, torch.int32), _lib.stream_ptr()),
               "tir_material_edit")
    return a_out, r_out, f_out, sel


@torch.no_grad()
def relight_edited(dataset, args, variants, tensoIR=None, include_original=True):
    """relight() (tensoir_b200.relighting) for several material variants at once: ``variants`` as load_edits takes it
    (its output, a dict or a JSON path); with ``include_original`` the unedited 'original' variant comes first.  The
    dataset contract, ``args`` (ckpt when tensoIR is None, hdrdir, geo_buffer_path, batch_size, the script flags of
    SCRIPT_DEFAULTS), the uniform draws (one _uniforms call per chunk) and the chunking are relight()'s.  Per view and
    variant it writes under {geo_buffer_path}/{split}_{idx:03d}/{variant}/: relighting_with_bg/{light}.png,
    relighting_without_bg/{light}.png, albedo_gamma_corrected.png (the edited scaled albedo, alpha the thresholded acc),
    roughness.png and selection.png (255 where a rule selected the pixel); when the items carry rgbs, also
    relighting_without_bg/relight_psnr.txt per view and {geo_buffer_path}/{variant}/relight_psnr.txt for the run, in
    relight()'s format.  Per-light videos go to {geo_buffer_path}/{variant}/video_{with,without}_bg/ when imageio is
    installed.  Returns {variant: {light: [PSNR per view]}} (empty lists without rgbs)."""
    from .relight import Environment_Light
    from .evaluation import compute_rescale_ratio
    runs = ([(ORIGINAL, [])] if include_original else []) + list(load_edits(variants).items())
    if not runs:
        raise ValueError("no variant to render")
    opt = {k: getattr(args, k, v) for k, v in R.SCRIPT_DEFAULTS.items()}
    tensoIR, device = R._model(args, tensoIR)
    if tensoIR is None:
        return None
    W, H = dataset.img_wh
    if H < 11 or W < 11:
        raise ValueError(f"SSIM needs images of at least 11x11 pixels, got {W}x{H}")
    names = list(dataset.light_names)
    L, S = len(names), R.NUM_SAMPLES
    thr = float(opt["acc_mask_threshold"])
    vis_eq = opt["vis_equation"]
    R.vis_kind(vis_eq)
    envir_light = Environment_Light(args.hdrdir, device=device)
    envs, keep = R.env_tables(envir_light, names)
    _, rescale_value = compute_rescale_ratio(tensoIR, dataset)
    scale = R.rescale3(rescale_value, device)
    ones = torch.ones(3, device=device)
    gp = args.geo_buffer_path
    V = len(runs)
    metrics = {v: R._new_metrics(names) for v, _ in runs}
    for idx in range(len(dataset)):
        view_dir = os.path.join(gp, f'{dataset.split}_{idx:0>3d}')
        item = dataset[idx]
        frame_rays = item['rays'].squeeze(0).to(device)
        n_pix = frame_rays.shape[0]
        with_map = torch.empty(V, L, n_pix, 3, device=device)
        without_map = torch.empty(V, L, n_pix, 3, device=device)
        alb = torch.empty(V, n_pix, 3, device=device)
        sel = torch.empty(V, n_pix, dtype=torch.int32, device=device)
        acc_v, rgh = torch.empty(n_pix, device=device), None
        for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(tensoIR, frame_rays,
                                                                                           args.batch_size):
            rays, maps = R.chunk_inputs(frame_rays[s:e], (depth, normal, albedo, rough, fresnel, acc))
            depth, normal, albedo, rough, fresnel, acc = maps
            acc_v[s:e] = acc
            if rgh is None:
                rgh = torch.empty(V, n_pix, rough.shape[1], device=device)
            u = R._uniforms(L, e - s, S, device)
            if tuple(u.shape) != (L, e - s, S) or u.dtype != torch.float64:
                raise ValueError(f"u must be float64 [{L}, {e - s}, {S}], got {u.dtype} {tuple(u.shape)}")
            u = u.to(device).contiguous()
            groups = list(R.env_groups(envs, L))
            vis = [R.relight_visibility(tensoIR, eg, Lg, rays, depth, normal, acc, u[g:g + Lg].contiguous(), S, thr,
                                        vis_eq) for g, Lg, eg in groups]
            for v, (_, rules) in enumerate(runs):
                a_o, r_o, f_o, sel_o = edit_materials(maps, rules, scale, thr, rays=rays)
                alb[v, s:e], rgh[v, s:e], sel[v, s:e] = a_o, r_o, sel_o
                for (g, Lg, eg), vs in zip(groups, vis):
                    R.relight_shade(eg, Lg, rays, normal, a_o, r_o, f_o, acc, S, thr, ones, vs, vis_eq,
                                    (with_map[v, g:g + Lg], without_map[v, g:g + Lg]), s)

        acc_u8 = R._acc_u8(acc_v, H, W)
        gt_rgb = item['rgbs'].squeeze(0).reshape(L, H * W, 3).to(device) if 'rgbs' in item else None
        for v, (vname, _) in enumerate(runs):
            d = os.path.join(view_dir, vname)
            R._write_pairs(d, names, H, W, with_map[v], without_map[v])
            gamma_u8 = (alb[v].clamp(0.0, 1.0).reshape(H, W, 3) ** (1 / 2.2) * 255).to(torch.uint8).cpu().numpy()
            R._imwrite(os.path.join(d, 'albedo_gamma_corrected.png'), np.concatenate([gamma_u8, acc_u8], axis=2))
            r = rgh[v].reshape(H, W, -1).expand(-1, -1, 3) * 255
            R._imwrite(os.path.join(d, 'roughness.png'),
                       np.concatenate([r.cpu().numpy(), acc_u8], axis=2).astype('uint8'))
            R._imwrite(os.path.join(d, 'selection.png'), ((sel[v] != 0).to(torch.uint8) * 255).reshape(H, W).cpu()
                       .numpy())
            if gt_rgb is None:
                continue
            R._view_metrics(metrics[vname], names, without_map[v], gt_rgb, H, W, device,
                            os.path.join(d, 'relighting_without_bg', 'relight_psnr.txt'))
    del keep

    for vname, _ in runs:
        m = metrics[vname]
        vdir = os.path.join(gp, vname)
        os.makedirs(vdir, exist_ok=True)
        if len(dataset) and all(m["psnr"][n] for n in names):
            R._run_metrics(m, names, os.path.join(vdir, 'relight_psnr.txt'))
        if opt["render_video"]:
            for sub in ('without_bg', 'with_bg'):
                vp = os.path.join(vdir, f'video_{sub}')
                os.makedirs(vp, exist_ok=True)
                for name in names:
                    R._video(os.path.join(vp, f'{name}_video.mp4'), gp, dataset.split, len(dataset),
                             os.path.join(vname, f'relighting_{sub}', f'{name}.png'))
    return {v: metrics[v]["psnr"] for v, _ in runs}
