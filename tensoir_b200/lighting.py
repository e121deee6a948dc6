"""Relight a trained model under analytic lights: directional, point and spot lights with marched shadows.

A rig is a dict of setups; a setup is what an environment map is to relight() (tensoir_b200.relighting): one image per
view.  It holds 1 to TIR_LIGHTS_MAX lights and a background colour.  Per chunk of primary rays the tir_lights_sample
kernel (csrc/tir_lights.cu, semantics in include/tensoir_b200.h) turns (surface hit, light, area sample) into shadow
rays, the existing density march gives their transmittance, and tir_lights_shade sums the lights' contributions,
tone-maps and composites.  A light without extent casts a hard shadow from one shadow ray per hit; a light with an
angular radius (directional) or a sphere radius (point, spot) is sampled ``samples`` times for a soft one.

Rigs are read from JSON (``load_rig``) of the form::

    {"noon": {"lights": [{"type": "directional", "direction": [0.2, 0.1, 1.0], "irradiance": [3.0, 3.0, 2.8],
                          "angular_radius_deg": 0.27, "samples": 16}]},
     "lamp": {"background": [0, 0, 0],
              "lights": [{"type": "point", "position": [2.5, 0, 2], "intensity": [40, 36, 30], "radius": 0.15,
                          "samples": 64},
                         {"type": "spot", "position": [-3, -3, 3], "target": [0, 0, 0], "intensity": 60,
                          "inner_deg": 10, "outer_deg": 18}]}}

Point and spot lights must lie outside the model's aabb, sphere included (``check_outside``).  The march takes one far
for all rays; a shadow ray that starts inside the convex box and aims at a light outside it leaves the box before it
reaches the light and never re-enters, so what lies past the light is never counted and the march is exact.
"""
from __future__ import annotations

import dataclasses
import json
import math
import os

import numpy as np
import torch

from . import _lib, ops
from . import relighting as R
from .editing import _NAME, _numbers

SHADOW_NEAR = 0.05                         # relight()'s second_near
SHADOW_STEP = (1.5 - 0.05) / 95            # relight()'s sample spacing: 96 samples over [0.05, 1.5]
SEED = 20211202                            # the reference scripts' seed
_KEYS = {"directional": {"type", "direction", "irradiance", "angular_radius_deg", "samples"},
         "point": {"type", "position", "intensity", "radius", "samples"},
         "spot": {"type", "position", "intensity", "radius", "samples", "target", "inner_deg", "outer_deg"}}


@dataclasses.dataclass(frozen=True)
class Light:
    """One light as the kernels take it (TirLight): ``kind`` 'directional', 'point' or 'spot'; ``direction`` unit,
    towards a directional light or along a spot's axis; ``power`` rgb irradiance (directional) or intensity;
    ``extent`` tan of the angular radius (directional) or the sphere radius; ``samples`` 1 when there is no extent."""
    kind: str
    power: tuple
    direction: tuple = (0.0, 0.0, 1.0)
    position: tuple = (0.0, 0.0, 0.0)
    extent: float = 0.0
    cos_inner: float = 1.0
    cos_outer: float = 1.0
    samples: int = 1


@dataclasses.dataclass(frozen=True)
class Setup:
    lights: tuple
    background: tuple = (1.0, 1.0, 1.0)


def _unit(v, what):
    n = math.sqrt(sum(x * x for x in v))
    if not n > 0:
        raise ValueError(f"{what}: zero length")
    return tuple(x / n for x in v)


def _rgb(v, what):
    v = _numbers(v, what, (3,)) if isinstance(v, (list, tuple)) else (_numbers(v, what, ()),) * 3
    if min(v) < 0:
        raise ValueError(f"{what}: negative value in {v}")
    return v


def _scalar(d, key, what, default=0.0):
    v = _numbers(d.get(key, default), f"{what} {key}", ())
    if v < 0:
        raise ValueError(f"{what} {key}: negative value {v}")
    return v


def parse_light(d, what="light"):
    """One light object of a rig file -> Light.  ``what`` names it in the ValueError of a malformed one."""
    if isinstance(d, Light):
        return d
    if not isinstance(d, dict):
        raise ValueError(f"{what}: expected an object, got {d!r}")
    kind = d.get("type")
    if kind not in _KEYS:
        raise ValueError(f"{what}: type must be one of {sorted(_KEYS)}, got {kind!r}")
    unknown = sorted(set(d) - _KEYS[kind])
    if unknown:
        raise ValueError(f"{what}: unknown field(s) {unknown} for a {kind} light; known: {sorted(_KEYS[kind])}")
    samples = d.get("samples", 1)
    if isinstance(samples, bool) or not isinstance(samples, int) or not 1 <= samples <= _lib.LIGHT_SAMPLES_MAX:
        raise ValueError(f"{what} samples: expected an integer in [1, {_lib.LIGHT_SAMPLES_MAX}], got {samples!r}")
    try:
        if kind == "directional":
            for k in ("direction", "irradiance"):
                if k not in d:
                    raise ValueError(f"missing {k}")
            ang = _scalar(d, "angular_radius_deg", "")
            if ang > 30:
                raise ValueError(f"angular_radius_deg {ang} above 30")
            ext = math.tan(math.radians(ang))
            return Light(kind, _rgb(d["irradiance"], "irradiance"),
                         direction=_unit(_numbers(d["direction"], "direction", (3,)), "direction"), extent=ext,
                         samples=samples if ext > 0 else 1)
        for k in ("position", "intensity") + (("target", "inner_deg", "outer_deg") if kind == "spot" else ()):
            if k not in d:
                raise ValueError(f"missing {k}")
        pos = _numbers(d["position"], "position", (3,))
        ext = _scalar(d, "radius", "")
        kw = {}
        if kind == "spot":
            inner, outer = _scalar(d, "inner_deg", ""), _scalar(d, "outer_deg", "")
            if not inner <= outer < 90:
                raise ValueError(f"need 0 <= inner_deg <= outer_deg < 90, got {inner}, {outer}")
            target = _numbers(d["target"], "target", (3,))
            kw = dict(direction=_unit(tuple(t - p for t, p in zip(target, pos)), "target - position"),
                      cos_inner=math.cos(math.radians(inner)), cos_outer=math.cos(math.radians(outer)))
        return Light(kind, _rgb(d["intensity"], "intensity"), position=pos, extent=ext,
                     samples=samples if ext > 0 else 1, **kw)
    except ValueError as e:
        raise ValueError(f"{what}: {e}") from None


def load_rig(src):
    """The setups of a rig: a JSON file (path), a JSON string or the mapping such a file holds,
    {setup name: {"lights": [light, ...], "background": [r, g, b]}} -> {name: Setup} in the given order.  Raises
    ValueError, naming the setup and the light index, for an unknown field, a wrong shape, a negative or non-finite
    number, a zero direction, more than TIR_LIGHTS_MAX lights or none, or a name that is not a plain directory name."""
    if isinstance(src, os.PathLike) or (isinstance(src, str) and not src.lstrip().startswith("{")):
        with open(src) as f:
            src = json.load(f)
    elif isinstance(src, str):
        src = json.loads(src)
    if not isinstance(src, dict):
        raise ValueError(f"a rig must map setup names to setups, got {type(src).__name__}")
    out = {}
    for name, s in src.items():
        if not isinstance(name, str) or not _NAME.fullmatch(name) or name in (".", ".."):
            raise ValueError(f"setup name {name!r} is not a plain directory name ([A-Za-z0-9][A-Za-z0-9_.-]*)")
        if isinstance(s, Setup):
            out[name] = s
            continue
        if not isinstance(s, dict) or set(s) - {"lights", "background"}:
            raise ValueError(f"setup {name!r}: expected an object with 'lights' and optionally 'background'")
        lights = s.get("lights")
        if not isinstance(lights, (list, tuple)) or not lights:
            raise ValueError(f"setup {name!r}: expected a non-empty list of lights")
        if len(lights) > _lib.LIGHTS_MAX:
            raise ValueError(f"setup {name!r}: {len(lights)} lights, at most {_lib.LIGHTS_MAX}")
        bg = _numbers(s.get("background", (1.0, 1.0, 1.0)), f"setup {name!r} background", (3,))
        if not all(0 <= c <= 1 for c in bg):
            raise ValueError(f"setup {name!r} background: {bg} outside [0, 1]")
        out[name] = Setup(tuple(parse_light(d, f"setup {name!r} light {k}") for k, d in enumerate(lights)), bg)
    if not out:
        raise ValueError("a rig needs at least one setup")
    return out


def olat_rig(n):
    """The light-stage sweep: n setups olat_000.., each one hard directional light of unit irradiance, on a Fibonacci
    sphere (tensorbase.fibonacci_sphere)."""
    from .tensorbase import fibonacci_sphere
    if n < 2:
        raise ValueError(f"an OLAT sweep needs at least 2 lights, got {n}")
    return {f"olat_{k:03d}": Setup((Light("directional", (1.0, 1.0, 1.0), direction=_unit(tuple(d), "direction")),))
            for k, d in enumerate(fibonacci_sphere(n).tolist())}


def check_outside(rig, aabb):
    """Raise ValueError, naming the light, unless every point and spot light of ``rig`` clears ``aabb`` ([2,3]: lower
    and upper corner) by more than its radius."""
    lo, hi = (np.asarray(c, dtype=np.float64) for c in torch.as_tensor(aabb).detach().cpu().tolist())
    for name, setup in rig.items():
        for k, l in enumerate(setup.lights):
            if l.kind == "directional":
                continue
            p = np.asarray(l.position)
            gap = np.linalg.norm(np.maximum(np.maximum(lo - p, p - hi), 0.0))
            if not gap > l.extent:
                raise ValueError(f"setup {name!r} light {k}: a {l.kind} light at {l.position} with radius {l.extent} "
                                 f"does not clear the model's aabb {lo.tolist()} .. {hi.tolist()}; lights must lie "
                                 f"outside it")


def light_table(setup):
    """ctypes array of TirLight for a Setup."""
    arr = (_lib.TirLight * max(len(setup.lights), 1))()
    kinds = {"directional": _lib.LIGHT_DIRECTIONAL, "point": _lib.LIGHT_POINT, "spot": _lib.LIGHT_SPOT}
    for k, l in enumerate(setup.lights):
        t = arr[k]
        t.type, t.n_samples = kinds[l.kind], l.samples
        t.dir[:], t.pos[:], t.power[:] = l.direction, l.position, l.power
        t.extent, t.cos_inner, t.cos_outer = l.extent, l.cos_inner, l.cos_outer
    return arr


def slots_per_ray(setup):
    return sum(l.samples for l in setup.lights)


def shadow_table(shadow_far, device):
    """z values of the shadow march: relight()'s near and sample spacing, out to at least ``shadow_far``.
    shadow_far = 1.5 gives relight()'s own 96-sample table."""
    n = math.ceil((float(shadow_far) - SHADOW_NEAR) / SHADOW_STEP - 1e-6) + 1
    if n < 2:
        raise ValueError(f"shadow_far must exceed {SHADOW_NEAR}, got {shadow_far}")
    return ops.equal_z_table(n, SHADOW_NEAR, SHADOW_NEAR + (n - 1) * SHADOW_STEP, device)


def default_shadow_far(tensoIR):
    """The aabb diagonal: no shadow caster inside the box is further from a receiver."""
    aabb = tensoIR.aabb.detach().double()
    return float((aabb[1] - aabb[0]).norm())


def _uniforms(slots, device, generator=None):
    """The uniform draws of one (chunk, setup): [slots, 2] fp64 in [0, 1).  Called in view-then-chunk-then-setup
    order."""
    return torch.rand(slots, 2, device=device, dtype=torch.float64, generator=generator)


def rig_sample(setup, rays, depth, normal, acc, u, acc_mask_threshold, ordered=False):
    """tir_lights_sample on contiguous fp32 device tensors (u fp64 [slots, 2]) -> (L, falloff, pos, list_o, list_d)
    with the list cut to its length, which is the one host read of the chunk.  ``ordered``: the list in slot order
    (relighting.slot_order)."""
    lib = _lib.load()
    dev = rays.device
    n = int(rays.shape[0])
    slots = n * slots_per_ray(setup)
    if tuple(u.shape) != (slots, 2) or u.dtype != torch.float64:
        raise ValueError(f"u must be float64 [{slots}, 2], got {u.dtype} {tuple(u.shape)}")
    u = u.to(dev).contiguous()
    L = torch.empty(slots, 3, device=dev)
    falloff = torch.empty(slots, device=dev)
    pos = torch.empty(slots, dtype=torch.int32, device=dev)
    list_o, list_d = R.append_list(
        slots, dev, "shadow-ray list", pos if ordered else None,
        lambda *tail: _lib.check(lib.tir_lights_sample(
            light_table(setup), len(setup.lights), _lib.dptr(rays), _lib.dptr(depth), _lib.dptr(normal),
            _lib.dptr(acc), n, float(acc_mask_threshold), _lib.dptr(u, torch.float64), _lib.dptr(L),
            _lib.dptr(falloff), _lib.dptr(pos, torch.int32), *tail, _lib.stream_ptr()), "tir_lights_sample"))
    return L, falloff, pos, list_o, list_d


def rig_visibility(tensoIR, setup, rays, depth, normal, acc, u, acc_mask_threshold, vis_equation, z_table,
                   ordered=False):
    """The material-independent half of relight_chunk_rig -> (L, falloff, pos, vis), what rig_shade reads.
    ``ordered``: march the list in slot order (relighting.slot_order)."""
    L, falloff, pos, list_o, list_d = rig_sample(setup, rays, depth, normal, acc, u, acc_mask_threshold, ordered)
    return L, falloff, pos, R.march_list(tensoIR, list_o, list_d, vis_equation, z_table)


def rig_shade(setup, rays, normal, albedo, rough, fresnel, acc, acc_mask_threshold, rescale_value, visibility,
              vis_equation, out, row0):
    """tir_lights_shade of the chunk's rows into out = (with_bg, without_bg, linear or None), [R, 3] maps, at rows
    row0.., with ``visibility`` = rig_visibility's result for the same setup, rays and maps."""
    lib = _lib.load()
    L, falloff, pos, vis = visibility
    with_bg, without_bg, linear = out
    dev = rays.device
    resc = R.rescale3(rescale_value, dev)
    bg = torch.tensor(setup.background, dtype=torch.float32, device=dev)
    assert with_bg.is_contiguous() and without_bg.is_contiguous() and (linear is None or linear.is_contiguous())
    _lib.check(lib.tir_lights_shade(light_table(setup), len(setup.lights), _lib.dptr(rays), _lib.dptr(normal),
                                    _lib.dptr(albedo), _lib.dptr(rough), int(rough.shape[1]), _lib.dptr(fresnel),
                                    _lib.dptr(acc), int(rays.shape[0]), float(acc_mask_threshold), _lib.dptr(resc),
                                    _lib.dptr(bg), _lib.dptr(L), _lib.dptr(falloff), _lib.dptr(pos, torch.int32),
                                    _lib.dptr(vis), R.vis_kind(vis_equation), _lib.dptr(with_bg),
                                    _lib.dptr(without_bg), _lib.dptr(linear, allow_none=True),
                                    int(with_bg.shape[0]), int(row0), _lib.stream_ptr()), "tir_lights_shade")


@torch.no_grad()
def relight_chunk_rig(tensoIR, setup, rays, maps, rescale_value, u, acc_mask_threshold=0.5, vis_equation='nerv',
                      shadow_far=None, out=None, row0=0):
    """One chunk of primary rays under one Setup, as relight_chunk_fused is for environment maps.  ``maps`` = (depth,
    normal, albedo, roughness [n,1] or [n,3], fresnel, acc) of the primary render of ``rays``; ``u`` [n * slots_per_ray,
    2] fp64 uniforms.  ``shadow_far``: how far a shadow ray is marched, default the aabb diagonal, or a z table from
    shadow_table.  -> (with_bg, without_bg, linear) [n, 3]; with ``out`` = three [R, 3] device maps the rows go to
    out[k][row0:row0+n] and views of them are returned."""
    R.vis_kind(vis_equation)
    n = int(rays.shape[0])
    rays, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(rays, maps)
    dev = rays.device
    if out is None:
        out, row0 = tuple(torch.empty(n, 3, device=dev) for _ in range(3)), 0
    if n:
        z = shadow_far if torch.is_tensor(shadow_far) else shadow_table(
            default_shadow_far(tensoIR) if shadow_far is None else shadow_far, dev)
        vis = rig_visibility(tensoIR, setup, rays, depth, normal, acc, u, acc_mask_threshold, vis_equation, z)
        rig_shade(setup, rays, normal, albedo, rough, fresnel, acc, acc_mask_threshold, rescale_value, vis,
                  vis_equation, out, row0)
    return tuple(None if o is None else o[row0:row0 + n] for o in out)


@torch.no_grad()
def relight_rig(dataset, args, rig, tensoIR=None):
    """relight()'s loop (tensoir_b200.relighting) under the setups of ``rig`` (as load_rig takes it).  ``dataset``
    follows relight()'s item contract (only rays, and what compute_rescale_ratio reads, are used); ``args`` needs ckpt
    (when ``tensoIR`` is None), geo_buffer_path and batch_size, and may carry acc_mask_threshold, vis_equation,
    render_video, seed, shadow_far (default: the aabb diagonal) and save_linear.  Per view it writes
    {geo_buffer_path}/{split}_{idx:03d}/relighting_with_bg/{setup}.png and relighting_without_bg/{setup}.png, with
    save_linear also relighting_linear/{setup}.hdr (the un-toned sum); per setup the video {geo_buffer_path}/{setup}.mp4
    when imageio is installed.  There are no metrics: an invented light has no ground truth."""
    from .evaluation import compute_rescale_ratio
    from .relight import write_hdr
    rig = load_rig(rig)
    tensoIR, device = R._model(args, tensoIR)
    if tensoIR is None:
        return
    check_outside(rig, tensoIR.aabb)
    thr = float(getattr(args, "acc_mask_threshold", R.SCRIPT_DEFAULTS["acc_mask_threshold"]))
    vis_eq = getattr(args, "vis_equation", R.SCRIPT_DEFAULTS["vis_equation"])
    R.vis_kind(vis_eq)
    save_linear = bool(getattr(args, "save_linear", False))
    far = getattr(args, "shadow_far", None)
    z_table = shadow_table(default_shadow_far(tensoIR) if far is None else far, device)
    gen = torch.Generator(device).manual_seed(int(getattr(args, "seed", SEED)))
    W, H = dataset.img_wh
    _, rescale_value = compute_rescale_ratio(tensoIR, dataset)
    rescale_value = rescale_value.to(device)
    names = list(rig)
    gp = args.geo_buffer_path
    for idx in range(len(dataset)):
        view_dir = os.path.join(gp, f'{dataset.split}_{idx:0>3d}')
        frame_rays = dataset[idx]['rays'].squeeze(0).to(device)
        n_pix = frame_rays.shape[0]
        with_map, without_map, linear_map = (torch.empty(len(names), n_pix, 3, device=device) for _ in range(3))
        for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(tensoIR, frame_rays,
                                                                                           args.batch_size):
            for k, name in enumerate(names):
                u = _uniforms((e - s) * slots_per_ray(rig[name]), device, gen)
                relight_chunk_rig(tensoIR, rig[name], frame_rays[s:e], (depth, normal, albedo, rough, fresnel, acc),
                                  rescale_value, u, thr, vis_eq, z_table,
                                  out=(with_map[k], without_map[k], linear_map[k]), row0=s)
        R._write_pairs(view_dir, names, H, W, with_map, without_map)
        if save_linear:
            os.makedirs(os.path.join(view_dir, 'relighting_linear'), exist_ok=True)
            lin = linear_map.reshape(len(names), H, W, 3).cpu().numpy()
            for k, name in enumerate(names):
                write_hdr(os.path.join(view_dir, 'relighting_linear', f'{name}.hdr'), lin[k])
    if getattr(args, "render_video", R.SCRIPT_DEFAULTS["render_video"]):
        for name in names:
            R._video(os.path.join(gp, f'{name}.mp4'), gp, dataset.split, len(dataset),
                     os.path.join('relighting_with_bg', f'{name}.png'))
