"""Relit camera-path videos: a trained model rendered from cameras that belong to no dataset, under environment maps
rotated per frame, over the map it is lit by, with a ground plane that catches the object's shadow.

Conventions (include/tensoir_b200.h, "camera-path frames"):
  * cameras are camera-to-world matrices [4,4] in the OpenCV convention (x right, y down, z forward), as the datasets
    and ops.generate_rays use;
  * a map rotated by ``a`` degrees turns about world +z with R(a) of the reference's light_rotation
    (``rotation_matrix``): the radiance arriving from world direction w is E(w @ R(a)).  So a rotation of 90 lights the
    object as the reference's rgba_{light}_090 images are lit.

Per frame and chunk of primary rays the object is shaded by the environment-map pass (relighting.relight_visibility
in slot order, then relighting.relight_shade) with the maps' direction tables rotated (``rotated_env_tables``); with a
ground, tir_ground_sample turns each ground pixel's light samples into shadow rays towards the model's occupied box,
the density march gives their visibility, and tir_path_composite writes the frame: the rotated background, darkened by
the ground's shadow ratio, under the object.  The estimators that look texels up by direction (MIS and the indirect
bounce) are not rotated by a direction table and are rejected.

Under a rig of analytic lights (lighting.load_rig) instead of maps, each setup is turned per frame (``rotated_setup``:
a light authored at direction d or position p ends up at R(a) d, R(a) p, as a map's texel does), the object is shaded
by lighting.rig_visibility in slot order and lighting.rig_shade, and with a ground tir_ground_lights_sample and
tir_path_lights_composite do for the lights' samples what the two map entries do for texels, over the setup's
background colour (``render_rig_frame``).
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import json
import math
import os

import numpy as np
import torch

from . import _lib, ops
from . import relighting as R
from .light_fit import srgb_to_linear
from .lighting import (SEED, SHADOW_NEAR, SHADOW_STEP, check_outside, default_shadow_far, light_table, load_rig,
                       rig_shade, rig_visibility, shadow_table, slots_per_ray)
from .lighting import _uniforms as rig_uniforms

NUM_SAMPLES = R.NUM_SAMPLES


# ---- cameras --------------------------------------------------------------------------------------------------------

def look_at(position, target):
    """OpenCV c2w [4,4] (float64 numpy) of a camera at ``position`` looking at ``target``, world +z up in the image."""
    pos, tgt = np.asarray(position, np.float64), np.asarray(target, np.float64)
    fwd = tgt - pos
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, np.array([0.0, 0.0, 1.0]))
    if not np.linalg.norm(right) > 1e-9:
        raise ValueError("a camera looking straight up or down has no image-up direction")
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, pos
    return c2w


def orbit_poses(n, radius, elevation_deg, target, start_deg=0.0, turns=1.0):
    """n cameras on a circle of ``radius`` around ``target`` at ``elevation_deg`` above its horizontal plane, azimuth
    start_deg + 360 * turns * k / n (counter-clockwise about +z), each looking at the target with world +z up in the
    image -> float32 OpenCV c2w [n,4,4]."""
    if int(n) != n or n < 1:
        raise ValueError(f"an orbit needs at least one frame, got {n!r}")
    if not radius > 0 or not abs(elevation_deg) < 90:
        raise ValueError(f"need radius > 0 and |elevation| < 90 degrees, got {radius}, {elevation_deg}")
    tgt = np.asarray(target, np.float64).reshape(3)
    el = math.radians(elevation_deg)
    out = []
    for k in range(int(n)):
        az = math.radians(start_deg + 360.0 * turns * k / n)
        pos = tgt + radius * np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
        out.append(look_at(pos, tgt))
    return torch.tensor(np.stack(out), dtype=torch.float32)


def orbit_of(c2w, target):
    """(radius, elevation_deg, azimuth_deg) of the camera c2w [4,4] seen from ``target``: orbit_poses' parameters of
    the orbit through it."""
    v = np.asarray(torch.as_tensor(c2w).double().cpu())[:3, 3] - np.asarray(target, np.float64).reshape(3)
    r = float(np.linalg.norm(v))
    return r, math.degrees(math.asin(v[2] / r)), math.degrees(math.atan2(v[1], v[0]))


def load_poses(path):
    """A JSON file holding a list of 4x4 camera-to-world matrices in the OpenCV convention -> float32 [n,4,4].
    ValueError for anything else."""
    with open(path) as f:
        data = json.load(f)
    try:
        poses = torch.tensor(data, dtype=torch.float64)
    except (TypeError, ValueError) as e:
        raise ValueError(f"{path}: expected a list of 4x4 matrices ({e})") from None
    if poses.ndim != 3 or poses.shape[1:] != (4, 4) or poses.shape[0] < 1 or not torch.isfinite(poses).all():
        raise ValueError(f"{path}: expected a non-empty list of finite 4x4 matrices, got shape {tuple(poses.shape)}")
    return poses.float()


def parse_rotation(spec):
    """``a0:a1`` in degrees -> (a0, a1).  ValueError for anything else."""
    parts = str(spec).split(":")
    try:
        if len(parts) != 2:
            raise ValueError
        a0, a1 = float(parts[0]), float(parts[1])
    except ValueError:
        raise ValueError(f"env_rotation must be a0:a1 in degrees, got {spec!r}") from None
    if not (math.isfinite(a0) and math.isfinite(a1)):
        raise ValueError(f"env_rotation must be finite, got {spec!r}")
    return a0, a1


def parse_path(spec):
    """``orbit``, ``test`` or the path of a poses JSON file -> ('orbit' | 'test' | 'file', spec).  ValueError for an
    empty spec or a file that does not exist."""
    if spec in ("orbit", "test"):
        return spec, spec
    if not spec or not os.path.isfile(spec):
        raise ValueError(f"path must be orbit, test or a poses JSON file, got {spec!r}")
    return "file", spec


def frame_angles(n, rotation):
    """The map rotation of each of n frames: linear from a0 at frame 0 towards a1 at frame n, as the orbit's azimuth
    steps, so that a0:a0+360 with an orbit of one turn keeps the background still (a turntable)."""
    a0, a1 = rotation
    return [a0 + (a1 - a0) * f / n for f in range(n)]


# ---- rotated maps ---------------------------------------------------------------------------------------------------

def rotation_matrix(angle_deg):
    """R(a) of the reference's light_rotation (tensorBase_rotated_lights.py:478-488), float32 [3,3]."""
    a = torch.tensor(float(angle_deg) / 180 * torch.pi).to(torch.float32)
    return torch.tensor([[torch.cos(a), -torch.sin(a), 0], [torch.sin(a), torch.cos(a), 0], [0, 0, 1]]).to(
        torch.float32)


def rotated_env_tables(envir_light, light_names, angle):
    """relighting.env_tables of the maps rotated by ``angle`` degrees: the same array with every dir table replaced
    by dir @ R(angle)^T, so that the sample taken from texel k arrives from the world direction whose lookup
    w @ R(angle) is texel k.  -> (array, tensors it points into)."""
    arr, keep = R.env_tables(envir_light, light_names)
    rot = rotation_matrix(angle)
    for k, name in enumerate(light_names):
        d = envir_light.hdr_dir[name].reshape(-1, 3).float()
        r = rot.to(d.device)
        # (R d)_j in fp32 elementwise (no matmul precision mode applies), exact for the identity
        d = (d[:, 0:1] * r[:, 0] + d[:, 1:2] * r[:, 1] + d[:, 2:3] * r[:, 2]).contiguous()
        keep.append(d)
        arr[k].dir = _lib.dptr(d)
    return arr, keep


# ---- rotated light rigs ---------------------------------------------------------------------------------------------

def rotated_setup(setup, angle):
    """The lighting.Setup ``setup`` turned by ``angle`` degrees about +z under the maps' convention: a map rotated by a
    gives E(w @ R(a)), so a light authored at direction d (position p, spot axis) ends up at R(a) d (column vector),
    R = rotation_matrix(angle).  The product is taken in float64 from R's fp32 entries and rounded to fp32 once, by
    lighting.light_table, with no renormalisation; angle 0 leaves every value as it is."""
    m = rotation_matrix(angle).double().tolist()

    def turn(v):
        return tuple(m[i][0] * v[0] + m[i][1] * v[1] + m[i][2] * v[2] for i in range(3))

    return dataclasses.replace(setup, lights=tuple(dataclasses.replace(l, direction=turn(l.direction),
                                                                       position=turn(l.position))
                                                   for l in setup.lights))


def frame_rigs(rig, angles, aabb):
    """The rig ``rig`` ({name: Setup}) turned by each frame's angle -> a list of {name: Setup}, one per frame.
    ValueError naming the frame, the setup and the light when a turned point or spot light does not clear ``aabb``
    (lighting.check_outside): a box that is not a cube can swallow a light that clears it unturned."""
    out = []
    for f, a in enumerate(angles):
        turned = {name: rotated_setup(s, a) for name, s in rig.items()}
        try:
            check_outside(turned, aabb)
        except ValueError as e:
            raise ValueError(f"frame {f} (rotation {a:g} degrees): {e}") from None
        out.append(turned)
    return out


# ---- the ground -----------------------------------------------------------------------------------------------------

def ground_box(tensoIR):
    """The box a shadow ray must meet to be occluded: the world-space occupied-cell box of the model's alpha mask
    (TirField.occ_lo / occ_hi, empty when no cell is occupied), or the aabb without an alpha mask -> (lo, hi) lists."""
    f = ops.device_field(tensoIR).refresh(tensoIR)
    if getattr(tensoIR, "alphaMask", None) is None:
        return [float(x) for x in f.aabb_lo], [float(x) for x in f.aabb_hi]
    return [float(x) for x in f.occ_lo], [float(x) for x in f.occ_hi]


def default_ground_z(tensoIR):
    """The bottom of the occupied-cell box (of the aabb when the box is empty)."""
    lo, hi = ground_box(tensoIR)
    return lo[2] if lo[2] <= hi[2] else float(tensoIR.aabb[0, 2])


def ground_table(box, device):
    """The ground's shadow march: lighting.shadow_table out to SHADOW_NEAR plus the box diagonal."""
    lo, hi = np.asarray(box[0]), np.asarray(box[1])
    diag = float(np.linalg.norm(hi - lo)) if (lo <= hi).all() else 0.0
    return shadow_table(SHADOW_NEAR + max(diag, SHADOW_STEP), device)   # an empty box's table is never read


def _c3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


def ground_visibility(tensoIR, envs, L, rays, ground_z, box, u, num_samples, vis_equation, z_table):
    """tir_ground_sample for up to RELIGHT_MAX_LIGHTS maps, the list in slot order, and its march.  Inputs are
    contiguous device tensors (rays fp32 [n,6], u fp64 [L,n,S]).  -> (bins, pos, vis), what path_composite reads."""
    lib = _lib.load()
    dev = rays.device
    n, S = int(rays.shape[0]), int(num_samples)
    bins = torch.empty(L, n, S, dtype=torch.int32, device=dev)
    pos = torch.empty(L, n, S, dtype=torch.int32, device=dev)
    list_o, list_d = R.append_list(
        L * n * S, dev, "ground visibility list", pos,
        lambda *tail: _lib.check(lib.tir_ground_sample(
            envs, L, _lib.dptr(rays), n, float(ground_z), _c3(box[0]), _c3(box[1]), S,
            _lib.dptr(u, dtype=torch.float64), _lib.dptr(bins, torch.int32), _lib.dptr(pos, torch.int32), *tail,
            _lib.stream_ptr()), "tir_ground_sample"))
    return bins, pos, R.march_list(tensoIR, list_o, list_d, vis_equation, z_table)


def path_composite(envs, L, rays, acc, angle, ground_z, visibility, num_samples, vis_equation, out, row0,
                   shadow=None):
    """tir_path_composite of the chunk's rows into out = (with_bg, without_bg) [L, R, 3] at rows row0.. (without_bg
    already shaded), with the background rotated by ``angle`` degrees.  ``ground_z`` None: no ground (``visibility``
    unused); else ``visibility`` = ground_visibility's result.  ``shadow`` [L, R, 3] or None gets the shadow ratio."""
    lib = _lib.load()
    with_bg, without_bg = out
    assert with_bg.is_contiguous() and without_bg.is_contiguous()
    rot = (C.c_float * 9)(*rotation_matrix(angle).reshape(-1).tolist())
    gz = float("nan") if ground_z is None else float(ground_z)
    bins, pos, vis = visibility if ground_z is not None else (None, None, None)
    _lib.check(lib.tir_path_composite(envs, L, _lib.dptr(rays), _lib.dptr(acc), int(rays.shape[0]), rot, gz,
                                      _lib.dptr(bins, torch.int32, allow_none=True),
                                      _lib.dptr(pos, torch.int32, allow_none=True), _lib.dptr(vis, allow_none=True),
                                      R.vis_kind(vis_equation), int(num_samples), _lib.dptr(without_bg),
                                      _lib.dptr(with_bg), _lib.dptr(shadow, allow_none=True), int(with_bg.shape[1]),
                                      int(row0), _lib.stream_ptr()), "tir_path_composite")


def rig_ground_box(tensoIR):
    """ground_box clipped to the model's aabb: the box of tir_ground_lights_sample.  Every point or spot light lies
    outside the aabb (lighting.check_outside), so a shadow ray that enters this box before the light also leaves it
    before the light, which makes the distance cull exact (DESIGN §3.8)."""
    lo, hi = ground_box(tensoIR)
    a_lo, a_hi = tensoIR.aabb.detach().float().cpu().tolist()
    return [max(x, y) for x, y in zip(lo, a_lo)], [min(x, y) for x, y in zip(hi, a_hi)]


def ground_lights_visibility(tensoIR, setup, rays, ground_z, box, u, vis_equation, z_table):
    """tir_ground_lights_sample for one lighting.Setup, the list in slot order, and its march.  Inputs are contiguous
    device tensors (rays fp32 [n,6], u fp64 [n * slots_per_ray, 2]).  -> (g, pos, vis), what path_lights_composite
    reads."""
    lib = _lib.load()
    dev = rays.device
    n = int(rays.shape[0])
    slots = n * slots_per_ray(setup)
    if tuple(u.shape) != (slots, 2) or u.dtype != torch.float64:
        raise ValueError(f"u must be float64 [{slots}, 2], got {u.dtype} {tuple(u.shape)}")
    g = torch.empty(slots, device=dev)
    pos = torch.empty(slots, dtype=torch.int32, device=dev)
    list_o, list_d = R.append_list(
        slots, dev, "ground visibility list", pos,
        lambda *tail: _lib.check(lib.tir_ground_lights_sample(
            light_table(setup), len(setup.lights), _lib.dptr(rays), n, float(ground_z), _c3(box[0]), _c3(box[1]),
            _lib.dptr(u, torch.float64), _lib.dptr(g), _lib.dptr(pos, torch.int32), *tail, _lib.stream_ptr()),
            "tir_ground_lights_sample"))
    return g, pos, R.march_list(tensoIR, list_o, list_d, vis_equation, z_table)


def path_lights_composite(setup, rays, acc, ground_z, visibility, vis_equation, out, row0, shadow=None):
    """tir_path_lights_composite of the chunk's rows into out = (with_bg, without_bg) [R, 3] at rows row0..
    (without_bg already shaded by lighting.rig_shade) over the setup's background colour, which the shadow darkens in
    linear light (light_fit.srgb_to_linear, float64).  ``ground_z`` None: no ground (``visibility`` unused); else
    ``visibility`` = ground_lights_visibility's result.  ``shadow`` [R, 3] or None gets the shadow ratio."""
    lib = _lib.load()
    with_bg, without_bg = out
    assert with_bg.is_contiguous() and without_bg.is_contiguous()
    gz = float("nan") if ground_z is None else float(ground_z)
    g, pos, vis = visibility if ground_z is not None else (None, None, None)
    _lib.check(lib.tir_path_lights_composite(
        light_table(setup), len(setup.lights), _lib.dptr(rays), _lib.dptr(acc), int(rays.shape[0]), gz,
        _c3(setup.background), _c3(srgb_to_linear(list(setup.background)).tolist()), _lib.dptr(g, allow_none=True),
        _lib.dptr(pos, torch.int32, allow_none=True), _lib.dptr(vis, allow_none=True), R.vis_kind(vis_equation),
        _lib.dptr(without_bg), _lib.dptr(with_bg), _lib.dptr(shadow, allow_none=True), int(with_bg.shape[0]),
        int(row0), _lib.stream_ptr()), "tir_path_lights_composite")


def check_estimator(args):
    """ValueError unless ``args`` asks for the environment-map pass's own estimator: MIS and the indirect bounce look
    texels up by direction, which a rotated direction table does not rotate."""
    sampling, _ = R.mis_options(args)
    if sampling == "mis":
        raise ValueError("camera paths rotate the maps' direction tables, which MIS does not read: "
                         "use sampling='light'")
    if int(getattr(args, "indirect_samples", 0) or 0) > 0:
        raise ValueError("camera paths rotate the maps' direction tables, which the indirect bounce does not read: "
                         "use indirect_samples=0")


def path_maps(args, tensoIR, dataset):
    """The maps of a path and the albedo scale they are shaded with -> (Environment_Light, names, rescale [3]).
    ``args.light == 'learned'``: the model's own lights (mesh.light_envmaps), one map per rotation named
    learned_{rotation}, scale 1; else the .hdr maps of args.hdrdir with compute_rescale_ratio, as relight() does."""
    from .evaluation import compute_rescale_ratio
    from .relight import Environment_Light
    dev = tensoIR.aabb.device
    light = getattr(args, "light", None)
    if light not in (None, "learned"):
        raise ValueError(f"light must be 'learned' or unset (the maps of hdrdir), got {light!r}")
    if light == "learned":
        if getattr(tensoIR, "general_lights", False):
            raise ValueError("a general multi-light checkpoint does not store its lights: fit environment maps with "
                             "tools/fit_lights.py and pass the directory of its .hdr output as hdrdir")
        from .mesh import light_envmaps
        maps = light_envmaps(tensoIR).cpu().numpy()
        names = [f"learned_{int(r):03d}" for r in tensoIR.light_rotation]
        env = Environment_Light({n: maps[k] for k, n in enumerate(names)}, device=dev)
        return env, names, torch.ones(3, device=dev)
    env = Environment_Light(args.hdrdir, device=dev)
    _, rescale = compute_rescale_ratio(tensoIR, dataset)
    return env, list(env.hdr_rgbs), torch.as_tensor(rescale, dtype=torch.float32).to(dev)


def dataset_focal(dataset):
    """The pinhole focal length of ``dataset``'s views: its ``focal``, or, for a dataset without one (the relighting
    test set), the one its first view's rays were built with."""
    if getattr(dataset, "focal", None) is not None:
        return float(np.asarray(dataset.focal).reshape(-1)[0])
    W, _ = dataset.img_wh
    item = dataset[0]
    c2w = torch.as_tensor(item["c2w"]).double()
    d = item["rays"].reshape(-1, 6)[0, 3:].double() @ c2w[:3, :3]       # pixel (0, 0) in camera coordinates
    return float((0.5 - W / 2) * d[2] / d[0])


def dataset_poses(dataset):
    """The c2w [n,4,4] of ``dataset``'s views: its ``poses``, or the c2w of every item."""
    if getattr(dataset, "poses", None) is not None:
        return torch.as_tensor(np.asarray(dataset.poses), dtype=torch.float32).reshape(-1, 4, 4)
    return torch.stack([torch.as_tensor(dataset[i]["c2w"], dtype=torch.float32) for i in range(len(dataset))])


def frame_rays(c2w, W, H, focal, device):
    """The [H*W, 6] rays of camera c2w [4,4] through ops.generate_rays, with the pinhole of focal length ``focal``."""
    n = W * H
    cam_angle_x = 2.0 * math.atan(0.5 * W / float(focal))
    return ops.generate_rays(torch.as_tensor(c2w, dtype=torch.float32).reshape(1, 4, 4).to(device),
                             torch.zeros(n, dtype=torch.int32, device=device),
                             torch.arange(n, dtype=torch.int32, device=device), H, W, cam_angle_x)


@torch.no_grad()
def render_frame(tensoIR, env, names, rays_f, angle, rescale, batch_size, generator, seed, ground_z=None, box=None,
                 num_samples=NUM_SAMPLES, acc_mask_threshold=0.5, vis_equation="nerv", shadow=False, timer=None):
    """One frame of every map in ``names`` of ``env`` from the rays ``rays_f`` [n,6], the maps rotated by ``angle``.
    ``generator`` is re-seeded with ``seed`` first; per chunk the object's uniforms [L,n,S] are drawn, then, with a
    ground, the ground's.  ``box``: ground_box (default the model's).  ``timer(phase)``, when given, is called after
    each phase.  -> (with_bg, without_bg, shadow ratio or None) [L, n, 3]."""
    dev = rays_f.device
    L, n_pix, S = len(names), int(rays_f.shape[0]), int(num_samples)
    tick = timer or (lambda phase: None)
    envs, keep = rotated_env_tables(env, names, angle)
    if ground_z is not None:
        box = ground_box(tensoIR) if box is None else box
        z_table = ground_table(box, dev)
    generator.manual_seed(int(seed))
    with_map = torch.empty(L, n_pix, 3, device=dev)
    without_map = torch.empty(L, n_pix, 3, device=dev)
    shadow_map = torch.empty(L, n_pix, 3, device=dev) if shadow else None
    for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(tensoIR, rays_f, batch_size):
        rays, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(rays_f[s:e],
                                                                            (depth, normal, albedo, rough, fresnel,
                                                                             acc))
        tick("primary")
        n = e - s
        u = torch.rand(L, n, S, device=dev, dtype=torch.float64, generator=generator)
        ug = torch.rand(L, n, S, device=dev, dtype=torch.float64, generator=generator) if ground_z is not None else None
        for g, Lg, eg in R.env_groups(envs, L):
            vis = R.relight_visibility(tensoIR, eg, Lg, rays, depth, normal, acc, u[g:g + Lg], S, acc_mask_threshold,
                                       vis_equation, ordered=True)
            tick("object_visibility")
            R.relight_shade(eg, Lg, rays, normal, albedo, rough, fresnel, acc, S, acc_mask_threshold, rescale, vis,
                            vis_equation, (with_map[g:g + Lg], without_map[g:g + Lg]), s)
            tick("object_shade")
            gvis = None
            if ground_z is not None:
                gvis = ground_visibility(tensoIR, eg, Lg, rays, ground_z, box, ug[g:g + Lg], S, vis_equation, z_table)
                tick("ground")
            path_composite(eg, Lg, rays, acc, angle, ground_z, gvis, S, vis_equation,
                           (with_map[g:g + Lg], without_map[g:g + Lg]), s,
                           None if shadow_map is None else shadow_map[g:g + Lg])
            tick("composite")
    del keep
    return with_map, without_map, shadow_map


@torch.no_grad()
def render_rig_frame(tensoIR, rig, rays_f, rescale, batch_size, generator, seed, ground_z=None, box=None,
                     acc_mask_threshold=0.5, vis_equation="nerv", shadow_table_z=None, shadow=False, timer=None):
    """One frame of every setup of ``rig`` ({name: lighting.Setup}, already turned for the frame: frame_rigs) from
    the rays ``rays_f`` [n,6], as render_frame is for maps.  ``generator`` is re-seeded with ``seed`` first; per chunk
    and setup the object's uniforms [n * slots, 2] are drawn, then, with a ground, the ground's.  ``box``:
    rig_ground_box (default the model's).  ``shadow_table_z``: the object's shadow march (lighting.shadow_table,
    default out to the aabb diagonal).  ``timer(phase)`` as render_frame's.  -> (with_bg, without_bg, shadow ratio or
    None) [setups, n, 3]."""
    dev = rays_f.device
    names = list(rig)
    n_pix = int(rays_f.shape[0])
    tick = timer or (lambda phase: None)
    z_obj = shadow_table(default_shadow_far(tensoIR), dev) if shadow_table_z is None else shadow_table_z
    if ground_z is not None:
        box = rig_ground_box(tensoIR) if box is None else box
        z_ground = ground_table(box, dev)
    generator.manual_seed(int(seed))
    with_map = torch.empty(len(names), n_pix, 3, device=dev)
    without_map = torch.empty(len(names), n_pix, 3, device=dev)
    shadow_map = torch.empty(len(names), n_pix, 3, device=dev) if shadow else None
    for s, e, (_, depth, normal, albedo, rough, fresnel, acc, *_) in R._primary_chunks(tensoIR, rays_f, batch_size):
        rays, (depth, normal, albedo, rough, fresnel, acc) = R.chunk_inputs(rays_f[s:e],
                                                                            (depth, normal, albedo, rough, fresnel,
                                                                             acc))
        tick("primary")
        for k, name in enumerate(names):
            setup = rig[name]
            slots = (e - s) * slots_per_ray(setup)
            u = rig_uniforms(slots, dev, generator)
            ug = rig_uniforms(slots, dev, generator) if ground_z is not None else None
            vis = rig_visibility(tensoIR, setup, rays, depth, normal, acc, u, acc_mask_threshold, vis_equation, z_obj,
                                 ordered=True)
            tick("object_visibility")
            rig_shade(setup, rays, normal, albedo, rough, fresnel, acc, acc_mask_threshold, rescale, vis,
                      vis_equation, (with_map[k], without_map[k], None), s)
            tick("object_shade")
            gvis = None
            if ground_z is not None:
                gvis = ground_lights_visibility(tensoIR, setup, rays, ground_z, box, ug, vis_equation, z_ground)
                tick("ground")
            path_lights_composite(setup, rays, acc, ground_z, gvis, vis_equation, (with_map[k], without_map[k]), s,
                                  None if shadow_map is None else shadow_map[k])
            tick("composite")
    return with_map, without_map, shadow_map


def _write_frame(out, names, f, H, W, with_map, without_map):
    """{out}/{map}/with_bg/{f:04d}.png and without_bg/{f:04d}.png of [L, H*W, 3] maps (relighting._write_pairs'
    encoding)."""
    for sub, m in (("with_bg", with_map), ("without_bg", without_map)):
        u8 = (m * 255).to(torch.uint8).reshape(len(names), H, W, 3).cpu().numpy()
        for k, name in enumerate(names):
            d = os.path.join(out, name, sub)
            os.makedirs(d, exist_ok=True)
            R._imwrite(os.path.join(d, f"{f:04d}.png"), u8[k])


@torch.no_grad()
def render_path(dataset, args, poses, angles, tensoIR=None, ground_z=None, rig=None):
    """Render the cameras ``poses`` [F,4,4] (OpenCV c2w) with the maps rotated by ``angles`` [F] degrees.
    ``dataset`` gives img_wh and the focal length (dataset_focal) and, for the maps of args.hdrdir or a rig, what
    compute_rescale_ratio reads; ``args`` needs ckpt (when ``tensoIR`` is None), out and batch_size, and may carry
    hdrdir, light ('learned'), seed (lighting.SEED), acc_mask_threshold, vis_equation and render_video.  ``ground_z``: the height of the
    shadow-catching ground plane, True for the bottom of the occupied-cell box, None for no ground.
    Writes {out}/{map}/with_bg/{f:04d}.png and without_bg/{f:04d}.png per frame and, with imageio, {out}/{map}.mp4 of
    with_bg.  ``rig`` (whatever lighting.load_rig takes): light the frames with its setups instead, turned by
    ``angles`` (frame_rigs), over each setup's background colour, the albedo scaled by compute_rescale_ratio and the
    object's shadow rays marched to args.shadow_far (default the aabb diagonal); images go to {out}/{setup}/... and
    {out}/{setup}.mp4 and hdrdir is not read.  ValueError for MIS, indirect light, learned lights of a general
    multi-light model, a rig with light 'learned', or a turned light inside the aabb."""
    check_estimator(args)
    poses = torch.as_tensor(poses, dtype=torch.float32).reshape(-1, 4, 4)
    angles = [float(a) for a in angles]
    if len(angles) != poses.shape[0]:
        raise ValueError(f"{poses.shape[0]} poses but {len(angles)} angles")
    if rig is not None:
        if getattr(args, "light", None) is not None:
            raise ValueError(f"a rig lights the frames itself: light must be unset, got {args.light!r}")
        rig = load_rig(rig)
    tensoIR, device = R._model(args, tensoIR)
    if tensoIR is None:
        return
    thr = float(getattr(args, "acc_mask_threshold", R.SCRIPT_DEFAULTS["acc_mask_threshold"]))
    vis_eq = getattr(args, "vis_equation", R.SCRIPT_DEFAULTS["vis_equation"])
    R.vis_kind(vis_eq)
    if rig is None:
        env, names, rescale = path_maps(args, tensoIR, dataset)
    else:
        from .evaluation import compute_rescale_ratio
        rigs = frame_rigs(rig, angles, tensoIR.aabb)
        names = list(rig)
        far = getattr(args, "shadow_far", None)
        z_obj = shadow_table(default_shadow_far(tensoIR) if far is None else far, device)
        _, rescale = compute_rescale_ratio(tensoIR, dataset)
        rescale = torch.as_tensor(rescale, dtype=torch.float32).to(device)
    if ground_z is True:
        ground_z = default_ground_z(tensoIR)
    seed = getattr(args, "seed", None)
    seed = SEED if seed is None else int(seed)
    gen = torch.Generator(device)
    W, H = dataset.img_wh
    focal = dataset_focal(dataset)
    out = args.out
    box = None
    if ground_z is not None:
        box = ground_box(tensoIR) if rig is None else rig_ground_box(tensoIR)
    for f in range(poses.shape[0]):
        rays_f = frame_rays(poses[f], W, H, focal, device)
        if rig is None:
            with_map, without_map, _ = render_frame(tensoIR, env, names, rays_f, angles[f], rescale, args.batch_size,
                                                    gen, seed, ground_z, box, acc_mask_threshold=thr,
                                                    vis_equation=vis_eq)
        else:
            with_map, without_map, _ = render_rig_frame(tensoIR, rigs[f], rays_f, rescale, args.batch_size, gen, seed,
                                                        ground_z, box, acc_mask_threshold=thr, vis_equation=vis_eq,
                                                        shadow_table_z=z_obj)
        _write_frame(out, names, f, H, W, with_map, without_map)
    if getattr(args, "render_video", True):
        for name in names:
            R._mimsave(os.path.join(out, f"{name}.mp4"),
                       lambda name=name: [R._imread(os.path.join(out, name, "with_bg", f"{f:04d}.png"))
                                          for f in range(poses.shape[0])])
