"""Relighting evaluation: relight() of the reference's scripts/relight_importance.py (:30-340) with the same file layout,
text formats and metric definitions, on the fused relighting kernels (csrc/tir_relight.cu) and the pair-metric kernel
(csrc/tir_eval.cu, tir_eval_pairs).

Per view, the primary maps are rendered in ``args.batch_size`` chunks into device maps.  Each chunk makes one
relight_chunk_fused call for all environment maps: importance sampling, the cosine test and the visibility list in one
kernel, the existing density march on the list, then shading, tone mapping and background compositing in one kernel that
writes straight into the view's [L, H*W, 3] maps.  One tir_eval_pairs call per view gives the PSNR and SSIM of every
map.  uint8 images reach the host only to be written.

Differences from the reference, all deliberate:
  * light directions are drawn by inverse-CDF sampling of the same distribution as the reference's torch.multinomial
    (a different random stream); the uniforms come from ``_uniforms``;
  * PNGs are written with cv2 and decode to the arrays the reference hands to imageio;
  * the videos need ``imageio`` and LPIPS needs ``lpips``; without them the videos are skipped and LPIPS is nan.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, ops
from .evaluation import _lpips, compute_rescale_ratio, visualize_depth_numpy

NUM_SAMPLES = 512          # samples per surface point (relight_importance.py:119)

# flags relight_importance.py's __main__ sets on args (:355-365); read with getattr, these are the defaults
SCRIPT_DEFAULTS = dict(if_save_rgb=False, if_save_depth=False, if_save_acc=True, if_save_rgb_video=False,
                       if_save_relight_rgb=True, if_save_albedo=True, if_save_albedo_gamma_corrected=True,
                       acc_mask_threshold=0.5, if_render_normal=True, vis_equation='nerv', render_video=True)


def _uniforms(L, n, S, device):
    """The uniform draws of one chunk: [L, n, S] fp64 in [0, 1).  Called once per chunk, in view-then-chunk order."""
    return torch.rand(L, n, S, device=device, dtype=torch.float64)


def env_tables(envir_light, light_names):
    """ctypes array of TirEnvMap for ``light_names`` of an Environment_Light (tensoir_b200.relight), plus the tensors
    it points into (keep them alive while the array is in use)."""
    arr = (_lib.TirEnvMap * max(len(light_names), 1))()
    keep = []
    for k, name in enumerate(light_names):
        rgb = envir_light.hdr_rgbs[name]
        H, W = int(rgb.shape[0]), int(rgb.shape[1])
        t = (rgb.reshape(-1, 3).float().contiguous(), envir_light.hdr_dir[name].reshape(-1, 3).float().contiguous(),
             envir_light.hdr_pdf_return[name].reshape(-1).float().contiguous(),
             envir_light._cdf[name].reshape(-1).double().contiguous())
        keep += t
        arr[k].H, arr[k].W = H, W
        arr[k].rgb, arr[k].dir, arr[k].pdf_return = (_lib.dptr(x) for x in t[:3])
        arr[k].cdf = _lib.dptr(t[3], dtype=torch.float64)
    return arr, keep


def chunk_inputs(rays, maps):
    """rays and maps = (depth, normal, albedo, roughness, fresnel, acc) of a chunk as the relighting kernels take them:
    contiguous fp32, depth and acc [n], roughness [n, 1] or [n, 3]."""
    depth, normal, albedo, rough, fresnel, acc = maps
    f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
    rays, depth, normal, albedo, fresnel, acc = (f32(t) for t in (rays, depth.reshape(-1), normal, albedo, fresnel,
                                                                   acc.reshape(-1)))
    return rays, (depth, normal, albedo, f32(rough).reshape(rays.shape[0], -1), fresnel, acc)


def env_group(envs, g):
    """The TirEnvMap array ``envs`` from entry g on: the first map of a group of up to RELIGHT_MAX_LIGHTS."""
    return C.cast(C.byref(envs, g * C.sizeof(_lib.TirEnvMap)), C.POINTER(_lib.TirEnvMap))


def env_groups(envs, L):
    """The kernels take up to RELIGHT_MAX_LIGHTS maps per call: -> (g, Lg, env_group(envs, g)) of each group of the
    L maps of ``envs``, maps g..g+Lg-1."""
    G = _lib.RELIGHT_MAX_LIGHTS
    for g in range(0, L, G):
        yield g, min(G, L - g), env_group(envs, g)


def vis_kind(vis_equation):
    """relight()'s vis_equation as the kernels take it: 0 for 'nerv' (t_last), 1 for 'nerfactor' (1 - acc).
    ValueError for anything else."""
    if vis_equation not in ('nerv', 'nerfactor'):
        raise ValueError(vis_equation)
    return 0 if vis_equation == 'nerv' else 1


def rescale3(rescale_value, device):
    """An albedo scale of one value or three as the kernels take it: contiguous fp32 [3] on ``device``."""
    return torch.as_tensor(rescale_value, dtype=torch.float32).to(device).reshape(-1).expand(3).contiguous()


def relight_table(device):
    """relight()'s visibility march: 96 equal-z samples over [0.05, 1.5]."""
    return ops.equal_z_table(96, 0.05, 1.5, device)


@torch.no_grad()
def relight_chunk_fused(tensoIR, envir_light, light_names, rays, maps, rescale_value, u, num_samples=NUM_SAMPLES,
                        acc_mask_threshold=0.5, vis_equation='nerv', out=None, row0=0, tables=None):
    """The chunk body of relight() (relight_importance.py:99-181) for every map in ``light_names`` at once.
    ``maps`` = (depth, normal, albedo, roughness [n,1] or [n,3], fresnel, acc) of the primary render of ``rays``;
    ``u`` [L, n, num_samples] fp64 uniforms (rows of non-hit rays are ignored).  Draws nothing itself.
    -> (with_bg, without_bg) [L, n, 3]; with ``out`` = ([L, R, 3], [L, R, 3]) device maps the rows go to
    out[:, row0:row0+n] and views of them are returned."""
    vis_kind(vis_equation)
    dev = rays.device
    L, n, S = len(light_names), int(rays.shape[0]), int(num_samples)
    rays, (depth, normal, albedo, rough, fresnel, acc) = chunk_inputs(rays, maps)
    if tuple(u.shape) != (L, n, S) or u.dtype != torch.float64:
        raise ValueError(f"u must be float64 [{L}, {n}, {S}], got {u.dtype} {tuple(u.shape)}")
    u = u.to(dev).contiguous()
    if out is None:
        out = (torch.empty(L, n, 3, device=dev), torch.empty(L, n, 3, device=dev))
        row0 = 0
    with_bg, without_bg = out
    if n == 0 or L == 0:
        return with_bg[:, row0:row0 + n], without_bg[:, row0:row0 + n]
    envs, keep = tables if tables is not None else env_tables(envir_light, light_names)
    for g, Lg, eg in env_groups(envs, L):
        vis = relight_visibility(tensoIR, eg, Lg, rays, depth, normal, acc, u[g:g + Lg], S, acc_mask_threshold,
                                 vis_equation)
        relight_shade(eg, Lg, rays, normal, albedo, rough, fresnel, acc, S, acc_mask_threshold, rescale_value, vis,
                      vis_equation, (with_bg[g:g + Lg], without_bg[g:g + Lg]), row0)
    del keep
    return with_bg[:, row0:row0 + n], without_bg[:, row0:row0 + n]


def slot_order(pos, list_o, list_d):
    """Rewrite a list appended in warp-scheduling order into slot order, in place of pos: the density march's result
    for a ray can change in its last bits with the rays next to it in the list, so this makes the march, and what
    reads it, reproducible.  -> (list_o, list_d) of the marched rows."""
    sel = pos >= 0
    rows = pos[sel].long()
    pos[sel] = torch.arange(rows.numel(), dtype=pos.dtype, device=pos.device)
    return list_o[rows], list_d[rows]


def relight_visibility(tensoIR, envs, L, rays, depth, normal, acc, u, num_samples, acc_mask_threshold, vis_equation,
                       ordered=False):
    """The material-independent half of relight_chunk_fused for up to RELIGHT_MAX_LIGHTS maps (``envs``, L entries):
    tir_relight_sample, the read-back of the list length and the density march on the list.  Inputs are contiguous
    fp32 (u fp64 [L, n, S]) device tensors.  ``ordered``: march the list in slot order (slot_order).
    -> (bins, pos, vis), what relight_shade reads."""
    lib = _lib.load()
    dev = rays.device
    n, S = int(rays.shape[0]), int(num_samples)
    bins = torch.empty(L, n, S, dtype=torch.int32, device=dev)
    pos = torch.empty(L, n, S, dtype=torch.int32, device=dev)
    list_o, list_d = append_list(
        L * n * S, dev, "relight visibility list", pos if ordered else None,
        lambda *tail: _lib.check(lib.tir_relight_sample(
            envs, L, _lib.dptr(rays), _lib.dptr(depth), _lib.dptr(normal), _lib.dptr(acc), n, S,
            float(acc_mask_threshold), _lib.dptr(u, dtype=torch.float64), _lib.dptr(bins, torch.int32),
            _lib.dptr(pos, torch.int32), *tail, _lib.stream_ptr()), "tir_relight_sample"))
    return bins, pos, march_list(tensoIR, list_o, list_d, vis_equation)


def append_list(cap, device, what, pos, sample):
    """The visibility list of a tir_*_sample entry: allocates ``cap`` (origin, direction) rows, runs ``sample(list_o,
    list_d, capacity, count)`` with the entry's four trailing list arguments, and reads the list length back (the
    one host sync of the chunk; TirError naming ``what`` if it overflowed).  ``pos``: the entry's slot map, to put the
    list in slot order (slot_order, rewriting pos), or None to keep the append order.
    -> (list_o, list_d) cut to the list length."""
    list_o = torch.empty(cap, 3, device=device)
    list_d = torch.empty(cap, 3, device=device)
    count = torch.zeros(1, dtype=torch.int64, device=device)
    sample(_lib.dptr(list_o), _lib.dptr(list_d), cap, _lib.dptr(count, torch.int64))
    m = int(count.item())
    if m > cap:
        raise _lib.TirError(f"{what} overflow: {m} > {cap}")
    if pos is not None and m > 0:
        return slot_order(pos, list_o[:m], list_d[:m])
    return list_o[:m], list_d[:m]


def march_list(tensoIR, list_o, list_d, vis_equation=None, table=None):
    """The density march of append_list's rows with ``table`` (default relight_table).  -> the visibility per row the
    shade kernels read, by ``vis_equation`` (t_last for nerv, acc for nerfactor), or with vis_equation None all three
    outputs (t_last, acc, depth); a list without rows gives a zero [1] for each."""
    if list_o.shape[0] == 0:
        out = (torch.zeros(1, device=list_o.device),) * 3
    else:
        out = ops.march_density(tensoIR, list_o, list_d,
                                table=relight_table(list_o.device) if table is None else table,
                                counters=tensoIR.__dict__.get("_tir_counters"))
    if vis_equation is not None:
        return out[vis_kind(vis_equation)].contiguous()
    return tuple(t.contiguous() for t in out)


def relight_shade(envs, L, rays, normal, albedo, rough, fresnel, acc, num_samples, acc_mask_threshold, rescale_value,
                  visibility, vis_equation, out, row0):
    """The material half of relight_chunk_fused: tir_relight_shade of the chunk's rows into out = (with_bg, without_bg)
    [L, R, 3] at rows row0.., with ``visibility`` = relight_visibility's (bins, pos, vis) for the same envs, rays and
    maps.  rough is [n, 1] or [n, 3]; inputs are contiguous fp32 device tensors."""
    lib = _lib.load()
    bins, pos, vis = visibility
    with_bg, without_bg = out
    n, dev = int(rays.shape[0]), rays.device
    resc = rescale3(rescale_value, dev)
    assert with_bg.is_contiguous() and without_bg.is_contiguous()
    _lib.check(lib.tir_relight_shade(envs, L, _lib.dptr(rays), _lib.dptr(normal), _lib.dptr(albedo), _lib.dptr(rough),
                                     int(rough.shape[1]), _lib.dptr(fresnel), _lib.dptr(acc), n, int(num_samples),
                                     float(acc_mask_threshold), _lib.dptr(resc), _lib.dptr(bins, torch.int32),
                                     _lib.dptr(pos, torch.int32), _lib.dptr(vis), vis_kind(vis_equation),
                                     _lib.dptr(with_bg), _lib.dptr(without_bg),
                                     int(with_bg.shape[1]), int(row0), _lib.stream_ptr()), "tir_relight_shade")


def pair_metrics(a, b, H, W):
    """One tir_eval_pairs call: a, b [P, H*W, 3] (or [P, H, W, 3]) device images -> float64 device tensor [P, 2] of
    (squared-error sum over H*W*3, mean SSIM of utils.rgb_ssim)."""
    lib = _lib.load()
    P = int(a.shape[0])
    a = a.detach().float().reshape(P, -1).contiguous()
    b = b.detach().float().reshape(P, -1).to(a.device).contiguous()
    if H < 11 or W < 11:
        raise ValueError(f"SSIM needs images of at least 11x11 pixels, got {W}x{H}")
    n = C.c_int64(0)
    _lib.check(lib.tir_eval_pairs_work_size(P, int(H), int(W), C.byref(n)), "tir_eval_pairs_work_size")
    work = torch.empty(max(n.value, 1), dtype=torch.float64, device=a.device)
    out = torch.empty(max(P, 1), 2, dtype=torch.float64, device=a.device)
    _lib.check(lib.tir_eval_pairs(_lib.dptr(a), _lib.dptr(b), P, int(H), int(W), _lib.dptr(work, torch.float64),
                                  n.value, _lib.dptr(out, torch.float64), _lib.stream_ptr()), "tir_eval_pairs")
    return out[:P]


def _imwrite(path, img):
    """Write a uint8 image (H,W gray, H,W,3 RGB or H,W,4 RGBA) so that decoding the PNG gives back ``img``."""
    import cv2
    if img.ndim == 3:
        img = np.ascontiguousarray(img[..., [2, 1, 0, 3]] if img.shape[2] == 4 else img[..., ::-1])
    if not cv2.imwrite(path, img):
        raise OSError(f"could not write {path}")


def _imread(path):
    """imageio.v2.imread of a PNG this module wrote (RGB / RGBA channel order)."""
    import cv2
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img.ndim == 3:
        img = img[..., [2, 1, 0, 3]] if img.shape[2] == 4 else img[..., ::-1]
    return np.ascontiguousarray(img)


def _mimsave(path, frames):
    """imageio.mimsave of the frames (a list, or a callable returning it) when imageio is importable."""
    try:
        import imageio
    except ImportError:
        print(f"relighting: imageio is not installed, {path} is not written")
        return
    imageio.mimsave(path, np.stack(frames() if callable(frames) else frames), fps=24, macro_block_size=1)


def _load_model(args, device):
    from . import TensorVMSplit
    if not os.path.exists(args.ckpt):
        print('the checkpoint path for tensoIR does not exists!!!')
        return None
    ckpt = torch.load(args.ckpt, map_location=device, weights_only=False)
    kwargs = dict(ckpt['kwargs'])
    kwargs.update({'device': device})
    model = TensorVMSplit(**kwargs)       # a light_name_list kwarg selects the general multi-light variant
    model.load(ckpt)
    return model


def _model(args, tensoIR):
    """``tensoIR``, or the checkpoint args.ckpt loaded on cuda -> (model, its device); (None, None) without one."""
    if tensoIR is None:
        tensoIR = _load_model(args, torch.device("cuda"))
        if tensoIR is None:
            return None, None
    return tensoIR, tensoIR.device if hasattr(tensoIR, "device") else torch.device("cuda")


def _primary_chunks(tensoIR, frame_rays, batch_size):
    """The primary render of one view's rays in chunks of ``batch_size`` -> (s, e, outputs of the eval forward)."""
    n_pix = frame_rays.shape[0]
    light_idx = torch.zeros((n_pix, 1), dtype=torch.int32, device=frame_rays.device)
    for s in range(0, n_pix, batch_size):
        e = min(s + batch_size, n_pix)
        yield s, e, tensoIR(frame_rays[s:e], light_idx[s:e], is_train=False, white_bg=True, ndc_ray=False,
                            N_samples=-1)


def _write_pairs(view_dir, names, H, W, with_map, without_map):
    """{view_dir}/relighting_with_bg/{name}.png and relighting_without_bg/{name}.png of [L, H*W, 3] maps."""
    for sub, m in (('with_bg', with_map), ('without_bg', without_map)):
        os.makedirs(os.path.join(view_dir, f'relighting_{sub}'), exist_ok=True)
        u8 = (m * 255).to(torch.uint8).reshape(len(names), H, W, 3).cpu().numpy()
        for k, name in enumerate(names):
            _imwrite(os.path.join(view_dir, f'relighting_{sub}', f'{name}.png'), u8[k])


def _acc_u8(acc, H, W):
    """The alpha of the view's images: the reference's `acc_temp = acc_chunk[..., None]; acc_temp[acc_temp <= 0.9] = 0`
    (relight_importance.py:179-180) zeroes the primary acc in place -> uint8 [H, W, 1]."""
    acc_t = acc.reshape(-1).clone()
    acc_t[acc_t <= 0.9] = 0.0
    return (acc_t.reshape(H, W, 1) * 255).to(torch.uint8).cpu().numpy()


def _new_metrics(names):
    return {k: {n: [] for n in names} for k in ("psnr", "ssim", "alex", "vgg")}


def _view_metrics(m, names, without_map, gt_rgb, H, W, device, path):
    """PSNR, SSIM and LPIPS of each map of one view against its ground truth (:212-226), appended to ``m``
    (_new_metrics), and the view's relight_psnr.txt at ``path``."""
    met = pair_metrics(without_map, gt_rgb, H, W).cpu().numpy()
    for k, name in enumerate(names):
        m["psnr"][name].append(-10.0 * np.log(met[k, 0] / (H * W * 3)) / np.log(10.0))
        m["ssim"][name].append(float(met[k, 1]))
        img, gt_img = without_map[k].reshape(H, W, 3), gt_rgb[k].reshape(H, W, 3)
        m["alex"][name].append(_lpips(gt_img, img, 'alex', device))
        m["vgg"][name].append(_lpips(gt_img, img, 'vgg', device))
    with open(path, 'w') as f:
        for name in names:
            f.write(f'{name}: PNSR {m["psnr"][name][-1]}; SSIM {m["ssim"][name][-1]}; L_Alex {m["alex"][name][-1]}; '
                    f'L_VGG {m["vgg"][name][-1]}\n')


def _run_metrics(m, names, path):
    """The run's relight_psnr.txt: the mean of each metric of ``m`` over the views."""
    with open(path, 'w') as f:
        for name in names:
            f.write(f'{name}:  PSNR {np.mean(m["psnr"][name])}; SSIM {np.mean(m["ssim"][name])}; '
                    f'L_Alex {np.mean(m["alex"][name])}; L_VGG {np.mean(m["vgg"][name])}\n')


def _video(path, gp, split, n_views, rel):
    """The video of one image over the views: {gp}/{split}_{i:03d}/{rel} for i < n_views."""
    _mimsave(path, lambda: [_imread(os.path.join(gp, f'{split}_{i:0>3d}', rel)) for i in range(n_views)])


def mis_options(args):
    """relight()'s estimator options from ``args``: -> (sampling, brdf_samples).  ValueError for an unknown sampling,
    brdf_samples outside [0, NUM_SAMPLES - 1], or sampling 'mis' with indirect light."""
    sampling = getattr(args, "sampling", None) or "light"
    n_brdf = getattr(args, "brdf_samples", None)
    given = n_brdf is not None
    n_brdf = 128 if n_brdf is None else n_brdf
    if sampling not in ("light", "mis"):
        raise ValueError(f"sampling must be 'light' or 'mis', got {sampling!r}")
    if (given or sampling == "mis") and (isinstance(n_brdf, bool) or int(n_brdf) != n_brdf
                                         or not 0 <= n_brdf <= NUM_SAMPLES - 1):
        raise ValueError(f"brdf_samples must be an integer in [0, {NUM_SAMPLES - 1}], got {n_brdf!r}")
    if sampling == "mis" and int(getattr(args, "indirect_samples", 0) or 0) > 0:
        raise ValueError("sampling='mis' does not combine with indirect_samples > 0")
    return sampling, int(n_brdf)


@torch.no_grad()
def relight(dataset, args, tensoIR=None, *, rescale_value=None):
    """relight_importance.py:30-340.  ``dataset`` follows the reference relighting test set's item contract
    (rays, rgbs [L, H*W, 3], rgbs_mask, albedo, ...) with ``split`` and ``light_names``; ``args`` needs ckpt (when
    ``tensoIR`` is None), hdrdir, geo_buffer_path and batch_size; the script-only flags default to SCRIPT_DEFAULTS.
    ``rescale_value``: the albedo rescale ratio [3] to shade with; None computes it from ``dataset``
    (compute_rescale_ratio), as the reference does.
    Indirect light (indirect.py) is read from ``args`` too: ``indirect_samples`` K (0, the default, shades direct light
    only), ``indirect_light_samples`` S2 (32), ``indirect_seed`` (lighting.SEED) and ``save_indirect``, which also
    writes the linear indirect-only image of every map as {view}/relighting_indirect/{light}.hdr.
    ``sampling``: 'light' (the default, the reference's estimator) or 'mis' (mis.relight_chunk_mis: S_b =
    ``brdf_samples`` (128) BRDF samples per hit and S_l = NUM_SAMPLES - S_b light samples per (map, hit), combined by
    multiple importance sampling; not with indirect light)."""
    from .relight import Environment_Light
    sampling, n_brdf = mis_options(args)
    opt = {k: getattr(args, k, v) for k, v in SCRIPT_DEFAULTS.items()}
    tensoIR, device = _model(args, tensoIR)
    if tensoIR is None:
        return
    W, H = dataset.img_wh
    if H < 11 or W < 11:
        raise ValueError(f"SSIM needs images of at least 11x11 pixels, got {W}x{H}")
    near_far = dataset.near_far
    names = list(dataset.light_names)
    L = len(names)
    thr = float(opt["acc_mask_threshold"])
    envir_light = Environment_Light(args.hdrdir, device=device)
    tables = env_tables(envir_light, names)
    if rescale_value is None:
        _, rescale_value = compute_rescale_ratio(tensoIR, dataset)
    rescale_value = torch.as_tensor(rescale_value, dtype=torch.float32).to(device)

    if sampling == 'mis':
        from .mis import mis_uniforms, relight_chunk_mis

    # one bounce of indirect light (indirect.py): off unless indirect_samples > 0
    n_ind = int(getattr(args, "indirect_samples", 0) or 0)
    save_ind = n_ind > 0 and bool(getattr(args, "save_indirect", False))
    if n_ind > 0:
        from .indirect import relight_chunk_indirect
        from .lighting import SEED
        seed = getattr(args, "indirect_seed", None)
        gen = torch.Generator(device).manual_seed(SEED if seed is None else int(seed))
        ind_kw = dict(indirect_samples=n_ind, indirect_light_samples=int(getattr(args, "indirect_light_samples", 32)
                                                                           or 32))

    metrics = _new_metrics(names)
    rgb_frames, aligned_albedo_list, roughness_list = [], [], []
    gp = args.geo_buffer_path
    for idx in range(len(dataset)):
        cur_dir_path = os.path.join(gp, f'{dataset.split}_{idx:0>3d}')
        os.makedirs(cur_dir_path, exist_ok=True)
        item = dataset[idx]
        frame_rays = item['rays'].squeeze(0).to(device)
        n_pix = frame_rays.shape[0]
        gt_mask = item['rgbs_mask'].squeeze(0).squeeze(-1).cpu()
        gt_rgb = item['rgbs'].squeeze(0).reshape(L, H * W, 3).to(device)
        gt_albedo = item['albedo'].squeeze(0).to(device)

        with_map = torch.empty(L, n_pix, 3, device=device)
        without_map = torch.empty(L, n_pix, 3, device=device)
        ind_map = torch.empty(L, n_pix, 3, device=device) if save_ind else None
        prim = {}
        for s, e, (rgb, depth, normal, albedo, rough, fresnel, acc, *_) in _primary_chunks(tensoIR, frame_rays,
                                                                                            args.batch_size):
            rays = frame_rays[s:e]
            for k, t in (("rgb", rgb), ("depth", depth), ("normal", normal), ("albedo", albedo), ("rough", rough),
                         ("acc", acc)):
                t = t.detach()
                if k not in prim:
                    prim[k] = torch.empty((n_pix,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
                prim[k][s:e] = t
            if sampling == 'mis':
                u_light, u_brdf = mis_uniforms(L, e - s, NUM_SAMPLES - n_brdf, n_brdf, device)
                relight_chunk_mis(tensoIR, envir_light, names, rays, (depth, normal, albedo, rough, fresnel, acc),
                                  rescale_value, u_light, u_brdf, acc_mask_threshold=thr,
                                  vis_equation=opt["vis_equation"], out=(with_map, without_map), row0=s, tables=tables)
                continue
            u = _uniforms(L, e - s, NUM_SAMPLES, device)
            if n_ind > 0:
                relight_chunk_indirect(tensoIR, envir_light, names, rays, (depth, normal, albedo, rough, fresnel, acc),
                                       rescale_value, u, gen, **ind_kw, acc_mask_threshold=thr,
                                       vis_equation=opt["vis_equation"], out=(with_map, without_map), row0=s,
                                       tables=tables, indirect_out=ind_map)
            else:
                relight_chunk_fused(tensoIR, envir_light, names, rays, (depth, normal, albedo, rough, fresnel, acc),
                                    rescale_value, u, NUM_SAMPLES, thr, opt["vis_equation"],
                                    out=(with_map, without_map), row0=s, tables=tables)

        # metrics of every map against its ground truth: the image without background
        for sub in ('with_bg', 'without_bg'):
            os.makedirs(os.path.join(cur_dir_path, f'relighting_{sub}'), exist_ok=True)
        _view_metrics(metrics, names, without_map, gt_rgb, H, W, device,
                      os.path.join(cur_dir_path, 'relighting_without_bg', 'relight_psnr.txt'))
        if opt["if_save_relight_rgb"]:
            _write_pairs(cur_dir_path, names, H, W, with_map, without_map)
        if save_ind:
            from .relight import write_hdr
            os.makedirs(os.path.join(cur_dir_path, 'relighting_indirect'), exist_ok=True)
            ind_np = ind_map.reshape(L, H, W, 3).cpu().numpy()
            for k, name in enumerate(names):
                write_hdr(os.path.join(cur_dir_path, 'relighting_indirect', f'{name}.hdr'), ind_np[k])

        # every image below uses the thresholded acc
        rgb_u8 = (prim["rgb"].reshape(H, W, 3) * 255).to(torch.uint8).cpu().numpy()
        rgb_frames.append(rgb_u8)
        acc_u8 = _acc_u8(prim["acc"], H, W)
        if opt["if_save_rgb"]:
            _imwrite(os.path.join(cur_dir_path, 'rgb.png'), rgb_u8)
        if opt["if_save_depth"]:
            depth_img, _ = visualize_depth_numpy(prim["depth"].reshape(H, W).cpu().numpy(), near_far)
            _imwrite(os.path.join(cur_dir_path, 'depth.png'), depth_img)
        if opt["if_save_acc"]:
            _imwrite(os.path.join(cur_dir_path, 'acc.png'), acc_u8[..., 0])
        if opt["if_save_albedo"]:
            m = gt_mask.reshape(-1).to(device)
            albedo_map = prim["albedo"].reshape(-1, 3).clone()
            # per-view three-channel lower median (:252)
            ratio = (gt_albedo[m] / albedo_map[m].clamp(min=1e-6)).median(dim=0)[0]
            albedo_map[m] = (ratio * albedo_map[m]).clamp(min=0.0, max=1.0)
            albedo_map = albedo_map.reshape(H, W, 3)
            alb_u8 = (albedo_map * 255).to(torch.uint8).cpu().numpy()
            _imwrite(os.path.join(cur_dir_path, 'albedo.png'), np.concatenate([alb_u8, acc_u8], axis=2))
            gamma_u8 = (albedo_map ** (1 / 2.2) * 255).to(torch.uint8).cpu().numpy()
            if opt["if_save_albedo_gamma_corrected"]:
                _imwrite(os.path.join(cur_dir_path, 'albedo_gamma_corrected.png'),
                         np.concatenate([gamma_u8, acc_u8], axis=2))
            gt_g = (gt_albedo.reshape(H, W, 3) ** (1 / 2.2) * 255).to(torch.uint8).cpu().numpy()
            _imwrite(os.path.join(cur_dir_path, 'gt_albedo_gamma_corrected.png'), np.concatenate([gt_g, acc_u8], axis=2))
            aligned_albedo_list.append(gamma_u8)
            # (roughness * 255) concatenated with the uint8 acc as float, then cast (:273-278)
            r = (prim["rough"].reshape(H, W, 1).expand(-1, -1, 3) * 255).cpu().numpy()
            rough_img = np.concatenate([r, acc_u8], axis=2).astype('uint8')
            _imwrite(os.path.join(cur_dir_path, 'roughness.png'), rough_img)
            roughness_list.append(rough_img)
        if opt["if_render_normal"]:
            nrm = F.normalize(prim["normal"].reshape(-1, 3), dim=-1) * 0.5 + 0.5
            nrm_u8 = (nrm.reshape(H, W, 3) * 255).to(torch.uint8).cpu().numpy()
            _imwrite(os.path.join(cur_dir_path, 'normal.png'), np.concatenate([nrm_u8, acc_u8], axis=2))

    _run_metrics(metrics, names, os.path.join(gp, 'relight_psnr.txt'))

    if opt["if_save_rgb_video"]:
        os.makedirs(os.path.join(gp, 'video'), exist_ok=True)
        _mimsave(os.path.join(gp, 'video', 'rgb_video.mp4'), rgb_frames)
    if opt["if_render_normal"]:
        os.makedirs(os.path.join(gp, 'video'), exist_ok=True)

        def normal_frames():
            frames = []
            for i in range(len(dataset)):
                nm = _imread(os.path.join(gp, f'{dataset.split}_{i:0>3d}', 'normal.png'))
                # the reference's expression as written (:302-304): mask[..., 3:4] is column 3 of the [H,W] mask,
                # broadcast against the image rows (square images only)
                mask = (nm[..., -1] / 255) > thr
                frames.append(nm[..., :3] * (mask[..., 3:4] / 255.0) + 255 * (1 - mask[..., 3:4] / 255.0))
            return frames
        _mimsave(os.path.join(gp, 'video', 'render_normal_video.mp4'), normal_frames)
    if opt["if_save_albedo"]:
        os.makedirs(os.path.join(gp, 'video'), exist_ok=True)
        _mimsave(os.path.join(gp, 'video', 'aligned_albedo_video.mp4'), aligned_albedo_list)
        _mimsave(os.path.join(gp, 'video', 'roughness_video.mp4'), roughness_list)
    if opt["render_video"]:
        for sub in ('without_bg', 'with_bg'):
            vp = os.path.join(gp, f'video_{sub}')
            os.makedirs(vp, exist_ok=True)
            for name in names:
                _video(os.path.join(vp, f'{name}_video.mp4'), gp, dataset.split, len(dataset),
                       os.path.join(f'relighting_{sub}', f'{name}.png'))

