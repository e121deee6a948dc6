"""Test-view evaluation: compute_rescale_ratio and the three evaluation loops of the reference's renderer.py (:12-53,
:134-516, :520-797, :801-1186) with the same signatures, defaults, return values, file layout and metric definitions.

What changes is where the work runs.  Each view is rendered in chunks of ``args.batch_size_test`` into device maps (no
host copy per chunk), and one call of the metric kernel (csrc/tir_eval.cu: PSNR sums, aligned albedo, gamma albedo
error, normal angular error and the four SSIMs of utils.rgb_ssim) replaces the host-side torch / numpy / scipy code.
uint8 images reach the host only when ``savePath`` is set (or a logger / the test_all videos need them).

Differences from the reference, all deliberate:
  * ``savePath=None`` writes nothing (the reference raises TypeError in os.makedirs);
  * the general multi-light loop returns the same 5-tuple as evaluation_iter_TensoIR;
  * PNGs are written with cv2 (RGB -> BGR, so the decoded pixels equal the arrays the reference hands to imageio);
    the test_all videos need ``imageio`` and are skipped with a notice without it;
  * LPIPS needs the ``lpips`` package (and its weights); without it the LPIPS values are reported as nan.
"""
from __future__ import annotations

import ctypes as C
import os
import random

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib

_GAMMA = 1.0 / 2.2
_LPIPS = {}


# ---- the metric kernel -------------------------------------------------------------------------------------------------
def view_metrics(H, W, rgb, rgb_brdf, gt_rgb, albedo=None, gt_albedo=None, gt_mask=None, ratio=None, normal=None,
                 gt_normal=None, ssim=True):
    """One call of tir_eval_view on device maps [H*W,3] (gt_mask [H*W] bool, ratio [4] = single, three-channel).
    Returns (out, aligned_single, aligned_three): out is a float64 device tensor [9] laid out as TIR_EVAL_N_OUT
    (include/tensoir_b200.h); the aligned albedo maps are None without the albedo terms."""
    lib = _lib.load()
    dev = rgb.device
    f32 = lambda t: None if t is None else t.detach().reshape(-1, 3).to(dev, torch.float32).contiguous()  # noqa: E731
    rgb, rgb_brdf, gt_rgb, albedo, gt_albedo, normal, gt_normal = (
        f32(t) for t in (rgb, rgb_brdf, gt_rgb, albedo, gt_albedo, normal, gt_normal))
    v = _lib.TirEvalView(H=int(H), W=int(W), ssim=int(bool(ssim)))
    keep = [rgb, rgb_brdf, gt_rgb]
    v.rgb, v.rgb_brdf, v.gt_rgb = (_lib.dptr(t) for t in keep)
    al1 = al3 = None
    if albedo is not None:
        mask = gt_mask.detach().reshape(-1).to(dev, torch.bool).contiguous()
        ratio = ratio.detach().reshape(4).to(dev, torch.float32).contiguous()
        al1, al3 = torch.empty_like(albedo), torch.empty_like(albedo)
        keep += [albedo, gt_albedo, mask, ratio]
        v.albedo, v.gt_albedo, v.ratio = _lib.dptr(albedo), _lib.dptr(gt_albedo), _lib.dptr(ratio)
        v.gt_mask = _lib.dptr(mask, dtype=torch.bool)
        v.aligned_single, v.aligned_three = _lib.dptr(al1), _lib.dptr(al3)
    if normal is not None:
        keep += [normal, gt_normal]
        v.normal, v.gt_normal = _lib.dptr(normal), _lib.dptr(gt_normal)
    n = C.c_int64(0)
    _lib.check(lib.tir_eval_work_size(int(H), int(W), C.byref(n)), "tir_eval_work_size")
    work = torch.empty(max(n.value, 1), dtype=torch.float64, device=dev)
    out = torch.empty(_lib.EVAL_N_OUT, dtype=torch.float64, device=dev)
    _lib.check(lib.tir_eval_view(C.byref(v), _lib.dptr(work, dtype=torch.float64), n.value,
                                 _lib.dptr(out, dtype=torch.float64), _lib.stream_ptr()), "tir_eval_view")
    return out, al1, al3


# ---- albedo rescale ratio ----------------------------------------------------------------------------------------------
@torch.no_grad()
def compute_rescale_ratio(tensoIR, dataset, sampled_num=20):
    """renderer.py:12-53: medians of gt_albedo / albedo.clamp(min=1e-6) over the gt_mask pixels of ``sampled_num``
    views taken every len(dataset) // sampled_num (0 repeats view 0, as in the reference).  Returns the single-channel
    (channel 0) and the per-channel ratio as device tensors (torch.median: the lower median)."""
    W, H = dataset.img_wh
    interval = len(dataset) // sampled_num
    dev = tensoIR.device
    gts, recs = [], []
    for idx in [i * interval for i in range(sampled_num)]:
        item = dataset[idx]
        rays = item['rays'].squeeze(0).to(dev)
        mask = item['rgbs_mask'].squeeze(0).reshape(-1).to(dev, torch.bool)
        gt_albedo = item['albedo'].squeeze(0).reshape(-1, 3).to(dev)
        light_idx = torch.zeros((rays.shape[0], 1), dtype=torch.int32, device=dev)
        albedo = torch.empty((rays.shape[0], 3), device=dev)
        for s in range(0, rays.shape[0], 65536):          # per-ray outputs: the chunk size does not change them
            out = tensoIR(rays[s:s + 65536], light_idx[s:s + 65536], is_train=False, white_bg=True, ndc_ray=False,
                          N_samples=-1)
            albedo[s:s + 65536] = out[3].detach()
        gts.append(gt_albedo[mask])
        recs.append(albedo[mask])
    q = torch.cat(gts, 0) / torch.cat(recs, 0).clamp(min=1e-6)
    single, three = q[..., 0].median(), q.median(dim=0)[0]
    print("single channel rescale ratio: ", single)
    print("three channels rescale ratio: ", three)
    return single, three


# ---- image helpers (host) ----------------------------------------------------------------------------------------------
def _u8(t):
    """(x.numpy() * 255).astype('uint8') of a float32 map, computed on the device, copied once."""
    return (t.float() * 255).to(torch.uint8).cpu().numpy()


def visualize_depth_numpy(depth, minmax):
    """utils.py:11-31 with minmax given: normalise to [0,1], uint8, cv2 JET colour map (channel order as cv2 returns
    it, which the reference then writes as if it were RGB)."""
    import cv2
    x = np.nan_to_num(depth)
    mi, ma = minmax
    x = (x - mi) / (ma - mi + 1e-8)
    x = (255 * x).astype(np.uint8)
    return cv2.applyColorMap(x, cv2.COLORMAP_JET), [mi, ma]


def _imwrite(path, img):
    """Write ``img`` (H,W,3 RGB or H,W gray, uint8) so that decoding the PNG gives back ``img``."""
    import cv2
    if img.ndim == 3:
        img = np.ascontiguousarray(img[..., ::-1])
    if not cv2.imwrite(path, img):
        raise OSError(f"could not write {path}")


def _lpips(gt, im, net_name, device):
    """utils.rgb_lpips (utils.py:69-81) when the lpips package is importable, else nan.  gt / im: [H,W,3] device."""
    try:
        import lpips
    except ImportError:
        return float("nan")
    if net_name not in _LPIPS:
        print(f'init_lpips: lpips_{net_name}')
        _LPIPS[net_name] = lpips.LPIPS(net=net_name, version='0.1').eval().to(device)
    g = gt.permute([2, 0, 1]).contiguous().to(device)
    i = im.permute([2, 0, 1]).contiguous().to(device)
    return float(_LPIPS[net_name](g, i, normalize=True).item())


def _envmap(tensoIR, test_dataset, device, variant):
    """renderer.py:183-202 / :568-577 / :851-870: the predicted SG environment map (all lights for the general
    variant), gamma 1/2.2, uint8; the GT probe on its left when the dataset has one (rotated variant)."""
    _, view_dirs = tensoIR.generate_envir_map_dir(256, 512)
    rgbs = tensoIR.get_light_rgbs(view_dirs.reshape(-1, 3).to(device), device=device)
    pred = (rgbs.reshape(256 * tensoIR.light_num, 512, 3) if variant == "general" else rgbs[0].reshape(256, 512, 3))
    pred = np.clip(pred.detach().cpu().numpy(), a_min=0, a_max=np.inf)
    pred = np.uint8(np.clip(np.power(pred, 1. / 2.2), 0., 1.) * 255.)
    if variant == "full" and getattr(test_dataset, "lights_probes", None) is not None:
        import cv2
        gt = test_dataset.lights_probes.reshape(test_dataset.envir_map_h, test_dataset.envir_map_w, 3).numpy()
        gt = np.uint8(np.clip(np.power(gt, 1. / 2.2), 0., 1.) * 255.)
        gt = cv2.resize(gt, (512, 256), interpolation=cv2.INTER_CUBIC)
        return np.concatenate((gt, pred), axis=1)
    return pred


_MAP_KEYS = ("rgb_map", "depth_map", "normal_map", "albedo_map", "roughness_map", "fresnel_map", "rgb_with_brdf_map",
             "normals_diff_map", "normals_orientation_loss_map", "acc_map")


def _render_view(renderer, tensoIR, rays, light_idx, args, N_samples, ndc_ray, white_bg, device):
    """renderer.py:225-250: the view in chunks of args.batch_size_test, written into device maps."""
    n = rays.shape[0]
    maps = {}
    for s in range(0, n, args.batch_size_test):
        e = min(s + args.batch_size_test, n)
        ret = renderer(rays[s:e], None, light_idx[s:e], tensoIR, N_samples=N_samples, ndc_ray=ndc_ray,
                       white_bg=white_bg, sample_method='fixed_envirmap', chunk_size=args.relight_chunk_size,
                       device=device, args=args)
        for k in _MAP_KEYS:
            t = ret[k].detach()
            if k not in maps:
                maps[k] = torch.empty((n,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
            maps[k][s:e] = t
    return maps


def _evaluate(variant, test_dataset, tensoIR, args, renderer, savePath, prtx, N_samples, white_bg, ndc_ray,
              compute_extra_metrics, device, logger, step, test_all, light_idx_to_test=-1):
    simple = variant == "simple"
    if savePath is not None:
        for d in ("", "/nvs_with_radiance_field", "/nvs_with_brdf", "/normal", "/normal_vis", "/brdf", "/envir_map/",
                  "/acc_map"):
            os.makedirs(savePath + d, exist_ok=True)
    near_far = test_dataset.near_far
    W, H = test_dataset.img_wh
    if compute_extra_metrics and (H < 11 or W < 11):
        raise ValueError(f"SSIM needs images of at least 11x11 pixels, got {W}x{H}")
    num_test = len(test_dataset) if test_all else min(args.N_vis, len(test_dataset))
    envirmap = _envmap(tensoIR, test_dataset, device, variant)
    if savePath is not None:
        _imwrite(f'{savePath}/envir_map/{prtx}envirmap.png', envirmap)
    test_duration = int(len(test_dataset) / num_test)
    global_ratio = None
    if test_all and not simple:
        single, three = compute_rescale_ratio(tensoIR, test_dataset, sampled_num=20)
        global_ratio = torch.cat([single.reshape(1), three.reshape(3)]).to(device, torch.float32)

    want_images = savePath is not None or bool(logger and step and not test_all) or (test_all and not simple)
    outs, lp = [], []
    vis = {k: [] for k in ("rgb", "rgb_brdf", "depth", "gt", "normal", "normal_vis", "normal_gt", "diff", "orient",
                           "albedo", "albedo_gamma", "single", "three", "gt_albedo", "rough", "fresnel")}
    for idx in range(num_test):
        if test_all and variant == "full":
            print(f"test {idx} / {num_test}")
        item = test_dataset.__getitem__(idx * test_duration)
        if variant == "general":
            li = light_idx_to_test if light_idx_to_test >= 0 else int(np.random.randint(tensoIR.light_num))
        else:
            li = 0
        rays = item['rays'].to(device)
        gt_rgb = item['rgbs'][li].to(device).reshape(-1, 3)
        light_idx = item['light_idx'][li]
        m = _render_view(renderer, tensoIR, rays, light_idx, args, N_samples, ndc_ray, white_bg, device)
        dev = m["rgb_map"].device
        gt_rgb = gt_rgb.to(dev)
        kw = {}
        if not simple:
            gt_albedo = item['albedo'].to(dev).reshape(-1, 3)
            gt_mask = item['rgbs_mask'].to(dev).reshape(-1).bool()
            albedo = m["albedo_map"].reshape(-1, 3)
            if global_ratio is not None:
                ratio = global_ratio.to(dev)
            else:                                            # renderer.py:282, :288: per-view medians
                q = gt_albedo[gt_mask] / albedo[gt_mask].clamp(min=1e-6)
                ratio = torch.cat([q[..., 0].median().reshape(1), q.median(dim=0)[0]])
            kw = dict(albedo=albedo, gt_albedo=gt_albedo, gt_mask=gt_mask, ratio=ratio, normal=m["normal_map"],
                      gt_normal=item['normals'].to(dev))
        out, al1, al3 = view_metrics(H, W, m["rgb_map"], m["rgb_with_brdf_map"], gt_rgb, ssim=compute_extra_metrics,
                                     **kw)
        outs.append(out)
        if compute_extra_metrics:
            pairs = [(gt_rgb, m["rgb_map"].clamp(0.0, 1.0)), (gt_rgb, m["rgb_with_brdf_map"].clamp(0.0, 1.0))]
            if not simple:
                pairs += [(kw["gt_albedo"], al1), (kw["gt_albedo"], al3)]
            lp.append([_lpips(g.reshape(H, W, 3), i.reshape(H, W, 3), net, tensoIR.device)
                       for g, i in pairs for net in ("alex", "vgg")])
        if not want_images:
            continue

        # ---- uint8 images (renderer.py:342-416) ----
        rgb = _u8(m["rgb_map"].clamp(0.0, 1.0).reshape(H, W, 3))
        rgb_brdf = _u8(m["rgb_with_brdf_map"].clamp(0.0, 1.0).reshape(H, W, 3))
        gt = _u8(gt_rgb.reshape(H, W, 3))
        albedo_u8 = _u8(m["albedo_map"].reshape(H, W, 3))
        rough = _u8(m["roughness_map"].reshape(H, W, 1).repeat(1, 1, 3))
        fresnel = _u8(m["fresnel_map"].reshape(H, W, 3))
        acc_t = (m["acc_map"].reshape(H, W).float() * 255).to(torch.uint8)
        acc = acc_t.cpu().numpy()
        depth, _ = visualize_depth_numpy(m["depth_map"].reshape(H, W).cpu().numpy(), near_far)
        nrm_t = (F.normalize(m["normal_map"].reshape(-1, 3), dim=-1) * 0.5 + 0.5).reshape(H, W, 3)
        nrm_u8 = (nrm_t * 255).to(torch.uint8)
        a = acc_t[:, :, None].double() / 255.0
        normal_vis = (nrm_u8.double() * a + (1 - a) * 255).to(torch.uint8).cpu().numpy()
        nrm = nrm_u8.cpu().numpy()
        diff = _u8(torch.clamp(m["normals_diff_map"], 0.0, 1.0).reshape(H, W, 1).repeat(1, 1, 3))
        orient = _u8(torch.clamp(m["normals_orientation_loss_map"], 0.0, 1.0).reshape(H, W, 1).repeat(1, 1, 3))
        if simple:
            albedo_gamma = _u8(m["albedo_map"].reshape(H, W, 3).clip(0, 1.) ** _GAMMA)
            normal_img = np.concatenate((nrm, diff, orient), axis=1)
            albedo_img = albedo_gamma
        else:
            gt_n = _u8((F.normalize(kw["gt_normal"].reshape(-1, 3), dim=-1) * 0.5 + 0.5).reshape(H, W, 3))
            single = _u8(al1.reshape(H, W, 3) ** _GAMMA)
            three = _u8(al3.reshape(H, W, 3) ** _GAMMA)
            gt_a = _u8(kw["gt_albedo"].reshape(H, W, 3) ** _GAMMA)
            normal_img = np.concatenate((nrm, gt_n, diff, orient), axis=1)
            albedo_img = np.concatenate((single, three, gt_a), axis=1)
        if savePath is not None:
            base = f'{prtx}{idx:03d}'
            _imwrite(f'{savePath}/nvs_with_radiance_field/{base}.png', np.concatenate((rgb, gt, depth), axis=1))
            _imwrite(f'{savePath}/nvs_with_brdf/{base}.png', np.concatenate((rgb_brdf, gt), axis=1))
            _imwrite(f'{savePath}/normal/{base}.png', normal_img)
            _imwrite(f'{savePath}/normal_vis/{base}.png', normal_vis)
            _imwrite(f'{savePath}/brdf/{base}.png', np.concatenate((albedo_u8, rough, fresnel), axis=1))
            _imwrite(f'{savePath}/brdf/{base}_albedo.png', albedo_img)
            _imwrite(f'{savePath}/brdf/{base}_roughness.png', rough)
            _imwrite(f'{savePath}/acc_map/{base}.png', acc)
        for k, v in (("rgb", rgb), ("rgb_brdf", rgb_brdf), ("depth", depth), ("gt", gt), ("normal", nrm),
                     ("normal_vis", normal_vis), ("diff", diff), ("orient", orient), ("albedo", albedo_u8),
                     ("rough", rough), ("fresnel", fresnel)):
            vis[k].append(v)
        if simple:
            vis["albedo_gamma"].append(albedo_gamma)
        else:
            vis["normal_gt"].append(gt_n)
            vis["single"].append(single)
            vis["three"].append(three)
            vis["gt_albedo"].append(gt_a)

    if logger and step and not test_all:
        _log_images(logger, step, vis, envirmap, simple)

    # ---- metrics (renderer.py:455-501): one host copy for all views ----
    o = torch.stack(outs).cpu().numpy()
    npix = float(H * W)
    psnr_v = [-10.0 * np.log(float(x) / (npix * 3)) / np.log(10.0) for x in o[:, 0]]
    psnr_b = [-10.0 * np.log(float(x) / (npix * 3)) / np.log(10.0) for x in o[:, 1]]
    psnr = np.mean(np.asarray(psnr_v))
    psnr_rgb_brdf = np.mean(np.asarray(psnr_b))
    if not simple:
        n_all = len(outs) * npix * 3
        PSNR_albedo_single = -10.0 * np.log(o[:, 2].sum() / n_all) / np.log(10.0)
        PSNR_albedo_three = -10.0 * np.log(o[:, 3].sum() / n_all) / np.log(10.0)
        MAE = o[:, 4].sum() / (len(outs) * npix)
    if compute_extra_metrics:
        ss = o[:, 5:9].mean(axis=0)
        lpm = np.asarray(lp, dtype=np.float64).mean(axis=0)
        head = f'Iteration:{prtx[:-1]}: \n'
        if simple:
            msg = head + f'\tPSNR_nvs: {psnr:.2f}, PSNR_nvs_brdf: {psnr_rgb_brdf:.2f}\n'
        else:
            msg = head + (f'\tPSNR_nvs: {psnr:.2f}, PSNR_nvs_brdf: {psnr_rgb_brdf:.2f}, '
                          f'PNSR_albedo_single_aligned: {PSNR_albedo_single:.2f}, '
                          f'PNSR_albedo_three_aligned: {PSNR_albedo_three:.2f}\n')
        names = ("rgb", "rgb_brdf") if simple else ("rgb", "rgb_brdf", "albedo_single", "albedo_three")
        for j, nm in enumerate(names):
            msg += (f'\tSSIM_{nm}: {ss[j]:.4f}, L_Alex_{nm}: {lpm[2 * j]:.4f}, '
                    f'L_VGG_{nm}: {lpm[2 * j + 1]:.4f}\n')
        if not simple:
            msg += f'\tMAE: {MAE:.2f}\n'
    elif simple:
        msg = f'Iteration:{prtx[:-1]}, PSNR_nvs: {psnr:.2f}, PSNR_nvs_brdf: {psnr_rgb_brdf:.2f}\n'
    else:
        msg = (f'Iteration:{prtx[:-1]}, PSNR_nvs: {psnr:.2f}, PSNR_nvs_brdf: {psnr_rgb_brdf:.2f}, MAE: {MAE:.2f}, '
               f'PSNR_albedo_single_aligned: {PSNR_albedo_single:.2f}, '
               f'PSNR_albedo_three_aligned: {PSNR_albedo_three:.2f}\n')
    if savePath is not None:
        with open(f'{savePath}/metrics_record.txt', 'a') as f:
            f.write(msg)

    if test_all and not simple and savePath is not None:
        _videos(savePath, vis)
    if simple:
        return psnr, psnr_rgb_brdf
    return psnr, psnr_rgb_brdf, MAE, PSNR_albedo_single, PSNR_albedo_three


def _videos(savePath, vis):
    """renderer.py:504-514, when imageio is importable."""
    try:
        import imageio
    except ImportError:
        print("evaluation: imageio is not installed, the test_all videos are not written")
        return
    p = savePath + "/video"
    os.makedirs(p, exist_ok=True)
    for name, key in (("rgb", "rgb"), ("rgb_brdf", "rgb_brdf"), ("gt_normal_video", "normal_gt"),
                      ("render_normal_video", "normal"), ("render_normal_vis_video", "normal_vis"),
                      ("single_aligned_albedo", "single"), ("three_aligned_albedo", "three"),
                      ("roughness", "rough")):
        imageio.mimsave(os.path.join(p, f'{name}.mp4'), np.stack(vis[key]), fps=24, quality=8)


def _log_images(logger, step, vis, envirmap, simple):
    """renderer.py:420-452 / :737-766: one random view's images to the logger."""
    import torchvision.utils as vutils
    i = random.choice(range(len(vis["rgb"])))
    t = lambda k: torch.from_numpy(vis[k][i])  # noqa: E731
    grid = lambda ks: torch.stack([t(k) for k in ks]).permute(0, 3, 1, 2).to(float)  # noqa: E731
    g = {'test/rgb': grid(["rgb", "rgb_brdf", "gt", "depth"]),
         'test/normal': grid(["normal", "diff", "orient"] if simple else ["normal", "normal_gt", "diff", "orient"]),
         'test/brdf': grid(["albedo", "rough", "fresnel"]),
         'test/envir_map': torch.from_numpy(envirmap).unsqueeze(0).permute(0, 3, 1, 2).to(float),
         'test/albedo': grid(["albedo", "albedo_gamma"] if simple else ["single", "three", "gt_albedo"])}
    for tag, x in g.items():
        logger.add_image(tag, vutils.make_grid(x, padding=0, normalize=True, value_range=(0, 255)), step)


@torch.no_grad()
def evaluation_iter_TensoIR(test_dataset, tensoIR, args, renderer, savePath=None, prtx='', N_samples=-1,
                            white_bg=False, ndc_ray=False, compute_extra_metrics=True, device='cuda', logger=None,
                            step=None, test_all=False):
    """renderer.py:134-516 -> (psnr, psnr_rgb_brdf, MAE, PSNR_albedo_single, PSNR_albedo_three)."""
    return _evaluate("full", test_dataset, tensoIR, args, renderer, savePath, prtx, N_samples, white_bg, ndc_ray,
                     compute_extra_metrics, device, logger, step, test_all)


@torch.no_grad()
def evaluation_iter_TensoIR_simple(test_dataset, tensoIR, args, renderer, savePath=None, prtx='', N_samples=-1,
                                   white_bg=False, ndc_ray=False, compute_extra_metrics=True, device='cuda',
                                   logger=None, step=None, test_all=False):
    """renderer.py:520-797 -> (psnr, psnr_rgb_brdf)."""
    return _evaluate("simple", test_dataset, tensoIR, args, renderer, savePath, prtx, N_samples, white_bg, ndc_ray,
                     compute_extra_metrics, device, logger, step, test_all)


@torch.no_grad()
def evaluation_iter_TensoIR_general_multi_lights(test_dataset, tensoIR, args, renderer, savePath=None, prtx='',
                                                 N_samples=-1, white_bg=False, ndc_ray=False,
                                                 compute_extra_metrics=True, device='cuda', logger=None, step=None,
                                                 test_all=False, light_idx_to_test=-1):
    """renderer.py:801-1186: one light per view (``light_idx_to_test``, or one np.random.randint(light_num) draw per
    view when negative) -> the same 5-tuple as evaluation_iter_TensoIR."""
    return _evaluate("general", test_dataset, tensoIR, args, renderer, savePath, prtx, N_samples, white_bg, ndc_ray,
                     compute_extra_metrics, device, logger, step, test_all, light_idx_to_test)
