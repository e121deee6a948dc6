"""Pure PyTorch / numpy / scipy restatement of the reference's test-view metrics (renderer.py:12-53, :211-501;
utils.py:93-139): what tensoir_b200.evaluation and csrc/tir_eval.cu are checked against on the CPU.

Every operation runs in the dtype the reference uses: the maps are float32 tensors / arrays, scipy's convolve2d promotes
to the float64 filter, numpy reduces float32 arrays in float32.  Sums that the kernel returns are also given here in
float64 over the float32 terms (``*_sum``), so a comparison does not depend on the summation order.
"""
import numpy as np
import scipy.signal
import torch
import torch.nn.functional as F


def gaussian_filter(size=11, sigma=1.5):
    """utils.py:104-109."""
    half = size // 2
    shift = (2 * half - size + 1) / 2
    f = np.exp(-0.5 * ((np.arange(size) - half + shift) / sigma) ** 2)
    return f / np.sum(f)


def rgb_ssim(img0, img1, max_val=1, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03):
    """utils.rgb_ssim: mean SSIM over the valid windows of the three channels of [H,W,3] float32 images."""
    a = np.asarray(img0)
    b = np.asarray(img1)
    assert a.ndim == 3 and a.shape[-1] == 3 and a.shape == b.shape
    filt = gaussian_filter(filter_size, filter_sigma)

    def blur(z):
        return np.stack([scipy.signal.convolve2d(scipy.signal.convolve2d(z[..., c], filt[:, None], mode='valid'),
                                                 filt[None, :], mode='valid') for c in range(3)], -1)

    mu0, mu1 = blur(a), blur(b)
    mu00, mu11, mu01 = mu0 * mu0, mu1 * mu1, mu0 * mu1
    s00 = np.maximum(0., blur(a * a) - mu00)              # a * a: float32 products, as img0**2 on a float32 tensor
    s11 = np.maximum(0., blur(b * b) - mu11)
    s01 = blur(a * b) - mu01
    s01 = np.sign(s01) * np.minimum(np.sqrt(s00 * s11), np.abs(s01))
    c1, c2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
    return float(np.mean((2 * mu01 + c1) * (2 * s01 + c2) / ((mu00 + mu11 + c1) * (s00 + s11 + c2))))


def view_ratios(albedo, gt_albedo, gt_mask):
    """renderer.py:282, :288: per-view medians of gt / albedo.clamp(min=1e-6) over the mask -> (single, three[3])."""
    m = gt_mask.reshape(-1).bool()
    q = gt_albedo.reshape(-1, 3)[m] / albedo.reshape(-1, 3)[m].clamp(min=1e-6)
    return q[..., 0].median(), q.median(dim=0)[0]


def rescale_ratio(albedos, gt_albedos, gt_masks):
    """compute_rescale_ratio (renderer.py:12-53) on already rendered albedo maps of the sampled views."""
    m = [g.reshape(-1).bool() for g in gt_masks]
    gt = torch.cat([g.reshape(-1, 3)[k] for g, k in zip(gt_albedos, m)])
    rec = torch.cat([a.reshape(-1, 3)[k] for a, k in zip(albedos, m)])
    q = gt / rec.clamp(min=1e-6)
    return q[..., 0].median(), q.median(dim=0)[0]


def view_metrics(H, W, rgb, rgb_brdf, gt_rgb, albedo=None, gt_albedo=None, gt_mask=None, ratio_single=None,
                 ratio_three=None, normal=None, gt_normal=None, ssim=True):
    """What one view contributes (renderer.py:265-321, :353-394): a dict of float64 sums over float32 terms, the
    SSIMs, and the aligned albedo maps [H,W,3] float32."""
    out = {}
    rgb = rgb.reshape(H, W, 3).float().clamp(0.0, 1.0)
    rgb_brdf = rgb_brdf.reshape(H, W, 3).float().clamp(0.0, 1.0)
    gt = gt_rgb.reshape(H, W, 3).float()
    out["sse_rgb"] = float(((rgb - gt) ** 2).double().sum())
    out["sse_rgb_brdf"] = float(((rgb_brdf - gt) ** 2).double().sum())
    out["mse_rgb"] = float(torch.mean((rgb - gt) ** 2))
    out["mse_rgb_brdf"] = float(torch.mean((rgb_brdf - gt) ** 2))
    if ssim:
        out["ssim_rgb"] = rgb_ssim(rgb, gt)
        out["ssim_rgb_brdf"] = rgb_ssim(rgb_brdf, gt)
    if albedo is not None:
        alb = albedo.reshape(H, W, 3).float()
        gta = gt_albedo.reshape(H, W, 3).float()
        m = gt_mask.reshape(H, W).bool()
        single, three = torch.ones_like(alb), torch.ones_like(alb)
        single[m] = (ratio_single * alb[m]).clamp(min=0.0, max=1.0)
        three[m] = (ratio_three * alb[m]).clamp(min=0.0, max=1.0)
        out["aligned_single"], out["aligned_three"] = single, three
        g = 1 / 2.2
        gt_g = gta.numpy() ** g
        out["gse_single"] = float(((gt_g - single.numpy() ** g) ** 2).astype(np.float64).sum())
        out["gse_three"] = float(((gt_g - three.numpy() ** g) ** 2).astype(np.float64).sum())
        if ssim:
            out["ssim_albedo_single"] = rgb_ssim(single, gta)
            out["ssim_albedo_three"] = rgb_ssim(three, gta)
    if normal is not None:
        p = F.normalize(normal.reshape(-1, 3).float(), dim=-1).numpy()
        g = F.normalize(gt_normal.reshape(-1, 3).float(), dim=-1).numpy()
        ang = np.arccos(np.clip(np.sum(g * p, axis=-1), -1, 1)) * 180 / np.pi
        out["angle_sum"] = float(ang.astype(np.float64).sum())
        out["angles"] = ang
    return out


def aggregate(views, H, W, simple=False):
    """renderer.py:455-498: the loop's returned metrics from the per-view dicts (float64 sums)."""
    n = H * W
    psnr = float(np.mean([-10.0 * np.log(v["sse_rgb"] / (n * 3)) / np.log(10.0) for v in views]))
    psnr_b = float(np.mean([-10.0 * np.log(v["sse_rgb_brdf"] / (n * 3)) / np.log(10.0) for v in views]))
    if simple:
        return psnr, psnr_b
    tot = len(views) * n * 3
    ps = -10.0 * np.log(sum(v["gse_single"] for v in views) / tot) / np.log(10.0)
    pt = -10.0 * np.log(sum(v["gse_three"] for v in views) / tot) / np.log(10.0)
    mae = sum(v["angle_sum"] for v in views) / (len(views) * n)
    return psnr, psnr_b, float(mae), float(ps), float(pt)
