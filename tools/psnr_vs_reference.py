"""PSNR of our image against the reference algorithm's image (BASELINE metric, second half) on the GPU.

Renders a centred W x W crop of one 800x800 test view of the synthetic lego scene twice — through the library
(`Renderer_TensoIR_train`, CUDA kernels) and through the oracle's restatement of the reference run as eager PyTorch on the
same GPU — with the same seed, and prints PSNR for the radiance-field image and the physically-based image.

    python tools/psnr_vs_reference.py [grid=128] [crop=96]
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                      # noqa: E402
import __graft_entry__ as g       # noqa: E402

g.build()
from oracle import tensoir_oracle as O                                        # noqa: E402  (checker only)
from tensoir_b200 import Renderer_TensoIR_train                               # noqa: E402
from tensoir_b200.synthetic import make_lego_model, hemisphere_poses, image_rays   # noqa: E402

dev = torch.device("cuda", 0)
grid = int(sys.argv[1]) if len(sys.argv) > 1 else 128
crop = int(sys.argv[2]) if len(sys.argv) > 2 else 96
model = make_lego_model(grid, dev)
rays = image_rays(hemisphere_poses(200)[7]).reshape(800, 800, 6)
lo = 400 - crop // 2
rays = rays[lo:lo + crop, lo:lo + crop].reshape(-1, 6).contiguous().to(dev)
li = torch.zeros(rays.shape[0], 1, dtype=torch.int32, device=dev)

field = bench.make_lego_state(grid).to(dev)     # same seed, same init order as make_lego_model: the twin field

ours, ref = {}, {}
with torch.no_grad():
    for s in range(0, rays.shape[0], 4096):
        torch.manual_seed(7 + s)
        a = Renderer_TensoIR_train(rays[s:s + 4096], None, li[s:s + 4096], model, N_samples=-1, ndc_ray=False,
                                   white_bg=True, is_train=False, is_relight=True, sample_method='fixed_envirmap',
                                   chunk_size=160000, device=dev, args=bench.Args)
        torch.manual_seed(7 + s)
        b = O.renderer_train(field, rays[s:s + 4096], li[s:s + 4096], -1, True, False, True, 'fixed_envirmap',
                             160000, 96, 0.05, 1.5)
        for k in ("rgb_map", "rgb_with_brdf_map"):
            ours.setdefault(k, []).append(a[k])
            ref.setdefault(k, []).append(b[k])


def psnr(x, y):
    mse = ((torch.cat(x).float() - torch.cat(y).float()) ** 2).mean()
    return float(-10.0 * torch.log10(mse.clamp_min(1e-20)))


print(json.dumps({"what": f"{crop}x{crop} crop of an 800x800 view, grid {grid}, fixed_envirmap",
                  "psnr_rgb_map_db": psnr(ours["rgb_map"], ref["rgb_map"]),
                  "psnr_rgb_with_brdf_map_db": psnr(ours["rgb_with_brdf_map"], ref["rgb_with_brdf_map"])}))
