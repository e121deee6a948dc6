"""PyTorch-GPU denominator (BASELINE.md §3 item 4): the reference's algorithm (oracle port = the same torch ops the
reference executes) run with device='cuda' on the same workload as bench.py — eager ATen kernels, no custom code."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import tensoir_oracle as O   # noqa: E402
from bench import make_lego_state  # noqa: E402
from tensoir_b200.synthetic import hemisphere_poses, training_batch, n_samples_for  # noqa: E402

grid, batch, steps, warm = 300, 4096, 5, 2
torch.set_num_threads(16)
f = make_lego_state(grid).to("cuda")
for p in f.parameters():
    p.requires_grad_(True)
opt = torch.optim.Adam([{"params": f.parameters(), "lr": 1e-3}], betas=(0.9, 0.99))
poses = hemisphere_poses(100)
n_s = n_samples_for(grid)
ts, rays_n = [], []
for it in range(warm + steps):
    rays, li = training_batch(poses, batch, it)
    rays, li = rays.cuda(), li.cuda()
    f.counters.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ret = O.renderer_train(f, rays, li, n_s, True, True, True, 'stratified_sampling', 160000, 96, 0.05, 1.5)
    target = torch.full_like(ret["rgb_map"], 0.5)
    loss = torch.mean((ret['rgb_map'] - target) ** 2) + 0.2 * torch.mean((ret['rgb_with_brdf_map'] - target) ** 2)
    loss = loss + 0.0005 * ret['normals_diff_map'].mean() + 0.001 * ret['normals_orientation_loss_map'].mean()
    loss = loss + 0.001 * ret['roughness_smoothness_loss'] + 0.001 * ret['albedo_smoothness_loss']
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    if it >= warm:
        ts.append(time.perf_counter() - t0)
        rays_n.append(batch + f.counters.get("secondary_rays", 0))
print(json.dumps({"what": "reference algorithm (oracle port, eager PyTorch) on one GPU, same workload as bench.py",
                  "grid": grid, "batch": batch, "steps": steps, "ms_per_step": 1e3 * sum(ts) / len(ts),
                  "rays_per_s": sum(rays_n) / sum(ts), "peak_mem_GB": torch.cuda.max_memory_allocated() / 1e9}))
