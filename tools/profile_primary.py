"""Eager training steps of the bench model (no CUDA graph) for ncu captures of the primary-march kernels:
    ncu --set full --import-source on --clock-control none -k regex:'heads_|app_mlp_kernel' --launch-skip 8 -c 3 \
        -o prim python tools/profile_primary.py"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--grid", type=int, default=300)
ap.add_argument("--steps", type=int, default=4)
a = ap.parse_args()
import __graft_entry__ as g   # noqa: E402
g.build()
from tensoir_b200 import Renderer_TensoIR_train  # noqa: E402
from tensoir_b200.synthetic import make_lego_model, hemisphere_poses, training_batch, n_samples_for  # noqa: E402
from bench import Args, loss_of  # noqa: E402

dev = torch.device("cuda:0")
m = make_lego_model(a.grid, dev)
opt = torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), betas=(0.9, 0.99), fused=True)
poses = hemisphere_poses(100)
target = torch.full((4096, 3), 0.5, device=dev)
for it in range(a.steps):
    rays, li = training_batch(poses, 4096, it)
    ret = Renderer_TensoIR_train(rays.to(dev), None, li.to(dev), m, N_samples=n_samples_for(a.grid), white_bg=True,
                                 is_train=True, is_relight=True, sample_method='stratified_sampling', device=dev,
                                 args=Args)
    loss = loss_of(ret, target, m)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
torch.cuda.synchronize()
print("loss", float(loss))
