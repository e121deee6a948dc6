"""Generate tests/golden/eval_reference.pt by running the REAL reference's evaluation loops (imported from a checkout of
TensoIR) on the CPU.  The reference import, its CPU stubs and the rotated-model builder are make_golden.py's.

    python tests/golden/make_eval_golden.py <path to the TensoIR checkout>

Only eval_reference.pt is written; the other fixtures are left as they are.  tests/test_eval_gpu.py checks the CUDA
evaluation path against it.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import REF, _args, build_rotated, import_reference  # noqa: E402  (REF: the checkout in argv[1])


def eval_fixture():
    """eval_reference.pt: the reference's evaluation loops (renderer.py:12-53, :134-1186) on the CPU, on 3 synthetic
    32x24 views (tensoir_b200.synthetic.SyntheticViews) of the rotated G=24 and the general G=20 fixture models, with
    batch_size_test 300 so every view is rendered in 3 chunks.  Records the returned tuples, metrics_record.txt, the
    rescale ratios, every imageio.imwrite (relative path + array; shape only for the environment maps), the renderer
    maps of each view of the first run, utils.rgb_ssim of the four pairs of each view and on standalone pairs."""
    import shutil
    import tempfile
    ru, rot, gen, _ = import_reference()
    import renderer as R
    import utils as U
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    sys.path.insert(0, os.path.join(REPO, "tests"))
    from gpu_helpers import load_fixture

    writes = []

    def imwrite(path, arr):
        writes.append((path, np.asarray(arr).copy()))
    R.imageio.imwrite = imwrite
    R.imageio.mimsave = lambda *a, **k: None
    ssims = []
    _ssim = U.rgb_ssim

    def rgb_ssim(a, b, max_val):
        v = _ssim(a, b, max_val)
        ssims.append(float(v))
        return v
    R.rgb_ssim = rgb_ssim
    R.rgb_lpips = lambda *a, **k: 0.0                 # no lpips weights: a constant stands in
    maps = []

    def recording_renderer(rays, normal_gt, light_idx, tensoIR, **kw):
        ret = R.Renderer_TensoIR_train(rays, normal_gt, light_idx, tensoIR, **kw)
        maps.append({k: ret[k].detach().clone() for k in ("rgb_map", "depth_map", "normal_map", "albedo_map",
                                                           "roughness_map", "fresnel_map", "rgb_with_brdf_map",
                                                           "normals_diff_map", "normals_orientation_loss_map",
                                                           "acc_map")})
        return ret

    def model(name):
        fx = load_fixture(name)
        if fx["kind"] == "rotated":
            m = build_rotated(rot, G=fx["grid_size"][0], lights=[f"{r:03d}" for r in fx["light_rotation"]])
        else:
            aabb = fx["aabb"]
            m = gen.TensorVMSplit(aabb, fx["grid_size"], 'cpu', density_n_comp=[16, 16, 16],
                                  appearance_n_comp=[48, 48, 48], app_dim=27, near_far=[2.0, 6.0],
                                  shadingMode='MLP_Fea', alphaMask_thres=0.001, density_shift=-10, distance_scale=25,
                                  pos_pe=2, view_pe=2, fea_pe=2, featureC=128, step_ratio=0.5,
                                  fea2denseAct='softplus', normals_kind='derived_plus_predicted',
                                  light_name_list=['sunset', 'snow', 'courtyard'], light_kind='sg', dataset=None,
                                  numLgtSGs=128)
            for p, v in zip(m.lgtSGs_list, fx["lgt_sgs_list"]):
                p.data.copy_(v)
        m.load_state_dict(fx["state_dict"])
        m.alphaMask = rot.AlphaGridMask('cpu', fx["alpha_aabb"], fx["alpha_volume"])
        glr = m.get_light_rgbs           # the loops omit device= (default 'cuda'); pin it to the CPU
        m.get_light_rgbs = lambda dirs=None, device='cpu': glr(dirs, device='cpu')
        return m

    H, W = 24, 32
    poses = hemisphere_poses(3)
    args = _args(24)
    args.N_vis, args.batch_size_test, args.relight_chunk_size = 5, 300, 160000
    out = {"H": H, "W": W, "poses": poses, "batch_size_test": 300, "N_vis": 5, "runs": {}}
    tmp = tempfile.mkdtemp()
    runs = (("full", "rotated_g24.pt", R.evaluation_iter_TensoIR, dict(test_all=False, compute_extra_metrics=False), 1),
            ("full_all", "rotated_g24.pt", R.evaluation_iter_TensoIR, dict(test_all=True, compute_extra_metrics=False), 1),
            ("full_extra", "rotated_g24.pt", R.evaluation_iter_TensoIR, dict(test_all=False, compute_extra_metrics=True), 1),
            ("simple", "rotated_g24.pt", R.evaluation_iter_TensoIR_simple, dict(test_all=False, compute_extra_metrics=False), 1),
            ("general", "general_g20.pt", R.evaluation_iter_TensoIR_general_multi_lights,
             dict(test_all=False, compute_extra_metrics=False, light_idx_to_test=1), 3))
    for name, fx_name, fn, kw, n_lights in runs:
        m = model(fx_name)
        ds = SyntheticViews(poses, H, W, n_lights=n_lights)
        writes.clear(), ssims.clear(), maps.clear()
        save = os.path.join(tmp, name)
        torch.manual_seed(123)
        ret = fn(ds, m, args, recording_renderer, savePath=save, prtx='7_', N_samples=-1, white_bg=True,
                 device='cpu', **kw)
        # arrays of the rotated-model runs, shapes only for the others and for the environment maps (size budget)
        keep = name.startswith("full")
        rec = {"kwargs": kw, "n_lights": n_lights, "model": fx_name, "returned": tuple(float(x) for x in ret),
               "metrics_record": open(os.path.join(save, "metrics_record.txt")).read(), "ssim": list(ssims),
               "writes": [(os.path.relpath(p, save), a if keep and "envir_map" not in p else a.shape)
                          for p, a in writes]}
        if name == "full":
            n_chunks = -(-H * W // 300)
            rec["maps"] = [{k: torch.cat([maps[v * n_chunks + c][k] for c in range(n_chunks)])
                            for k in maps[0]} for v in range(len(ds))]
        out["runs"][name] = rec
        if name == "full_all":
            out["rescale_ratio"] = tuple(t.clone() for t in R.compute_rescale_ratio(m, ds, sampled_num=20))
    shutil.rmtree(tmp)
    g = torch.Generator().manual_seed(4)
    pairs = [torch.rand(2, 37, 53, 3, generator=g),
             torch.stack([torch.full((19, 23, 3), 0.5), torch.full((19, 23, 3), 0.25)]),
             torch.rand(2, 11, 30, 3, generator=g)]
    pairs[1][0, 5:9, 3:12] = torch.rand(4, 9, 3, generator=g)
    out["ssim_pairs"] = [(p[0].clone(), p[1].clone(), float(U.rgb_ssim(p[0], p[1], 1))) for p in pairs]
    path = os.path.join(HERE, "eval_reference.pt")
    torch.save(out, path)
    print("eval_reference.pt", os.path.getsize(path) // 1024, "KiB")



if __name__ == "__main__":
    if REF is None or not os.path.isdir(REF):
        raise SystemExit(__doc__)
    eval_fixture()
