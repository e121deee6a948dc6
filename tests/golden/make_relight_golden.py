"""Generate tests/golden/relight_reference.pt by running the REAL reference's relight() (scripts/relight_importance.py,
imported from a checkout of TensoIR) on the CPU.  The reference import, its CPU stubs and the rotated-model builder are
make_golden.py's.

    python tests/golden/make_relight_golden.py <path to the TensoIR checkout>

Only relight_reference.pt is written; the other fixtures are left as they are.  tests/test_relighting_gpu.py replays the
recorded draws through tensoir_b200.relighting._uniforms and checks relight() against it.
"""
import os
import sys
import types
import lzma

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_golden import REF, build_rotated, import_reference  # noqa: E402  (REF: the checkout in argv[1])

NAMES = ["bridge", "city"]
H, W, BATCH = 24, 32, 300


def hdr_maps():
    """Two small HDR maps, each a dim sky with a bright sun that holds most of the sampling mass (16x32 and 32x64); the
    concentrated draws keep the recorded indices compressible."""
    out = {}
    for k, (name, (h, w)) in enumerate(zip(NAMES, ((16, 32), (32, 64)))):
        g = torch.Generator().manual_seed(31 + k)
        env = torch.exp(0.5 * torch.randn(h, w, 3, generator=g)) * 0.03
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        env[((yy - h // 4) ** 2 + (xx - (w // 3 + 7 * k)) ** 2) <= max(1, h // 16) ** 2] = 40.0
        out[name] = env.numpy().astype(np.float32)
    return out


def relight_fixture():
    import shutil
    import tempfile

    import cv2
    ru, rot, _, _ = import_reference()
    sys.path.insert(0, os.path.join(REF, "scripts"))
    import relight_importance as RI
    from tensoir_b200.synthetic import SyntheticViews, hemisphere_poses
    sys.path.insert(0, os.path.join(REPO, "tests"))
    from gpu_helpers import load_fixture

    tmp = tempfile.mkdtemp()
    hdrdir = os.path.join(tmp, "hdr")
    os.makedirs(hdrdir)
    maps = hdr_maps()
    for name, arr in maps.items():
        cv2.imwrite(os.path.join(hdrdir, f"{name}.hdr"), np.ascontiguousarray(arr[..., ::-1]))
    # the model: the rotated G=24 fixture, saved as a reference checkpoint
    fx = load_fixture("rotated_g24.pt")
    m = build_rotated(rot, G=fx["grid_size"][0], lights=[f"{r:03d}" for r in fx["light_rotation"]])
    m.load_state_dict(fx["state_dict"])
    m.alphaMask = rot.AlphaGridMask('cpu', fx["alpha_aabb"], fx["alpha_volume"])
    ckpt = os.path.join(tmp, "model.th")
    m.save(ckpt)

    # recorders
    draws, writes, ssims, accs, ratios = [], [], [], [], []
    multinomial = torch.multinomial

    def rec_multinomial(*a, **k):
        r = multinomial(*a, **k)
        draws.append(r.clone())
        return r
    RI.torch.multinomial = rec_multinomial       # RI.torch is the torch module: restored below
    load = torch.load
    RI.torch.load = lambda *a, **k: load(*a, **dict(k, weights_only=False))   # the checkpoint written just above
    env_cls = RI.Environment_Light
    RI.Environment_Light = lambda path: env_cls(path, device='cpu')
    save = os.path.join(tmp, "out")
    imageio = types.SimpleNamespace()

    def imwrite(path, arr):
        writes.append((os.path.relpath(path, save), np.asarray(arr).copy()))
    imageio.imwrite = imwrite
    imageio.mimsave = lambda *a, **k: None
    imageio.v2 = types.SimpleNamespace(imread=lambda path: dict(writes)[os.path.relpath(path, save)])
    RI.imageio = imageio
    ssim = RI.rgb_ssim

    def rec_ssim(a, b, max_val):
        v = ssim(a, b, max_val)
        ssims.append(float(v))
        return v
    RI.rgb_ssim = rec_ssim
    RI.rgb_lpips = lambda *a, **k: 0.0            # no lpips weights: a constant stands in
    crr = RI.compute_rescale_ratio

    def rec_ratio(*a, **k):
        r = crr(*a, **k)
        ratios.append(tuple(t.clone() for t in r))
        return r
    RI.compute_rescale_ratio = rec_ratio
    fwd = rot.TensorVMSplit.forward

    def rec_forward(self, *a, **k):
        r = fwd(self, *a, **k)
        accs.append(r[6].detach().clone())        # the primary acc, before relight() zeroes it in place
        return r
    rot.TensorVMSplit.forward = rec_forward
    RI.light_name_list = list(NAMES)

    ds = SyntheticViews(hemisphere_poses(2), H, W, light_names=NAMES)
    args = types.SimpleNamespace(ckpt=ckpt, model_name="TensorVMSplit", hdrdir=hdrdir, geo_buffer_path=save,
                                 batch_size=BATCH, if_save_rgb=False, if_save_depth=False, if_save_acc=True,
                                 if_save_rgb_video=False, if_save_relight_rgb=True, if_save_albedo=True,
                                 if_save_albedo_gamma_corrected=True, acc_mask_threshold=0.5, if_render_normal=True,
                                 vis_equation='nerv', render_video=True)
    torch.manual_seed(20211202)
    np.random.seed(20211202)
    video_error = None
    try:
        RI.relight(ds, args)
    except ValueError as e:
        # the normal video (relight_importance.py:302-304) broadcasts mask[..., 3:4] (column 3 of the [H,W] mask)
        # against the image rows: it raises for non-square images after everything else has been written
        video_error = str(e)
    finally:
        RI.torch.multinomial = multinomial
        RI.torch.load = load
        rot.TensorVMSplit.forward = fwd
    n_chunks = -(-H * W // BATCH)
    prim = accs[-len(ds) * n_chunks:]
    idx = torch.cat([d.reshape(-1) for d in draws]).numpy()
    assert idx.max() < 32768
    out = {
        "H": H, "W": W, "batch_size": BATCH, "light_names": list(NAMES), "hdr": maps, "n_samples": 512,
        "draw_shapes": [tuple(d.shape) for d in draws],
        "draws_int16_xz": lzma.compress(idx.astype(np.int16).tobytes(), preset=9),
        "writes": writes, "ssim": ssims,
        "rescale_ratio": ratios[0],
        "acc": [torch.cat(prim[v * n_chunks:(v + 1) * n_chunks]) for v in range(len(ds))],
        "psnr_view": [open(os.path.join(save, f"test_{v:03d}", "relighting_without_bg", "relight_psnr.txt")).read()
                      for v in range(len(ds))],
        "psnr_all": open(os.path.join(save, "relight_psnr.txt")).read(),
        "video_error": video_error,
    }
    shutil.rmtree(tmp)
    path = os.path.join(HERE, "relight_reference.pt")
    torch.save(out, path)
    print("relight_reference.pt", os.path.getsize(path) // 1024, "KiB;", len(draws), "draws,", len(writes), "writes")


if __name__ == "__main__":
    if REF is None or not os.path.isdir(REF):
        raise SystemExit(__doc__)
    relight_fixture()
