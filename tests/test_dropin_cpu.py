"""The drop-in tree exposes the reference's import surface (train_tensoIR.py:11-12)."""
import importlib
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dropin_import_surface():
    sys.path.insert(0, os.path.join(REPO, "dropin"))
    try:
        for m in ("models", "models.tensoRF_rotated_lights", "models.relight_utils", "renderer"):
            sys.modules.pop(m, None)
        rot = importlib.import_module("models.tensoRF_rotated_lights")
        for n in ("raw2alpha", "TensorVMSplit", "AlphaGridMask"):
            assert hasattr(rot, n)
        gen = importlib.import_module("models.tensoRF_general_multi_lights")
        assert issubclass(gen.TensorVMSplit, rot.TensorVMSplit)
        ini = importlib.import_module("models.tensoRF_init")
        assert hasattr(ini, "TensorVMSplit")
        ru = importlib.import_module("models.relight_utils")
        for n in ("render_with_BRDF", "compute_transmittance", "compute_radiance", "GGX_specular",
                  "linear2srgb_torch", "compute_secondary_shading_effects"):
            assert hasattr(ru, n)
        rnd = importlib.import_module("renderer")
        assert hasattr(rnd, "Renderer_TensoIR_train") and hasattr(rnd, "OctreeRender_trilinear_fast")
    finally:
        sys.path.remove(os.path.join(REPO, "dropin"))
        for m in ("models", "models.tensoRF_rotated_lights", "models.tensoRF_general_multi_lights",
                  "models.tensoRF_init", "models.relight_utils", "renderer"):
            sys.modules.pop(m, None)


def _reference_fixture():
    import torch
    return torch.load(os.path.join(REPO, "tests", "golden", "dropin_reference.pt"), weights_only=False)


# names the drop-in renderer takes from the reference's own renderer.py when that is importable (evaluation loops)
REFERENCE_EVAL_ONLY = {"compute_rescale_ratio"}


def test_reference_importers_resolve_against_dropin():
    """Every `from models.* / renderer import ...` of the reference's scripts and data loaders (recorded from the
    reference in tests/golden/dropin_reference.pt, e.g. dataLoader/tensoIR_rotation_setting.py:13,
    tensoIR_simple.py:12, tensoIR_general_multi_lights.py:13) finds its module and names when dropin/ shadows models/."""
    imports = _reference_fixture()["imports"]
    assert len(imports) >= 10 and any(f.startswith("dataLoader/") for f, _, _ in imports)
    sys.path.insert(0, os.path.join(REPO, "dropin"))
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.")
             or k == "renderer"}
    try:
        for f, module, names in imports:
            mod = importlib.import_module(module)
            assert mod.__file__.startswith(os.path.join(REPO, "dropin")), (f, module, mod.__file__)
            for n in names:
                assert n == "*" or n in REFERENCE_EVAL_ONLY or hasattr(mod, n), (f, module, n)
        ru = importlib.import_module("models.relight_utils")
        for n in ("read_hdr", "Environment_Light", "grid_sample", "compute_visibility",
                  "compute_visibility_and_indirect_light", "sample_ray_equally", "render_with_BRDF", "np", "F", "os"):
            assert hasattr(ru, n), n
    finally:
        sys.path.remove(os.path.join(REPO, "dropin"))
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.") or k == "renderer"]:
            sys.modules.pop(k)
        sys.modules.update(saved)


def test_grid_sample_matches_torch_inside_and_clamps_outside():
    """relight_utils.grid_sample == F.grid_sample(align_corners=True) inside [-1,1]; outside it extrapolates from the
    clamped border taps instead of zero padding (SURVEY.md §8c)."""
    import torch
    import torch.nn.functional as F
    from tensoir_b200.relight_utils import grid_sample
    g = torch.Generator().manual_seed(0)
    img = torch.randn(2, 5, 7, 9, generator=g, requires_grad=True)
    grid = torch.rand(2, 6, 4, 2, generator=g) * 1.96 - 0.98
    a, b = grid_sample(img, grid), F.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=True)
    assert torch.allclose(a, b, atol=1e-5)
    ga, = torch.autograd.grad(a.sum(), img)
    gb, = torch.autograd.grad(b.sum(), img)
    assert torch.allclose(ga, gb, atol=1e-5)
    # a W=1 "line": x coordinate beyond the border keeps the border value (weights sum to 1 with clamped taps)
    line = torch.arange(4.).view(1, 1, 4, 1)
    out = grid_sample(line, torch.tensor([[[[0.0, 1.5]]]]))
    assert torch.isfinite(out).all()
    # outside [-1, 1]: the reference's own grid_sample on the same inputs (tests/golden/dropin_reference.pt)
    ref = _reference_fixture()["grid_sample"]
    assert torch.allclose(grid_sample(ref["img"], ref["wide"]), ref["out"], atol=1e-5)
