"""The oracle restatement vs. the real reference on a shrunk, upsampled, non-cubic field (fixture made by
tests/golden/make_shrunk_golden.py): grid 30x31x29 on an aabb whose three axes differ, with the alpha mask either still
24^3 on the old +-1.5 box (state A) or 29x31x30 on the shrunk box (state B).  CPU only; bit-exact like
test_oracle_golden.py (gradients 1e-6, as there), so the GPU tests may use the oracle on these shapes."""
import pytest
import torch

from oracle import tensoir_oracle as O
from gpu_helpers import load_shrunk_state
from helpers import oracle_field, named_oracle_params
from test_oracle_golden import eq

STATES = ("A", "B")


@pytest.fixture(scope="module", params=STATES)
def fx(request):
    return load_shrunk_state(request.param)


def test_fixture_shapes(fx):
    """The shapes the fixture exists for: nothing cubic, no two axes alike."""
    assert fx["grid_size"] == [30, 31, 29] and fx["nSamples"] == 101
    size = fx["aabb"][1] - fx["aabb"][0]
    assert len(set(size.tolist())) == 3
    vol = tuple(fx["alpha_volume"].shape[-3:])
    if fx["state"] == "A":
        assert vol == (24, 24, 24) and torch.equal(fx["alpha_aabb"], torch.tensor([[-1.5] * 3, [1.5] * 3]))
    else:
        assert vol == (29, 31, 30) and torch.equal(fx["alpha_aabb"], fx["aabb"])
    assert 0 < float(fx["alpha_volume"].mean()) < 1


def test_unit_functions(fx):
    f = oracle_field(fx)
    pts = fx["pts"]
    xn = O.normalize_coord(f, pts)
    assert bool((xn.abs() > 1).any())                   # some points leave the box: zero-padding taps
    eq(O.sample_alpha(f, pts), fx["sample_alpha"])
    eq(O.density_feature(f, xn), fx["density_feature"])
    eq(O.feature2density(f, O.density_feature(f, xn)), fx["sigma"])
    rad, intr = O.both_feature(f, xn, fx["li"])
    eq(rad, fx["rad_feat"])
    eq(intr, fx["intr_feat"])
    eq(O.app_feature(f, xn, fx["li"]), fx["app_feat"])
    eq(O.intrin_feature(f, xn), fx["intrin_only"])
    eq(O.mlp_render_fea(f, f.mlp_rgb, fx["viewdirs"], rad), fx["mlp_rgb"])
    eq(O.mlp_pe_and_feature(f, f.mlp_brdf, xn, intr, torch.sigmoid), fx["mlp_brdf"])
    eq(O.mlp_pe_and_feature(f, f.mlp_normal, xn, intr, torch.tanh), fx["mlp_normal"])
    assert bool((fx["xj"].abs() > 1).any())             # clamped sampler outside [-1, 1]
    eq(O.derived_normals(f, fx["xj"].clone()).detach(), fx["derived_normals"])


def test_sample_ray(fx):
    f = oracle_field(fx)
    rays = fx["rays"]
    _, _, _, step, n = f.derived()
    assert n == fx["nSamples"] and float(step) == fx["stepSize"]
    for got, want in zip(O.sample_ray(f, rays[:, :3], rays[:, 3:6], False, -1), fx["sample_ray_eval"]):
        eq(got, want)
    for got, want in zip(O.sample_ray(f, rays[:, :3], rays[:, 3:6], True, 40, jitter=fx["jitter40"]),
                         fx["sample_ray_train"]):
        eq(got, want)


def test_secondary(fx):
    f = oracle_field(fx)
    for g, w in zip(O.compute_transmittance(f, fx["surf"], fx["dirs"], 96, 0.05, 1.5), fx["transmittance"]):
        eq(g, w)
    for g, w in zip(O.compute_radiance(f, fx["surf"], fx["dirs"], fx["li2"], 96, 0.05, 1.5), fx["radiance"]):
        eq(g, w)
    assert f.counters["density"] > 0 and f.counters["app"] > 0


def test_boundary_eval(fx):
    f = oracle_field(fx)
    torch.manual_seed(102)
    got = O.renderer_train(f, fx["rays"], fx["light_idx"], -1, True, False, True, 'fixed_envirmap', 160000, 24)
    for k, w in fx["renderer_eval"].items():
        eq(got[k].detach(), w)
    assert float(fx["renderer_eval"]["acc_map"].max()) > 0.5         # the rays hit the shrunk scene


def test_boundary_train_with_grads(fx):
    f = oracle_field(fx, requires_grad=True)
    torch.manual_seed(fx["train_seed"])
    got = O.renderer_train(f, fx["rays"], fx["light_idx"], 60, True, True, True, 'stratified_sampling', 160000, 24)
    for k, w in fx["renderer_train"].items():
        eq(got[k].detach(), w)
    target = torch.full_like(got["rgb_map"], 0.5)
    loss = (((got["rgb_map"] - target) ** 2).mean() + 0.2 * ((got["rgb_with_brdf_map"] - target) ** 2).mean()
            + 0.0005 * got["normals_diff_map"].mean() + 0.001 * got["normals_orientation_loss_map"].mean()
            + 0.001 * got["albedo_smoothness_loss"] + 0.001 * got["roughness_smoothness_loss"])
    loss.backward()
    eq(loss.detach(), fx["renderer_train_loss"])
    params = named_oracle_params(f)
    n_checked = 0
    for k, g in fx["renderer_train_grads"].items():
        if g is None:
            assert params[k].grad is None or float(params[k].grad.abs().max()) == 0.0
            continue
        eq(params[k].grad, g, tol=1e-6)
        n_checked += 1
    assert n_checked >= 20


def test_update_alpha_mask_on_the_shrunk_field():
    """updateAlphaMask(gridSize) from state A gives state B's volume and aabb."""
    a, b = load_shrunk_state("A"), load_shrunk_state("B")
    f = oracle_field(a)
    new_aabb = O.update_alpha_mask(f, tuple(a["grid_size"]))
    eq(f.alpha_volume, b["alpha_volume"])
    eq(f.alpha_aabb, b["alpha_aabb"])
    eq(new_aabb, b["new_aabb"])
