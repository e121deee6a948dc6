"""GPU parity on a shrunk, upsampled, non-cubic field (tests/golden/shrunk_g30*.pt, made by make_shrunk_golden.py):
grid 30x31x29 on an aabb whose three axes differ, alpha mask 24^3 on the old +-1.5 box (state A) or 29x31x30 on the
shrunk box (state B).  These are the shapes a training run has after its first updateAlphaMask + shrink; on a cubic
grid with a symmetric box a swapped axis, scale or box would go unnoticed.

The checks and tolerances are test_gpu_parity.py's: unit kernels 2e-5 / 5e-5 relative, maps 1e-4 relative, every
parameter gradient 5e-4 of its max, sample lists and counts exact.  The oracle (bit-exact against this fixture on the
CPU, test_oracle_shrunk_golden.py) supplies the references the fixture does not store."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import tensoir_oracle as O                        # noqa: E402
from helpers import oracle_field                             # noqa: E402
from gpu_helpers import app_mlp_list, load_shrunk_state, model_from_fixture, renderer_args   # noqa: E402
from test_gpu_parity import DEV, TOL, _train_loss, close      # noqa: E402


@pytest.fixture(scope="module", params=("A", "B"))
def shr(request):
    from tensoir_b200 import _lib
    _lib.load()
    fx = load_shrunk_state(request.param)
    return fx, model_from_fixture(fx, DEV)


def test_device_geometry_follows_every_axis(shr):
    """The TirField the kernels get: per-axis grid, aabb and inverse size of the field and of the alpha mask."""
    from tensoir_b200 import ops
    fx, m = shr
    f = ops.device_field(m).refresh(m)
    lo, hi = fx["aabb"][0].tolist(), fx["aabb"][1].tolist()
    alo, ahi = fx["alpha_aabb"][0].tolist(), fx["alpha_aabb"][1].tolist()
    Z, Y, X = fx["alpha_volume"].shape[-3:]
    assert list(f.grid) == fx["grid_size"] and list(f.agrid) == [X, Y, Z]
    # the step of a model on the GPU is the reference's (CPU) value bit for bit: every sample position depends on it
    assert float(m.stepSize) == fx["stepSize"] and m.nSamples == fx["nSamples"]
    for i in range(3):
        assert f.aabb_lo[i] == pytest.approx(lo[i], abs=1e-6) and f.aabb_hi[i] == pytest.approx(hi[i], abs=1e-6)
        assert f.inv_aabb[i] == pytest.approx(2.0 / (hi[i] - lo[i]), rel=1e-6)
        assert f.a_lo[i] == pytest.approx(alo[i], abs=1e-6)
        assert f.a_inv[i] == pytest.approx(2.0 / (ahi[i] - alo[i]), rel=1e-6)
        cell = (ahi[i] - alo[i]) / ([X, Y, Z][i] - 1)          # the occupied-cell box reaches at most a cell past the mask
        assert alo[i] - cell - 1e-5 <= f.occ_lo[i] < f.occ_hi[i] <= ahi[i] + cell + 1e-5


def test_unit_kernels(shr):
    from tensoir_b200 import ops
    from tensoir_b200.device_field import mlp_struct
    fx, m = shr
    pts = fx["pts"].to(DEV)
    xn = m.normalize_coord(pts)
    assert torch.equal(ops.alpha_mask_points(m, pts).cpu(), fx["sample_alpha"] > 0)
    feat, sig = ops.density_points(m, xn)
    close(feat, fx["density_feature"], 2e-5, "density_feature")
    close(sig, fx["sigma"], 2e-5, "sigma")
    li = fx["li"].to(DEV)
    rad, intr = m.compute_bothfeature(xn, li)
    close(rad, fx["rad_feat"], 2e-5, "rad")
    close(intr, fx["intr_feat"], 2e-5, "intr")
    close(m.compute_appfeature(xn, li), fx["app_feat"], 2e-5, "app")
    close(m.compute_intrinfeature(xn), fx["intrin_only"], 2e-5, "intrin")
    # the three heads on the mma.sync kernel (tir_app_mlp_points_save), renderModule on the wgmma list kernel
    # (tir_app_mlp, one sample per ray at weight 1)
    vd = fx["viewdirs"].to(DEV)
    for head, light, x_in, want in (("renderModule", "index", vd, fx["mlp_rgb"]),
                                    ("renderModule_brdf", "mean", xn, fx["mlp_brdf"]),
                                    ("renderModule_normal", "mean", xn, fx["mlp_normal"])):
        out = ops.app_mlp_points(m, xn, x_in, li if light == "index" else None, head=head, light=light)
        close(out, want, 5e-5, f"{head} mma.sync")
    keep = []
    close(app_mlp_list(m, mlp_struct(m, "renderModule", keep), xn, vd, li), fx["mlp_rgb"], 5e-5, "renderModule wgmma")
    # derived-normal gradient, absolute vs its scale (as in test_gpu_parity.test_unit_kernels)
    from tensoir_b200.primary import _derived_normals
    from tensoir_b200 import vm_autograd as vm
    fo = oracle_field(fx)
    xj = fx["xj"].clone().requires_grad_(True)
    g_ref = torch.autograd.grad(O.feature2density(fo, O.density_feature_with_xyz_grad(fo, xj)).sum(), xj)[0]
    ft, dfdx = vm.density_feature_and_grad(m, fx["xj"].to(DEV))
    g_got = (torch.sigmoid(ft - 10)[:, None] * dfdx).cpu()
    assert float((g_got - g_ref).abs().max()) < 1e-4 * float(g_ref.abs().max())
    well = g_ref.norm(dim=-1) > 1e-3 * float(g_ref.norm(dim=-1).max())
    assert int(well.sum()) > 20
    close(_derived_normals(m, fx["xj"].to(DEV))[well.to(DEV)], fx["derived_normals"][well], 5e-4, "derived_normals")


def _edge_rays(m):
    """Rays aimed at the corners and edge midpoints of the occupied-cell box (the box the marches cull with), just
    inside and just outside it, from random directions."""
    from tensoir_b200 import ops
    f = ops.device_field(m).refresh(m)
    lo, hi = torch.tensor(list(f.occ_lo)), torch.tensor(list(f.occ_hi))
    g = torch.Generator().manual_seed(17)
    targets = []
    for c in range(27):
        sel = torch.tensor([c % 3, (c // 3) % 3, c // 9])
        if int((sel != 1).sum()) < 2:
            continue                                    # corners and edge midpoints only
        p = torch.where(sel == 0, lo, torch.where(sel == 2, hi, (lo + hi) / 2))
        for eps in (-2e-2, -1e-3, 1e-3, 2e-2):
            targets.append(p + eps * torch.where(sel == 0, -1.0, torch.where(sel == 2, 1.0, 0.0)))
    t = torch.stack(targets)
    d = torch.nn.functional.normalize(torch.randn(t.shape[0], 3, generator=g), dim=-1)
    return torch.cat([t - 4.0 * d, d], 1)


@pytest.mark.parametrize("bricks", [True, False])
def test_valid_sample_lists_bit_exact(shr, bricks, monkeypatch):
    from tensoir_b200 import _lib, vm_autograd as vm
    fx, m = shr
    if not bricks:
        monkeypatch.setattr(_lib, "MARCH_CELL_BRICKS", 0)
    f = oracle_field(fx)
    edge = _edge_rays(m)
    for rays, cases in ((fx["rays"], ((False, -1, None), (True, 40, fx["jitter40"]))),
                        (edge, ((False, -1, None), (True, 60, torch.rand(edge.shape[0], 1,
                                                                        generator=torch.Generator().manual_seed(3)))))):
        for is_train, ns, jit in cases:
            pts, z, valid = O.sample_ray(f, rays[:, :3], rays[:, 3:6], is_train, ns, jitter=jit)
            valid = O._refine_valid(f, pts, valid)
            lst = vm.valid_samples(m, rays[:, :3].to(DEV), rays[:, 3:6].to(DEV), n_samples=ns,
                                   jitter=None if jit is None else jit.to(DEV))
            idx = valid.nonzero()
            assert idx.shape[0] > 0
            assert torch.equal(lst["ray"].cpu().long(), idx[:, 0])
            assert torch.equal(lst["sample"].cpu().long(), idx[:, 1])
            assert torch.equal(lst["z"].cpu(), z.expand(valid.shape)[valid])
            assert torch.equal(lst["xn"].cpu(), O.normalize_coord(f, pts)[valid])


def test_secondary_marches(shr):
    from tensoir_b200 import ops, relight_utils as RU
    fx, m = shr
    f = oracle_field(fx)
    surf, dirs, li2 = fx["surf"].to(DEV), fx["dirs"].to(DEV), fx["li2"].to(DEV)
    cnt = ops.new_counters(DEV)
    m.__dict__["_tir_counters"] = cnt
    try:
        nerv, nerf = RU.compute_transmittance(m, surf, dirs, nSample=96, vis_near=0.05, vis_far=1.5)
        close(nerv, fx["transmittance"][0], 2e-5, "nerv_vis")
        close(nerf, fx["transmittance"][1], 2e-5, "nerfactor_vis")
        O.compute_transmittance(f, fx["surf"], fx["dirs"], 96, 0.05, 1.5)
        c = ops.counters_dict(cnt)
        assert c["density"] == f.counters["density"] and c["mask"] == f.counters["mask"]
        cnt.zero_()
        f.counters.clear()
        nerv, nerf, ind = RU.compute_radiance(m, surf, dirs, li2, nSample=96, vis_near=0.05, vis_far=1.5)
        close(nerv, fx["radiance"][0], 2e-5, "radiance nerv")
        close(nerf, fx["radiance"][1], 2e-5, "radiance nerf")
        close(ind, fx["radiance"][2], TOL, "indirect")
        *_, app_mask, _ = O.compute_radiance(f, fx["surf"], fx["dirs"], fx["li2"], 96, 0.05, 1.5, return_aux=True)
        c = ops.counters_dict(cnt)
        assert c["overflow"] == 0
        assert (c["mask"], c["density"], c["app"]) == (f.counters["mask"], f.counters["density"], f.counters["app"])
        sm = m.__dict__["_tir_scratch"].samples()
        key = (sm["ray"].long() * 96 + sm["sample"].long()).cpu().sort().values
        want = app_mask.nonzero()
        assert torch.equal(key, (want[:, 0] * 96 + want[:, 1]).sort().values)
    finally:
        del m.__dict__["_tir_counters"]


def test_dense_secondary_vs_explicit(shr):
    """tir_secondary_radiance (point-major dense march over the packed mask and its bricks; in state B a 29x31x30 mask,
    so the last brick along every axis is partial) == compute_radiance on the expanded explicit ray list."""
    from tensoir_b200 import ops
    fx, m = shr
    f = oracle_field(fx)
    g = torch.Generator().manual_seed(4)
    lo, hi = fx["aabb"][0], fx["aabb"][1]
    pts = (lo + hi) / 2 + (hi - lo) / 2 * (torch.rand(9, 3, generator=g) * 2 - 1) * 0.9
    nrm = torch.nn.functional.normalize(torch.randn(9, 3, generator=g), dim=-1)
    li = (torch.arange(9) % 2).view(-1, 1).to(torch.int32)
    dirs = O.gen_light_incident_dirs(f, 'fixed_envirmap')
    vis, ind, _ = ops.secondary_radiance(m, pts.to(DEV), nrm.to(DEV), li.to(DEV), dirs.to(DEV), n_sample=24)
    cos = torch.clamp(torch.einsum("jk,ik->ij", dirs, nrm), min=0)
    mask = cos > 1e-6
    P = pts[:, None, :].expand(-1, dirs.shape[0], -1)[mask]
    D = dirs[None].expand(9, -1, -1)[mask]
    L = li.view(-1, 1, 1).expand(-1, dirs.shape[0], 1)[mask]
    v, _, i = O.compute_radiance(f, P, D, L, 24, 0.05, 1.5)
    want_v = torch.zeros(9, dirs.shape[0], 1)
    want_i = torch.zeros(9, dirs.shape[0], 3)
    want_v[mask] = v[:, None]
    want_i[mask] = i
    assert 0 < float(want_v.mean()) < 1
    close(vis, want_v, 2e-5, "vis")
    close(ind, want_i, TOL, "indirect")


def ill_conditioned_rays(fx, n_samples, jitter=None):
    """Rays whose normals_diff_map fp32 cannot pin down to TOL: 4 sum_s w_s |n32_s - n64_s| > TOL, with n32 / n64 the
    derived normals -normalize(d sigma / d x) of the fp32 and the float64 oracle and w_s the float64 weights (a unit
    normal moving by e moves |n_pred - n_derived|^2 by at most 4 e).  Where the density gradient is ~1e-7 of its size
    on the ray (flat density inside the solid boxes) it is a difference of tap sums that cancels to rounding noise and
    the fp32 normal has no direction: on this fixture the fp32 reference's own normal is up to ~1.9 away from the
    float64 one there, and the kernel's is as far.  normals_diff_map of those rays says nothing about the kernel."""
    f, f64 = oracle_field(fx), oracle_field(fx).to("cpu", torch.float64)
    rays = fx["rays"]
    pts, z, valid = O.sample_ray(f, rays[:, :3], rays[:, 3:6], jitter is not None, n_samples, jitter=jitter)
    valid = O._refine_valid(f, pts, valid)
    xn = O.normalize_coord(f, pts[valid])
    x32 = xn.clone().requires_grad_(True)
    g32 = torch.autograd.grad(O.feature2density(f, O.density_feature_with_xyz_grad(f, x32)).sum(), x32)[0]
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        x64 = xn.double().requires_grad_(True)
        sigma = O.feature2density(f64, O.density_feature_with_xyz_grad(f64, x64))
        g64 = torch.autograd.grad(sigma.sum(), x64)[0]
        sig = torch.zeros(valid.shape)
        sig[valid] = sigma.detach()
        zz = z.double().expand(valid.shape)
        dist = torch.cat((zz[:, 1:] - zz[:, :-1], torch.zeros_like(zz[:, :1])), dim=-1) * f.distance_scale
        _, w, _ = O.raw2alpha(sig, dist)
    finally:
        torch.set_default_dtype(old)
    nrm = torch.nn.functional.normalize
    e = torch.zeros(valid.shape, dtype=torch.float64)
    e[valid] = (nrm(g32.double(), dim=-1) - nrm(g64, dim=-1)).norm(dim=-1)
    return 4 * (w * e).sum(1) > TOL


def close_maps(got, want, ill, what):
    """Every map at TOL; normals_diff_map at TOL on the rays whose derived normals are well conditioned, at most 1 ray in
    8 excluded (``ill_conditioned_rays``)."""
    assert int(ill.sum()) <= ill.numel() // 8, int(ill.sum())
    for k, w in want.items():
        if k == "normals_diff_map":
            close(got[k].reshape(-1)[~ill.to(got[k].device)], w.reshape(-1)[~ill], TOL, f"{what} {k}")
        else:
            close(got[k], w, TOL, f"{what} {k}")


def test_boundary_eval(shr):
    from tensoir_b200 import Renderer_TensoIR_train
    fx, m = shr
    torch.manual_seed(102)
    m.__dict__["_tir_randn_like"] = lambda t: torch.randn(t.shape).to(t.device)
    try:
        with torch.no_grad():
            got = Renderer_TensoIR_train(fx["rays"], None, fx["light_idx"], m, N_samples=-1, white_bg=True,
                                         is_train=False, is_relight=True, sample_method='fixed_envirmap',
                                         chunk_size=160000, device=DEV, args=renderer_args(24))
    finally:
        del m.__dict__["_tir_randn_like"]
    close_maps(got, fx["renderer_eval"], ill_conditioned_rays(fx, -1), "eval")


@pytest.mark.parametrize("state", ["A", "B"])
def test_boundary_train_step_grads(state):
    """Training-mode boundary + backward on the shrunk field: outputs and loss vs the reference, every parameter gradient
    at 5e-4 of its max (as in test_gpu_parity.test_boundary_train_step_grads).  The gradient of normals_diff_map goes
    through d normalize(g) / d g ~ 1 / |g|, so on the rays of ``ill_conditioned_rays`` it is rounding noise amplified
    ~1e5 times and swamps the density-factor gradients of the whole batch (~0.9 of their max, in the reference's fp32
    as much as here).  The gradients are therefore compared for the loss with those rays' normals_diff_map left out,
    against the oracle (bit-exact with the reference on this fixture, test_oracle_shrunk_golden.py) with the same
    random stream."""
    from tensoir_b200 import Renderer_TensoIR_train
    from helpers import named_oracle_params
    fx = load_shrunk_state(state)
    m = model_from_fixture(fx, DEV)
    m.__dict__["_tir_randn_like"] = lambda t: torch.randn(t.shape).to(t.device)
    torch.manual_seed(fx["train_seed"])
    got = Renderer_TensoIR_train(fx["rays"], None, fx["light_idx"], m, N_samples=60, white_bg=True, is_train=True,
                                 is_relight=True, sample_method='stratified_sampling', chunk_size=160000,
                                 device=DEV, args=renderer_args(24))
    jitter = torch.rand(fx["rays"].shape[0], 1, generator=torch.Generator().manual_seed(fx["train_seed"]))  # first draw
    ill = ill_conditioned_rays(fx, 60, jitter)
    close_maps(got, fx["renderer_train"], ill, "train")
    close(_train_loss(got), fx["renderer_train_loss"], TOL, "loss")

    def loss_without_ill(ret):
        keep = (~ill).to(ret["normals_diff_map"].device).reshape(ret["normals_diff_map"].shape)
        return _train_loss(dict(ret, normals_diff_map=ret["normals_diff_map"] * keep))
    loss_without_ill(got).backward()
    f = oracle_field(fx, requires_grad=True)
    torch.manual_seed(fx["train_seed"])
    want = O.renderer_train(f, fx["rays"], fx["light_idx"], 60, True, True, True, 'stratified_sampling', 160000, 24)
    loss_without_ill(want).backward()
    params = named_oracle_params(f)
    n, worst = 0, {}
    for k, p in m.named_parameters():
        w = params[k].grad
        if w is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        g = p.grad.detach().cpu()
        assert g.shape == w.shape, k
        worst[k] = float((g - w).abs().max()) / (float(w.abs().max()) + 1e-12)
        n += 1
    assert n >= 20
    bad = {k: v for k, v in worst.items() if v > 5e-4}
    assert not bad, (bad, max(worst.values()))


@pytest.mark.parametrize("kind", ["derived_plus_predicted", "purely_predicted", "purely_derived"])
def test_fused_primary_matches_modular_path(kind):
    """State B: the fused primary march against the modular autograd path, every map and parameter gradient (the
    tolerances of test_gpu_parity.test_fused_primary_matches_modular_path)."""
    from tensoir_b200 import Renderer_TensoIR_train
    fx = load_shrunk_state("B")
    rays, li = fx["rays"].to(DEV), fx["light_idx"].to(DEV)
    outs = []
    for modular in (True, False):
        m = model_from_fixture(fx, DEV)
        m.normals_kind = kind
        m.__dict__["_tir_modular"] = modular
        m.__dict__["_tir_randn_like"] = lambda t: torch.sin(t * 977.0)
        torch.manual_seed(11)
        got = Renderer_TensoIR_train(rays, None, li, m, N_samples=60, white_bg=True, is_train=True, is_relight=True,
                                     sample_method='stratified_sampling', device=DEV, args=renderer_args(24))
        loss = _train_loss(got) + 0.3 * got["acc_map"].mean() + 0.1 * got["depth_map"].mean() \
            + 0.05 * (got["albedo_map"] ** 2).mean() + 0.05 * (got["roughness_map"] ** 2).mean() \
            + 0.05 * (got["normal_map"][:, 2]).mean()
        loss.backward()
        outs.append((got, loss, {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}))
    (g0, l0, gr0), (g1, l1, gr1) = outs
    for k in g0:
        close(g1[k], g0[k], 2e-5, k)
    close(l1, l0, 2e-5, "loss")
    assert set(gr0) == set(gr1), set(gr0) ^ set(gr1)
    worst = {k: float((gr0[k] - gr1[k]).abs().max()) / (float(gr0[k].abs().max()) + 1e-12) for k in gr0}
    bad = {k: v for k, v in worst.items() if v > 2e-4}
    assert not bad, bad


def test_update_alpha_mask_from_state_a():
    """updateAlphaMask(gridSize) on the GPU from state A: the reference's state B volume (29x31x30 on the shrunk box)
    and new_aabb, exactly, as the cubic test_gpu_parity.test_update_alpha_mask_and_filtering requires."""
    a, b = load_shrunk_state("A"), load_shrunk_state("B")
    m = model_from_fixture(a, DEV)
    new_aabb = m.updateAlphaMask(tuple(a["grid_size"]))
    vol = m.alphaMask.alpha_volume.cpu()
    assert vol.shape[-3:] == b["alpha_volume"].shape[-3:]
    assert torch.equal(vol.view(b["alpha_volume"].shape), b["alpha_volume"]), int((vol.view(-1) != b["alpha_volume"].view(-1)).sum())
    close(m.alphaMask.aabb, b["alpha_aabb"], 1e-6, "alpha aabb")
    close(new_aabb, b["new_aabb"], 1e-6, "new_aabb")
