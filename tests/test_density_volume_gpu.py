"""The baked density volume of the secondary march (include/tensoir_b200.h, TirDensityVolume): the builder against a
float64 sum of the factor products, the volume path of the dense secondary march against the factor path on identical
inputs, the sub-box against the whole grid, and freshness after in-place parameter updates (fused Adam, CUDA-graph
replay)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from gpu_helpers import load_shrunk_state, model_from_fixture   # noqa: E402

DEV = "cuda:0"
EPS32 = 2.0 ** -23
# Weights of the volume path against the factor path.  sigma = softplus(feature - 10) with features of up to ~30 on
# these scenes: where the weight is small, its relative change is about the ABSOLUTE change of the feature, and the
# two paths round a sum of 48 products of that size differently (|feature error| <= 18 * eps32 * sum|P*L|, about
# 1e-4 at sum|P*L| = 50).  Measured on H100: at most 6e-4 relative, on weights near rayMarch_weight_thres (inside the
# 1e-7 absolute term), while two launches of the same path agree to 1e-6.
W_RTOL = 2e-4


def _factors(model):
    return [p.detach().clone() for p in model.density_plane], [l.detach().clone() for l in model.density_line]


def _grid(model):
    from tensoir_b200 import ops
    return list(ops.device_field(model).refresh(model).grid)


def _d64(factors, lo, n, slab=16):
    """sum_k sum_c plane_k[c] * line_k[c] at the vertices of the box, in float64 on the factors' device, ``slab`` z
    planes at a time -> (D, sum_k sum_c |plane*line|), both [n_z, n_y, n_x] on the CPU."""
    dev = factors[0][0].device
    P = [p.double()[0] for p in factors[0]]                    # [C, G[m1], G[m0]]
    L = [l.double()[0, :, :, 0] for l in factors[1]]           # [C, G[v]]
    xs, ys = (torch.arange(lo[a], lo[a] + n[a], device=dev) for a in range(2))
    D = torch.empty(n[2], n[1], n[0], dtype=torch.float64, device=dev)
    mag = torch.empty_like(D)
    for z0 in range(0, n[2], slab):
        zs = torch.arange(lo[2] + z0, lo[2] + min(n[2], z0 + slab), device=dev)
        terms = (torch.einsum("cyx,cz->czyx", P[0][:, ys][:, :, xs], L[0][:, zs]),
                 torch.einsum("czx,cy->czyx", P[1][:, zs][:, :, xs], L[1][:, ys]),
                 torch.einsum("czy,cx->czyx", P[2][:, zs][:, :, ys], L[2][:, xs]))
        D[z0:z0 + zs.numel()] = sum(t.sum(0) for t in terms)
        mag[z0:z0 + zs.numel()] = sum(t.abs().sum(0) for t in terms)
    return D.cpu(), mag.cpu()


def _built(model):
    """Extent + build through ops.density_volume -> (lo, n, D [n_z, n_y, n_x] on the CPU)."""
    from tensoir_b200 import ops
    f = ops.device_field(model).refresh(model)
    vol = ops.density_volume(model, f)
    torch.cuda.synchronize()
    lo, n = list(vol.lo), list(vol.n)
    buf = model.__dict__["_tir_density_vol"]
    return lo, n, buf[:n[0] * n[1] * n[2]].view(n[2], n[1], n[0]).cpu()


def _check_against_f64(factors, lo, n, got):
    """-> the largest err / bound"""
    want, mag = _d64(factors, lo, n)
    # recursive fp32 summation of 3 x 16 products (each rounded): |err| <= (16 + 2) * u * sum|terms|, u = eps32 / 2;
    # c = 18 with eps32 leaves a factor 2 of slack and does not depend on the summation order
    bound = EPS32 * 18 * mag
    err = (got.double() - want).abs()
    assert bool((err <= bound).all()), float((err - bound).max())
    assert float(want.abs().max()) > 0
    return float((err / bound.clamp_min(1e-300)).max())


@pytest.fixture(scope="module", params=("A", "B"))
def shrunk(request):
    fx = load_shrunk_state(request.param)
    return fx, model_from_fixture(fx, DEV)


def test_builder_matches_float64_on_shrunk_states(shrunk):
    _, m = shrunk
    lo, n, got = _built(m)
    assert all(n[a] >= 1 and lo[a] + n[a] <= _grid(m)[a] for a in range(3))
    _check_against_f64(_factors(m), lo, n, got)


def test_builder_matches_float64_on_a_non_cubic_random_field():
    """37 x 18 x 61 (no axis size repeats) with random factors and no alpha mask: the whole grid; a swapped axis in
    the builder's plane / line indexing cannot pass."""
    from tensoir_b200 import TensorVMSplit
    torch.manual_seed(3)
    m = TensorVMSplit(torch.tensor([[-1.0, -0.7, -1.3], [1.1, 0.8, 1.2]], device=DEV), [37, 18, 61], DEV,
                      density_n_comp=[16] * 3, appearance_n_comp=[48] * 3, app_dim=27, near_far=[2.0, 6.0],
                      shadingMode='MLP_Fea', density_shift=-10, distance_scale=25, pos_pe=2, view_pe=2, fea_pe=2,
                      featureC=128, step_ratio=0.5, fea2denseAct='softplus', normals_kind='derived_plus_predicted',
                      light_rotation=["000"], light_kind='sg', numLgtSGs=128)
    with torch.no_grad():
        for p in list(m.density_plane) + list(m.density_line):
            p.normal_()
    assert m.alphaMask is None
    lo, n, got = _built(m)
    assert (lo, n) == ([0, 0, 0], [37, 18, 61])
    _check_against_f64(_factors(m), lo, n, got)


# ---- the march: volume path against the factor path ---------------------------------------------------------------
def _march(model, pts, nrm, li, dirs, n_sample, vol=None, use_vol=True):
    """One tir_secondary_radiance(_vol) call with counters -> dict of outputs.  vol: a TirDensityVolume to read
    instead of the one ops.density_volume builds."""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.device_field import mlp_struct
    lib = _lib.load()
    f = ops.device_field(model).refresh(model)
    keep = []
    cfg = ops.march_cfg(model, table=ops.equal_z_table(n_sample, 0.05, 1.5, DEV), keep=keep)
    mlp = mlp_struct(model, "renderModule", keep, light="index")
    n_pts, n_dirs = pts.shape[0], dirs.shape[0]
    vis = torch.zeros(n_pts, n_dirs, 1, device=DEV)
    ind = torch.zeros(n_pts, n_dirs, 3, device=DEV)
    cnt = ops.new_counters(DEV)
    sc = ops.SampleScratch(DEV, max(1 << 16, 4 * n_pts * n_dirs))
    li32 = li.reshape(-1).to(torch.int32).contiguous()
    common = (_lib.dptr(pts), _lib.dptr(nrm), _lib.dptr(li32, torch.int32), n_pts, _lib.dptr(dirs), n_dirs,
              C.byref(cfg))
    tail = (_lib.dptr(vis), _lib.dptr(ind), _lib.dptr(sc.buf, torch.uint8), _lib.dptr(sc.count, torch.int32),
            sc.capacity, _lib.dptr(cnt, torch.int64), _lib.stream_ptr())
    if use_vol:
        v = vol if vol is not None else ops.density_volume(model, f)
        rc = lib.tir_secondary_radiance_vol(C.byref(f), C.byref(mlp), *common, C.byref(v), *tail)
    else:
        rc = lib.tir_secondary_radiance(C.byref(f), C.byref(mlp), *common, *tail)
    _lib.check(rc, "secondary radiance")
    torch.cuda.synchronize()
    sm = sc.samples()
    key = (sm["ray"].long() * n_sample + sm["sample"].long()).sort()
    return {"vis": vis, "ind": ind, "cnt": ops.counters_dict(cnt), "key": key.values,
            "w": sm["weight"][key.indices]}


def _compare(a, b, w_rtol):
    for k in ("mask", "density", "rays", "overflow"):
        assert a["cnt"][k] == b["cnt"][k], k
    assert a["cnt"]["overflow"] == 0
    same, same_b = torch.isin(a["key"], b["key"]), torch.isin(b["key"], a["key"])
    # the association order of the transmittance scan differs between launches (atomics), and the two density paths
    # round differently: at most a sample whose weight rounds across rayMarch_weight_thres
    assert int((~same).sum()) + int((~same_b).sum()) <= 2
    wa, wb = a["w"][same], b["w"][same_b]
    rel_w = float(((wa - wb).abs() / wb.abs().clamp_min(1e-30)).max())
    d_vis = float((a["vis"] - b["vis"]).abs().max())
    d_ind = float(((a["ind"] - b["ind"]).abs() / (1 + b["ind"].abs())).max())
    print(f"max relative weight difference {rel_w:.3e}, vis {d_vis:.3e}, indirect {d_ind:.3e}")
    assert torch.allclose(wa, wb, rtol=w_rtol, atol=1e-7)
    assert d_vis <= 1e-5
    assert d_ind <= 1e-4


def _lego_inputs(grid=128, n_rays=1024, m=None):
    """A lego model (``m``, or make_lego_model(grid)) and the surface points, normals and light ids its own forward
    gives on a training batch, with the step's 512 stratified directions."""
    from tensoir_b200.synthetic import make_lego_model, hemisphere_poses, training_batch, n_samples_for
    if m is None:
        m = make_lego_model(grid, DEV)
    grid = int(m.gridSize[0])
    rays, li = (t.to(DEV) for t in training_batch(hemisphere_poses(100), n_rays, 3))
    with torch.no_grad():
        out = m(rays, li, is_train=False, is_relight=True, N_samples=n_samples_for(grid))
    depth, normal, acc_mask = out[1], out[2], out[9]
    hit = acc_mask.reshape(-1).bool()
    surf = (rays[:, :3] + depth.reshape(-1, 1) * rays[:, 3:])[hit].contiguous()
    dirs = m.gen_light_incident_dirs(method='stratified_sampling').to(DEV).contiguous()
    return m, surf, normal[hit].contiguous(), li.reshape(-1)[hit].contiguous(), dirs


def _shrunk_inputs(fx, m):
    from oracle import tensoir_oracle as O
    from helpers import oracle_field
    g = torch.Generator().manual_seed(4)
    lo, hi = fx["aabb"][0], fx["aabb"][1]
    pts = (lo + hi) / 2 + (hi - lo) / 2 * (torch.rand(64, 3, generator=g) * 2 - 1) * 0.9
    nrm = torch.nn.functional.normalize(torch.randn(64, 3, generator=g), dim=-1)
    li = (torch.arange(64) % 2).to(torch.int32)
    dirs = O.gen_light_incident_dirs(oracle_field(fx), 'fixed_envirmap')
    return pts.to(DEV), nrm.to(DEV), li.to(DEV), dirs.to(DEV).contiguous()


def volume_path_matches_factor_path(m, surf, nrm, li, dirs):
    assert dirs.shape[0] == 512 and surf.shape[0] > 50
    fac = _march(m, surf, nrm, li, dirs, 96, use_vol=False)
    vol = _march(m, surf, nrm, li, dirs, 96)
    assert fac["cnt"]["density"] > 10000 and fac["cnt"]["app"] > 1000
    _compare(vol, fac, W_RTOL)


def test_volume_path_matches_factor_path_on_lego_128():
    volume_path_matches_factor_path(*_lego_inputs())


def test_volume_path_matches_factor_path_on_shrunk_states(shrunk):
    fx, m = shrunk
    pts, nrm, li, dirs = _shrunk_inputs(fx, m)
    fac = _march(m, pts, nrm, li, dirs, 96, use_vol=False)
    vol = _march(m, pts, nrm, li, dirs, 96)
    assert fac["cnt"]["density"] > 0
    _compare(vol, fac, W_RTOL)


# ---- the sub-box against the whole grid ---------------------------------------------------------------------------
def _whole_grid_volume(model, poison_outside=None):
    """The volume over the whole grid in a buffer of its own; with poison_outside=(lo, n), every vertex outside that
    box is NaN, so a march that reads one of them produces NaN."""
    from tensoir_b200 import _lib, ops
    lib = _lib.load()
    f = ops.device_field(model).refresh(model)
    G = list(f.grid)
    buf = torch.empty(G[2], G[1], G[0], device=DEV)
    v = _lib.TirDensityVolume()
    v.data, v.lo[:], v.n[:] = buf.data_ptr(), [0, 0, 0], G
    _lib.check(lib.tir_density_volume_build(C.byref(f), C.byref(v), buf.numel(), _lib.stream_ptr()), "build")
    if poison_outside is not None:
        lo, n = poison_outside
        keep = buf[lo[2]:lo[2] + n[2], lo[1]:lo[1] + n[1], lo[0]:lo[0] + n[0]].clone()
        buf.fill_(float("nan"))
        buf[lo[2]:lo[2] + n[2], lo[1]:lo[1] + n[1], lo[0]:lo[0] + n[0]] = keep
    return v, buf


@pytest.mark.parametrize("scene", ["lego", "A", "B"])
def test_sub_box_holds_every_vertex_a_valid_sample_reads(scene):
    """The march over the extent's sub-box gives what the march over the whole-grid volume gives, and with every
    vertex outside the sub-box set to NaN the whole-grid march stays finite: no valid sample reads outside it."""
    if scene == "lego":
        m, pts, nrm, li, dirs = _lego_inputs()
    else:
        fx = load_shrunk_state(scene)
        m = model_from_fixture(fx, DEV)
        pts, nrm, li, dirs = _shrunk_inputs(fx, m)
    sub_box_holds_every_vertex_a_valid_sample_reads(m, pts, nrm, li, dirs, proper=scene == "lego")


def sub_box_holds_every_vertex_a_valid_sample_reads(m, pts, nrm, li, dirs, proper):
    """``proper``: the extent must be smaller than the grid"""
    lo, n, _ = _built(m)
    assert all(n[a] >= 1 for a in range(3))
    if proper:
        assert n != _grid(m)                                    # the box really is a sub-box here
    sub = _march(m, pts, nrm, li, dirs, 96)
    v_full, buf_full = _whole_grid_volume(m)
    full = _march(m, pts, nrm, li, dirs, 96, vol=v_full)
    v_pois, buf_pois = _whole_grid_volume(m, poison_outside=(lo, n))
    pois = _march(m, pts, nrm, li, dirs, 96, vol=v_pois)
    assert bool(torch.isfinite(pois["vis"]).all()) and bool(torch.isfinite(pois["ind"]).all())
    for other in (full, pois):
        _compare(sub, other, 1e-5)


def test_mask_without_occupied_cells_and_model_without_mask():
    """No occupied cell: the field has no box, the extent is the whole grid and nothing is valid.  No alpha mask: the
    extent is the whole grid and the volume path matches the factor path."""
    from tensoir_b200 import AlphaGridMask
    fx = load_shrunk_state("A")
    m = model_from_fixture(fx, DEV)
    pts, nrm, li, dirs = _shrunk_inputs(fx, m)
    m.alphaMask = AlphaGridMask(DEV, fx["alpha_aabb"].to(DEV), torch.zeros_like(fx["alpha_volume"]).to(DEV))
    lo, n, _ = _built(m)
    assert (lo, n) == ([0, 0, 0], _grid(m))
    r = _march(m, pts, nrm, li, dirs, 96)
    assert r["cnt"]["density"] == 0 and r["cnt"]["app"] == 0
    assert bool((r["vis"][r["vis"] != 0] == 1).all()) and float(r["ind"].abs().max()) == 0
    m.alphaMask = None
    lo, n, got = _built(m)
    assert (lo, n) == ([0, 0, 0], _grid(m))
    _check_against_f64(_factors(m), lo, n, got)
    _compare(_march(m, pts, nrm, li, dirs, 96), _march(m, pts, nrm, li, dirs, 96, use_vol=False), W_RTOL)


# ---- freshness ------------------------------------------------------------------------------------------------------
def test_volume_follows_a_fused_adam_step():
    """A fused Adam step updates the density factors in place without a version bump.  The next secondary_radiance
    reads the new factors: it equals that of a model built fresh from the updated state."""
    from tensoir_b200 import ops
    fx = load_shrunk_state("B")
    m = model_from_fixture(fx, DEV)
    pts, nrm, li, dirs = _shrunk_inputs(fx, m)
    li = li.view(-1, 1)
    ops.secondary_radiance(m, pts, nrm, li, dirs)                 # the volume buffer exists and holds the old field
    params = list(m.density_plane) + list(m.density_line)
    versions = [p._version for p in params]
    opt = torch.optim.Adam(params, lr=0.05, fused=True)
    torch.manual_seed(9)
    for p in params:
        p.grad = torch.randn_like(p)                              # same memory format as the parameter
    opt.step()
    assert [p._version for p in params] == versions               # in place, invisible to the version counter
    vis, ind, _ = ops.secondary_radiance(m, pts, nrm, li, dirs)
    fresh = model_from_fixture(fx, DEV)
    with torch.no_grad():
        for p, q in zip(list(fresh.density_plane) + list(fresh.density_line), params):
            p.copy_(q)
    vis2, ind2, _ = ops.secondary_radiance(fresh, pts, nrm, li, dirs)
    torch.cuda.synchronize()
    assert float((vis - vis2).abs().max()) <= 1e-5
    assert bool(((ind - ind2).abs() <= 1e-4 * (1 + ind2.abs())).all())
    lo, n, got = _built(m)
    _check_against_f64(_factors(m), lo, n, got)


def test_graph_replay_builds_from_the_parameters_the_previous_replay_wrote():
    """In a CUDA-graph training step the volume build is a node of the graph: after replay k the volume holds the
    field of the parameters replay k-1's Adam wrote (the forward runs before this replay's own update)."""
    from test_gpu_parity import _train_loss
    from gpu_helpers import load_fixture, renderer_args
    from tensoir_b200.static_step import StaticTrainStep
    fx = load_fixture("rotated_g24.pt")
    m = model_from_fixture(fx, DEV)
    opt = torch.optim.Adam(m.get_optparam_groups(0.02, 0.001), betas=(0.9, 0.99), fused=True, capturable=True)
    rays, li = fx["rays"].to(DEV), fx["light_idx"].to(DEV)
    st = StaticTrainStep(m, opt, 64, 60, renderer_args(24), lambda ret, mm: _train_loss(ret), device=DEV)
    st.calibrate([(rays, li)])
    st.capture(warmup=1)
    buf = m.__dict__["_tir_density_vol"]
    assert any(buf is k for k in st._keepalive)
    from tensoir_b200 import _lib, ops
    f = ops.device_field(m).refresh(m)
    lo, n = (C.c_int32 * 3)(), (C.c_int32 * 3)()
    _lib.check(_lib.load().tir_density_volume_extent(C.byref(f), lo, n), "extent")
    lo, n = list(lo), list(n)
    prev = None
    for _ in range(3):
        torch.cuda.synchronize()
        before = _factors(m)
        st.run(rays, li)
        torch.cuda.synchronize()
        got = buf[:n[0] * n[1] * n[2]].view(n[2], n[1], n[0]).cpu()
        _check_against_f64(before, lo, n, got)
        if prev is not None:
            assert not torch.equal(got, prev)                      # Adam moved the field and the build followed
        prev = got
    st.flush()
    assert st.overflowed() == 0
    st.release()
