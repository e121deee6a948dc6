"""The float64 stage checks of the training step, run on the benchmark's own configuration: bench.py's model and batch
(config 2, make_lego_model(300): a 300^3 VM grid under a 256^3 alpha mask, a 4 096-ray training_batch(.., 0) of
hemisphere_poses(100), n_samples_for(300) = 1 039 samples, 512 stratified secondary directions x 96 samples, the
marches in lean-counter mode).  The other float64 files check the same kernels on the lego field at 128^3 or below,
where the mask and the field have the same size, the brick summary is 16^3 bits, rays are at most a few 32-sample
chunks long and texel coordinates stay below 128; what the metric measures runs at none of those.

No reference is new here: every case runs a check of another file on the 300 model.
  * the shape itself (VM grid, mask, samples, brick geometry, the valid samples per ray against the 128 field);
  * the primary path (test_primary_kernels_fp64): the four entry points with random map gradients, and the dumps of
    real eager steps (test_train_step_primary_fp64.captured_step): the relight step bench.py times, phase 1, and the
    relight step of config 4 (general model, lights sunset / snow / courtyard);
  * the dense secondary march and its list MLP (test_secondary_kernels_fp64.launch_dense / check_dense) on surface
    points of the 300 model's own forward: the step's instance (volume, z table, N = 96, 512 directions, lean), 128
    directions as config 3 uses (8 x 16), and one count-parity launch (mask, density and app counters exact);
  * the density volume (test_density_volume_gpu): the builder against float64 on the extent's box, the sub-box
    check, and the volume path against the factor path;
  * the VM gradient scatters (test_vm_scatter_runs_gpu) of the density and appearance products on the 4 096-ray valid
    list of the 300 field, with its own factors, in ray order and shuffled.

Measured on an H100: the bench batch has 1 917 rays without a valid sample; of the others the median ray has 111 valid
samples, the longest 460 (15 chunks of 32), against 197 on the 128 field with the same rays.  The 300 model and its
batch are built once per module; every case prints its wall time and the peak device memory
the process allocated while it ran."""
import contextlib
import io
import time
import types

import pytest
import torch

import test_density_volume_gpu as DV
import test_primary_kernels_fp64 as P
import test_secondary_kernels_fp64 as S
import test_vm_kernels_fp64 as V
import test_vm_scatter_runs_gpu as VS
from gpu_helpers import renderer_args
from test_train_step_primary_fp64 import captured_step, own_stats, run

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GRID, MASK, N_RAYS = 300, 256, 4096
N_SAMPLES = 1039                  # n_samples_for(300)
BRICK_SHIFT, BRICK_BITS = 3, 32768


def _lego(**kw):
    from tensoir_b200.synthetic import make_lego_model
    with contextlib.redirect_stdout(io.StringIO()):
        return make_lego_model(GRID, DEV, **kw)


@pytest.fixture(scope="module")
def bench():
    """bench.build_model(config 2) and the first batch of bench.measure"""
    from tensoir_b200 import _lib
    from tensoir_b200.synthetic import hemisphere_poses, n_samples_for, training_batch
    _lib.load()
    t0 = time.perf_counter()
    m = _lego()
    rays, li = training_batch(hemisphere_poses(100), N_RAYS, 0)
    torch.cuda.synchronize()
    print(f"\n[cost] lego {GRID} model: {time.perf_counter() - t0:.1f} s")
    yield types.SimpleNamespace(m=m, rays=rays.to(DEV), li=li.to(DEV), n_samples=n_samples_for(GRID))
    S._SCENES.pop(("lego", id(m)), None)


@pytest.fixture(autouse=True)
def cost(request):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[cost] {request.node.name}: {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _lengths(m, rays, li, n_samples):
    """valid samples per ray of the march test_primary_stages_random_map_gradients launches (seed 3's jitter)"""
    cs = P.Case(m, rays, li, n_samples, 3)
    return P.march_reference(m, cs.rays, n_samples, cs.jitter, None)["counts"].long()


# ------------------------------------------------------------------------------------------------------------ shape
def test_bench_shape(bench):
    """What this file exists for: a change to make_lego_model or n_samples_for that shrinks the configuration fails
    here instead of turning the file into a second 128^3 test."""
    from tensoir_b200 import _lib, ops
    from tensoir_b200.synthetic import make_lego_model, n_samples_for
    from test_occupancy_bricks import _cells_bytes, _edge
    m = bench.m
    assert [int(g) for g in m.gridSize] == [GRID] * 3
    assert tuple(m.alphaMask.alpha_volume.shape[-3:]) == (MASK,) * 3
    assert bench.n_samples == N_SAMPLES and tuple(bench.rays.shape) == (N_RAYS, 6)
    f = ops.device_field(m).refresh(m)
    assert list(f.grid) == [GRID] * 3 and list(f.agrid) == [MASK] * 3
    # 2^3 cells per brick edge, 32^3 bricks: one bit each behind the 256^3 cell bytes
    assert _edge(MASK, MASK, MASK) == 1 << BRICK_SHIFT and (MASK >> BRICK_SHIFT) ** 3 == BRICK_BITS
    assert _cells_bytes(_lib.load(), MASK, MASK, MASK) == MASK ** 3 + BRICK_BITS // 8
    lens = _lengths(m, bench.rays, bench.li, bench.n_samples)
    with contextlib.redirect_stdout(io.StringIO()):
        m128 = make_lego_model(128, DEV)
    lens128 = _lengths(m128, bench.rays, bench.li, n_samples_for(128))
    del m128
    q = torch.tensor([0.5, 0.9, 0.99, 1.0], dtype=torch.float64, device=DEV)
    hit = lens[lens > 0].double()
    print(f"\nvalid samples per ray at {GRID}: {int((lens == 0).sum())} rays without any; of the others median / p90 / "
          f"p99 / max {[int(v) for v in torch.quantile(hit, q).tolist()]}, mean {float(hit.mean()):.1f}, total "
          f"{int(lens.sum())}; 32-sample chunks per ray up to {-(-int(lens.max()) // 32)}")
    print(f"at 128 on the same rays: max {int(lens128.max())}, total {int(lens128.sum())}")
    assert int(lens.max()) > int(lens128.max())


# ---------------------------------------------------------------------------------------------------- primary path
def test_primary_stages_random_map_gradients(bench):
    key = f"lego {GRID}"
    with own_stats():
        res = P.run_case(P.Case(bench.m, bench.rays, bench.li, bench.n_samples, 3), stats_key=key)
        P.assert_gates(res["gates"], res["total_app"], key)
        P.report(key)
    assert res["total_app"] > 0


@pytest.mark.parametrize("mode", ["relight", "phase1"])
def test_step_stages(monkeypatch, bench, mode):
    """the primary node's dumps of an eager training step on the bench's model and batch: the relight step is the one
    bench.py times"""
    m = bench.m
    m.__dict__["_tir_lean"] = True
    try:
        d = captured_step(monkeypatch, m, bench.rays, bench.li, 11, mode == "relight", bench.n_samples,
                          renderer_args(96))
    finally:
        m.__dict__.pop("_tir_lean")
    r = run(d, mode == "relight", f"lego {GRID} {mode}")
    assert int(r["lengths"].max()) > 4 * 32


def test_general_relight_step_stages(monkeypatch):
    """bench.py --config 4: the general model with three named lights, its relight step"""
    from tensoir_b200.synthetic import hemisphere_poses, n_samples_for, training_batch
    m = _lego(lights=("sunset", "snow", "courtyard"), general=True)
    rays, li = training_batch(hemisphere_poses(100), N_RAYS, 0, n_lights=3)
    assert set(li.view(-1).tolist()) == {0, 1, 2}
    m.__dict__["_tir_lean"] = True
    d = captured_step(monkeypatch, m, rays.to(DEV), li.to(DEV), 11, True, n_samples_for(GRID), renderer_args(96))
    run(d, True, f"lego {GRID} general, 3 lights, relight")


# -------------------------------------------------------------------------------------------------- secondary path
def _dirs_8x16(m):
    """the stratified directions of an 8 x 16 environment map (bench.py --config 3)"""
    h, w = m.envmap_h, m.envmap_w
    m.envmap_h, m.envmap_w = 8, 16
    try:
        return m.gen_light_incident_dirs(method='stratified_sampling').to(DEV).float().contiguous()
    finally:
        m.envmap_h, m.envmap_w = h, w


@pytest.mark.parametrize("n_dirs,pts_spec,lean", [(512, "1g+5", True), (128, "3g+7", True), (512, "1g+2", False)],
                         ids=["step", "config3_dirs", "count_parity"])
def test_secondary_march_and_list_mlp(bench, n_dirs, pts_spec, lean):
    sc, pts, nrm, li = S.scene("lego", bench.m)
    n = S._n_pts(pts_spec, True)
    assert pts.shape[0] >= n
    pts, nrm, li = pts[:n].contiguous(), nrm[:n].clone(), li[:n].contiguous()
    nrm[-2:] = 0.0
    dirs = S.stratified_dirs(sc, 512) if n_dirs == 512 else _dirs_8x16(sc.m)
    assert dirs.shape[0] == n_dirs
    out = S.launch_dense(sc, pts, nrm, li, dirs, 96, True, lean)
    torch.cuda.synchronize()
    what = f"lego {GRID} vol dirs {n_dirs} pts {n} N 96 {'lean' if lean else 'count'}"
    st = S.check_dense(sc, pts, nrm, li, dirs, 96, True, lean, out, what)
    S.report(what, st)


# ------------------------------------------------------------------------------------------------- density volume
@pytest.fixture(scope="module")
def surface(bench):
    """surface points, normals and light ids of the 300 model's forward on a 1 024-ray batch, 512 directions"""
    return DV._lego_inputs(n_rays=1024, m=bench.m)


def test_density_volume_builder(bench):
    m = bench.m
    lo, n, got = DV._built(m)
    assert n != DV._grid(m)
    print(f"\ndensity volume box lo {lo} n {n}: {n[0] * n[1] * n[2] * 4 / 1e6:.1f} MB")
    print(f"err / bound {DV._check_against_f64(DV._factors(m), lo, n, got):.3g}")


def test_density_volume_sub_box(surface):
    DV.sub_box_holds_every_vertex_a_valid_sample_reads(*surface, proper=True)


def test_volume_path_matches_factor_path(surface):
    DV.volume_path_matches_factor_path(*surface)


# ------------------------------------------------------------------------------------------------------ VM scatters
@pytest.fixture(scope="module")
def step_list(bench):
    """the valid-sample list of the bench batch on the 300 field, and that field's factors as a VM-kernel field"""
    return VS.lego_valid_list(bench.m, N_RAYS), V.Field(model=bench.m)


@pytest.mark.parametrize("order", ["ray_order", "shuffled"])
@pytest.mark.parametrize("kind", ["density", "app"])
def test_vm_scatter(step_list, kind, order):
    x, field = step_list
    assert field.grid == (GRID,) * 3
    if order == "shuffled":
        x = x[torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(5))]
    r = (VS.density_bwd if kind == "density" else VS.app_products_bwd)(field, x, f"lego {GRID} {order}")
    print(f"\n{x.shape[0]} rows, err / bound {r:.3g}")
