// Fused ray march: sample generation -> bbox / alpha-mask filter -> VM density gather -> softplus ->
// alpha -> transmittance scan -> compositing (+ compaction of the samples that need appearance).
//
// Mapping: one warp per ray, lanes = consecutive samples along the ray.  Valid samples (in bbox and
// alpha-mask > 0) are compacted into a per-warp shared-memory queue and the expensive gather runs on
// full 32-lane batches; invalid samples have sigma = 0 => alpha = 0 => T factor (1 - 0 + 1e-10) == 1.0f
// in fp32, so dropping them is exact (raw2alpha, tensorBase:21-28).
#include <type_traits>

#include "tir_device.cuh"

using namespace tir;

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kQueue = 64;
// Resident CTAs per SM.  The dense VOL instance with a z table (the secondary march of the training step) has no factor
// gather and fits in 80 registers, so it runs 3 CTAs (24 warps) per SM to hide the latency of its mask, volume and
// queue loads; the other instances need more registers and run 2.
template <int SAMPLING, bool DENSE, bool VOL>
constexpr bool kThreeCtas = DENSE && VOL && SAMPLING == TIR_SAMPLE_TABLE;
template <int SAMPLING, bool DENSE, bool VOL> constexpr int kBlocksPerSM = kThreeCtas<SAMPLING, DENSE, VOL> ? 3 : 2;

// Work counter of the dense secondary march: the next surface point a CTA takes.  The last CTA of a launch to finish
// puts it back to 0, so consecutive launches on a stream (and CUDA-graph replays) start from a zeroed counter without a
// host write.  There is one counter per device: two dense marches running at the same time on different streams would
// take points from each other's counter and each skip points of its own batch, so they must be ordered on the device.
__device__ unsigned long long g_dense_next_point = 0;
__device__ unsigned int g_dense_done_ctas = 0;

struct QEntry {
  float x, y, z;   // normalised coords
  float zs;        // z value of the sample
  float dist;      // z[s+1] - z[s] (0 for the last sample)
  int s;           // sample index along the ray
  int ray;         // ray the sample belongs to
};                 // 7 words: odd stride => conflict-free per-lane access

struct MarchParams {
  TirField f;
  TirMarchCfg cfg;
  // explicit rays
  const float* rays_o;
  const float* rays_d;
  // dense secondary generation
  const float* surf_xyz;
  const float* normals;
  const float* dirs;
  int n_dirs;
  int64_t n_pts;
  int64_t n_rays;   // dense: n_pts * n_dirs (ray = point * n_dirs + direction)
  float* t_last;
  float* acc;
  float* depth;
  TirAppSample* samples;
  uint32_t* sample_count;
  int64_t capacity;
  unsigned long long* counters;
  // density volume (VOL instances): the box [vlo, vlo+vn) of grid vertices, [z][y][x]; nullptr when the box is empty
  const float* vol;
  int vlo[3], vn[3];
};

// The density feature at a normalised point as the trilinear interpolation of the baked volume (TirDensityVolume).  The
// per-axis taps and weights are linear_setup's, i.e. the same unnormalize / floor_fi / zero-weight rule the factor path
// uses for the plane and line taps of that axis; only the association of the products differs.  Clamping into the box
// keeps every read in bounds; a valid sample's taps lie inside the box by construction (tir_density_volume_extent).
__device__ __forceinline__ float volume_feature(const MarchParams& p, float x, float y, float z) {
  if (!p.vol) return 0.f;
  const Linear1 tx = linear_setup(x, p.f.grid[0]), ty = linear_setup(y, p.f.grid[1]), tz = linear_setup(z, p.f.grid[2]);
  const int nx = p.vn[0], ny = p.vn[1], nz = p.vn[2];
  const int x0 = min(max(tx.o0 - p.vlo[0], 0), nx - 1), x1 = min(max(tx.o1 - p.vlo[0], 0), nx - 1);
  const int y0 = min(max(ty.o0 - p.vlo[1], 0), ny - 1), y1 = min(max(ty.o1 - p.vlo[1], 0), ny - 1);
  const int z0 = min(max(tz.o0 - p.vlo[2], 0), nz - 1), z1 = min(max(tz.o1 - p.vlo[2], 0), nz - 1);
  const float* r00 = p.vol + ((size_t)z0 * ny + y0) * nx;
  const float* r01 = p.vol + ((size_t)z0 * ny + y1) * nx;
  const float* r10 = p.vol + ((size_t)z1 * ny + y0) * nx;
  const float* r11 = p.vol + ((size_t)z1 * ny + y1) * nx;
  const float a00 = fmaf(__ldg(r00 + x1), tx.w1, __fmul_rn(__ldg(r00 + x0), tx.w0));
  const float a01 = fmaf(__ldg(r01 + x1), tx.w1, __fmul_rn(__ldg(r01 + x0), tx.w0));
  const float a10 = fmaf(__ldg(r10 + x1), tx.w1, __fmul_rn(__ldg(r10 + x0), tx.w0));
  const float a11 = fmaf(__ldg(r11 + x1), tx.w1, __fmul_rn(__ldg(r11 + x0), tx.w0));
  const float b0 = fmaf(a01, ty.w1, __fmul_rn(a00, ty.w0));
  const float b1 = fmaf(a11, ty.w1, __fmul_rn(a10, ty.w0));
  return fmaf(b1, tz.w1, __fmul_rn(b0, tz.w0));
}

// Segmented warp scans over lanes whose segment heads are flagged (consecutive samples of one ray form a segment).
__device__ __forceinline__ float seg_scan_mul(float v, bool head, int lane) {
  bool f = head;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float vu = __shfl_up_sync(0xffffffffu, v, o);
    const bool fu = __shfl_up_sync(0xffffffffu, (int)f, o) != 0;
    if (lane >= o) {
      if (!f) v = __fmul_rn(vu, v);
      f = f | fu;
    }
  }
  return v;
}
__device__ __forceinline__ float seg_scan_add(float v, bool head, int lane) {
  bool f = head;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float vu = __shfl_up_sync(0xffffffffu, v, o);
    const bool fu = __shfl_up_sync(0xffffffffu, (int)f, o) != 0;
    if (lane >= o) {
      if (!f) v += vu;
      f = f | fu;
    }
  }
  return v;
}

template <int C, int SAMPLING, bool WITH_APP, bool DENSE, bool VOL>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kBlocksPerSM<SAMPLING, DENSE, VOL>)
    march_kernel(const MarchParams p) {
  __shared__ QEntry queue[kWarpsPerBlock][kQueue];
  __shared__ uint32_t brick_bits[kBrickMaxWords];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  QEntry* q = queue[warp];
  const TirField& f = p.f;
  // the occupancy bricks of the alpha mask, copied once per (persistent) CTA
  CellBricks bricks{nullptr, 0, 0, 0};
  if (const uint32_t* src = f.amask ? global_bricks(f, p.cfg) : nullptr) {
    bricks = cell_bricks(f, brick_bits);
    const int words = (int)brick_geom(f.agrid[0], f.agrid[1], f.agrid[2]).words;
    for (int i = threadIdx.x; i < words; i += blockDim.x) brick_bits[i] = __ldg(src + i);
    __syncthreads();
  }
  const int N = p.cfg.n_samples;
  const float scale = f.distance_scale;
  const bool need_sums = (p.acc != nullptr) | (p.depth != nullptr);
  // per-lane counts; 32 bits in the 3-CTA instance, which needs the registers (launch_instance bounds the counts)
  using Count = typename std::conditional<kThreeCtas<SAMPLING, DENSE, VOL>, unsigned, unsigned long long>::type;
  Count c_mask = 0, c_density = 0, c_app = 0, c_rays = 0, c_over = 0;

  // Valid samples of CONSECUTIVE rays share 32-lane gather batches (a ray rarely has a multiple of 32 valid samples;
  // flushing per ray left the 72-load gather ~40 % occupied).  The compositing scan is segmented by ray; the state of
  // the one ray that may straddle two batches is carried in (c_ray, c_T, c_acc, c_dep).
  int qn = 0;
  int c_ray = -1;
  float c_T = 1.f, c_acc = 0.f, c_dep = 0.f;

  // gather + composite the first `nb` queue entries (nb <= 32).  Segments of rays other than `open_ray` are complete.
  auto process = [&](int nb, int open_ray) {
    const bool active = lane < nb;
    const QEntry e = q[active ? lane : 0];
    const int ray_l = active ? e.ray : -2 - lane;
    float sigma = 0.f;
    if (active) {
      const float feat = VOL ? volume_feature(p, e.x, e.y, e.z) : density_feature<C>(f, e.x, e.y, e.z);
      sigma = feature_to_sigma(f, feat);
    }
    // raw2alpha: alpha = 1 - exp(-sigma * (dist*scale)); T = cumprod(1 - alpha + 1e-10)
    const float alpha = active ? __fsub_rn(1.f, expf(__fmul_rn(-sigma, __fmul_rn(e.dist, scale)))) : 0.f;
    const int prev_ray = __shfl_up_sync(0xffffffffu, ray_l, 1);
    const int next_ray = __shfl_down_sync(0xffffffffu, ray_l, 1);
    const bool head = (lane == 0) | (prev_ray != ray_l);
    const bool tail = active & ((lane == 31) | (next_ray != ray_l));
    const bool cont = (ray_l == c_ray);                       // continues the carried ray
    const float incl = seg_scan_mul(__fadd_rn(__fsub_rn(1.f, alpha), 1e-10f), head, lane);
    const float incl_prev = __shfl_up_sync(0xffffffffu, incl, 1);
    const float start = cont ? c_T : 1.f;
    const float excl = __fmul_rn(start, head ? 1.f : incl_prev);
    const float w = __fmul_rn(alpha, excl);
    const float seg_T = __fmul_rn(start, incl);
    float seg_acc = 0.f, seg_dep = 0.f;
    if (need_sums) {
      seg_acc = seg_scan_add(w, head, lane) + (cont ? c_acc : 0.f);
      seg_dep = seg_scan_add(w * e.zs, head, lane) + (cont ? c_dep : 0.f);
    }
    if (tail & (ray_l != open_ray)) {                         // ray complete: emit its outputs
      if (p.t_last) p.t_last[ray_l] = seg_T;
      if (p.acc) p.acc[ray_l] = seg_acc;
      if (p.depth) p.depth[ray_l] = seg_dep;
    }
    // carry the straddling ray (if the last entry belongs to the ray still being sampled)
    const int last_ray = __shfl_sync(0xffffffffu, ray_l, nb - 1);
    const float last_T = __shfl_sync(0xffffffffu, seg_T, nb - 1);
    const float last_acc = __shfl_sync(0xffffffffu, seg_acc, nb - 1);
    const float last_dep = __shfl_sync(0xffffffffu, seg_dep, nb - 1);
    if (last_ray == open_ray) { c_ray = last_ray; c_T = last_T; c_acc = last_acc; c_dep = last_dep; }
    else { c_ray = -1; c_T = 1.f; c_acc = 0.f; c_dep = 0.f; }
    if (WITH_APP) {
      const bool app = active && (w > f.weight_thres);
      const unsigned m = __ballot_sync(0xffffffffu, app);
      if (m) {
        unsigned base = 0;
        const int cnt = __popc(m);
        if (lane == 0) base = atomicAdd(p.sample_count, (unsigned)cnt);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (app) {
          const unsigned slot = base + __popc(m & ((1u << lane) - 1u));
          if ((int64_t)slot < p.capacity) {
            // re-read from the queue rather than kept in registers across the gather and the scans
            const volatile QEntry& r = q[lane];
            TirAppSample sm;
            sm.xn[0] = r.x; sm.xn[1] = r.y; sm.xn[2] = r.z; sm.weight = w; sm.ray = r.ray; sm.sample = r.s;
            p.samples[slot] = sm;
            c_app += 1;
          } else {
            c_over += 1;
          }
        }
      }
    } else {
      c_app += (active && (w > f.weight_thres));
    }
    c_density += active;
  };

  // march one ray (all of its samples) through this warp's queue
  auto march_ray = [&](int64_t ray64, float ox, float oy, float oz, float dx, float dy, float dz) {
    const int ray = (int)ray64;
    c_rays += (lane == 0);

    float tmin = 0.f, jit = 0.f;
    if (SAMPLING == TIR_SAMPLE_STEP) {
      // sample_ray (tensorBase:705-724)
      const float vx = dx == 0.f ? 1e-6f : dx, vy = dy == 0.f ? 1e-6f : dy, vz = dz == 0.f ? 1e-6f : dz;
      const float ax = __fdiv_rn(__fsub_rn(f.aabb_hi[0], ox), vx), bx = __fdiv_rn(__fsub_rn(f.aabb_lo[0], ox), vx);
      const float ay = __fdiv_rn(__fsub_rn(f.aabb_hi[1], oy), vy), by = __fdiv_rn(__fsub_rn(f.aabb_lo[1], oy), vy);
      const float az = __fdiv_rn(__fsub_rn(f.aabb_hi[2], oz), vz), bz = __fdiv_rn(__fsub_rn(f.aabb_lo[2], oz), vz);
      tmin = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz));
      tmin = fminf(fmaxf(tmin, p.cfg.near), p.cfg.far);
      jit = p.cfg.jitter ? __ldg(p.cfg.jitter + ray64) : 0.f;
    }
    auto z_of = [&](int s) -> float {
      if (SAMPLING == TIR_SAMPLE_STEP) return __fadd_rn(tmin, __fmul_rn(p.cfg.step, __fadd_rn((float)s, jit)));
      return __ldg(p.cfg.z_table + s);
    };

    int pushed = 0;
    const bool lean = (p.cfg.flags & TIR_MARCH_LEAN_COUNTERS) != 0;
    // parametric interval of the ray inside the occupied-cell box (slab test); samples outside cannot be valid
    const bool use_occ = f.amask != nullptr && f.occ_lo[0] <= f.occ_hi[0];
    float z_in = -3.0e38f, z_out = 3.0e38f;
    if (use_occ) {
      const float d3[3] = {dx, dy, dz}, o3[3] = {ox, oy, oz};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (fabsf(d3[a]) > 1e-12f) {
          const float t0 = (f.occ_lo[a] - o3[a]) / d3[a], t1 = (f.occ_hi[a] - o3[a]) / d3[a];
          z_in = fmaxf(z_in, fminf(t0, t1)); z_out = fminf(z_out, fmaxf(t0, t1));
        } else if (o3[a] < f.occ_lo[a] || o3[a] > f.occ_hi[a]) {
          z_in = 3.0e38f;                       // parallel to the slab and outside it: never inside the box
        }
      }
      // safety margin against the rounding of the slab arithmetic (the per-sample box test below stays exact)
      const float pad = 1e-3f * (fabsf(z_in) + fabsf(z_out) + 1.f);
      z_in -= pad; z_out += pad;
    }
    for (int base = 0; base < N; base += 32) {
      // lean mode: a whole 32-sample chunk that lies outside the occupied box holds no valid sample, and nobody asked
      // for the mask counts of its in-aabb samples
      if (lean && use_occ) {
        const float za = z_of(base), zb = z_of(min(base + 31, N - 1));
        if (zb < z_in || za > z_out) continue;
      }
      // lean mode: a ray whose carried transmittance is exactly 0 cannot change any output any more (see below), and
      // nobody asked for the mask / density counts of its remaining samples, so the rest of the ray is skipped
      if (lean && c_ray == ray && c_T == 0.f) break;
      const int s = base + lane;
      bool valid = false;
      float nx = 0.f, ny = 0.f, nz = 0.f, z = 0.f;
      if (s < N) {
        z = z_of(s);
        const float px = __fadd_rn(ox, __fmul_rn(dx, z)), py = __fadd_rn(oy, __fmul_rn(dy, z)),
                    pz = __fadd_rn(oz, __fmul_rn(dz, z));
        const bool out = (f.aabb_lo[0] > px) | (px > f.aabb_hi[0]) | (f.aabb_lo[1] > py) | (py > f.aabb_hi[1]) |
                         (f.aabb_lo[2] > pz) | (pz > f.aabb_hi[2]);
        if (!out) {
          valid = true;
          if (f.amask) {
            c_mask += 1;                       // the reference looks every in-aabb sample up (count parity)
            // outside the bounding box of the occupied mask cells the trilinear lookup is exactly 0: no byte load
            const bool in_occ = !use_occ || ((px >= f.occ_lo[0]) & (px <= f.occ_hi[0]) & (py >= f.occ_lo[1]) &
                                             (py <= f.occ_hi[1]) & (pz >= f.occ_lo[2]) & (pz <= f.occ_hi[2]));
            valid = in_occ && alpha_mask_positive(f, px, py, pz, bricks);
          }
          // normalize_coord (tensorBase:640-641)
          nx = __fsub_rn(__fmul_rn(__fsub_rn(px, f.aabb_lo[0]), f.inv_aabb[0]), 1.f);
          ny = __fsub_rn(__fmul_rn(__fsub_rn(py, f.aabb_lo[1]), f.inv_aabb[1]), 1.f);
          nz = __fsub_rn(__fmul_rn(__fsub_rn(pz, f.aabb_lo[2]), f.inv_aabb[2]), 1.f);
        }
      }
      // Exact early termination: once the transmittance carried for THIS ray has underflowed to exactly 0.0f, every
      // later weight is alpha * 0 = 0 and T stays 0 (0 * finite), so the remaining samples cannot change t_last, acc,
      // depth or the appearance list.  Their gather is skipped; they are still counted, so the counters keep meaning
      // "samples the reference evaluates".  (c_ray, c_T are warp-uniform; samples of the ray that are still queued
      // simply keep the state unknown, which is conservative.)
      if (c_ray == ray && c_T == 0.f) {
        c_density += valid;
        valid = false;
      }
      const unsigned m = __ballot_sync(0xffffffffu, valid);
      if (valid) {
        QEntry e;
        e.x = nx; e.y = ny; e.z = nz; e.zs = z; e.s = s; e.ray = ray;
        e.dist = (s + 1 < N) ? __fsub_rn(z_of(s + 1), z) : 0.f;
        q[qn + __popc(m & ((1u << lane) - 1u))] = e;
      }
      qn += __popc(m);
      pushed += __popc(m);
      __syncwarp();
      if (qn >= 32) {
        process(32, ray);
        __syncwarp();
        const int rest = qn - 32;
        QEntry mv;
        if (lane < rest) mv = q[32 + lane];
        __syncwarp();
        if (lane < rest) q[lane] = mv;
        qn = rest;
        __syncwarp();
      }
    }
    // the ray is complete; if none of its samples is still queued its outputs are final now
    const bool queued = (qn > 0) && (q[qn - 1].ray == ray);
    if (!queued) {
      if (c_ray == ray) {
        if (lane == 0) {
          if (p.t_last) p.t_last[ray] = c_T;
          if (p.acc) p.acc[ray] = c_acc;
          if (p.depth) p.depth[ray] = c_dep;
        }
        c_ray = -1; c_T = 1.f; c_acc = 0.f; c_dep = 0.f;
      } else if (pushed == 0 && lane == 0) {
        if (p.t_last) p.t_last[ray] = 1.f;
        if (p.acc) p.acc[ray] = 0.f;
        if (p.depth) p.depth[ray] = 0.f;
      }
    }
  };

  if (!DENSE) {
    const int64_t warp_stride = (int64_t)gridDim.x * kWarpsPerBlock;
    for (int64_t ray = (int64_t)blockIdx.x * kWarpsPerBlock + warp; ray < p.n_rays; ray += warp_stride) {
      march_ray(ray, __ldg(p.rays_o + ray * 3 + 0), __ldg(p.rays_o + ray * 3 + 1), __ldg(p.rays_o + ray * 3 + 2),
                __ldg(p.rays_d + ray * 3 + 0), __ldg(p.rays_d + ray * 3 + 1), __ldg(p.rays_d + ray * 3 + 2));
    }
  } else {
    // Point-major: the CTA takes one surface point at a time from the work counter and its warps take that point's
    // directions one by one, so the density texels around the point are fetched into this SM's L1 and reused by all of
    // its rays.  Double-buffered slots: a slot is rewritten two points later, after a barrier every warp has passed
    // since it last read it.
    __shared__ long long s_pt[2];
    __shared__ int s_dir[2];
    for (int it = 0;; ++it) {
      const int b = it & 1;
      if (threadIdx.x == 0) {
        s_pt[b] = (long long)atomicAdd(&g_dense_next_point, 1ull);
        s_dir[b] = 0;
      }
      __syncthreads();
      const int64_t pt = s_pt[b];
      if (pt >= p.n_pts) break;
      const float nx = __ldg(p.normals + pt * 3 + 0), ny = __ldg(p.normals + pt * 3 + 1),
                  nz = __ldg(p.normals + pt * 3 + 2);
      // a zero normal (non-hit ray, tir_hits_prepare) fails the cosine test for every direction
      if ((nx == 0.f) & (ny == 0.f) & (nz == 0.f)) continue;
      const float ox = __ldg(p.surf_xyz + pt * 3 + 0), oy = __ldg(p.surf_xyz + pt * 3 + 1),
                  oz = __ldg(p.surf_xyz + pt * 3 + 2);
      for (;;) {
        int di = 0;
        if (lane == 0) di = atomicAdd(&s_dir[b], 1);
        di = __shfl_sync(0xffffffffu, di, 0);
        if (di >= p.n_dirs) break;
        const float dx = __ldg(p.dirs + di * 3 + 0), dy = __ldg(p.dirs + di * 3 + 1), dz = __ldg(p.dirs + di * 3 + 2);
        // cosine = clamp(einsum(surf2l, normal), 0) > 1e-6 (relight_utils.py:433-435)
        const float cosine = fmaxf(fmaf(dz, nz, fmaf(dy, ny, __fmul_rn(dx, nx))), 0.f);
        if (!(cosine > 1e-6f)) continue;
        march_ray(pt * p.n_dirs + di, ox, oy, oz, dx, dy, dz);
      }
    }
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(&g_dense_done_ctas, 1u) == gridDim.x - 1) {   // every CTA has taken its last point
        atomicExch(&g_dense_next_point, 0ull);
        atomicExch(&g_dense_done_ctas, 0u);
      }
    }
  }
  if (qn > 0) process(qn, -1);

  const unsigned long long t_mask = warp_sum_u64(c_mask), t_density = warp_sum_u64(c_density),
                           t_app = warp_sum_u64(c_app), t_rays = warp_sum_u64(c_rays), t_over = warp_sum_u64(c_over);
  if (lane == 0 && p.counters) {
    if (t_mask) atomicAdd(p.counters + TIR_CNT_MASK, t_mask);
    if (t_density) atomicAdd(p.counters + TIR_CNT_DENSITY, t_density);
    if (t_app) atomicAdd(p.counters + TIR_CNT_APP, t_app);
    if (t_rays) atomicAdd(p.counters + TIR_CNT_RAYS, t_rays);
    if (t_over) atomicAdd(p.counters + TIR_CNT_OVERFLOW, t_over);
  }
}

template <int SAMPLING, bool WITH_APP, bool DENSE, bool VOL>
int launch_instance(const MarchParams& p, cudaStream_t stream) {
  // a lane's count grows by at most 2 per 32-sample chunk its warp walks: the 32-bit counts of the 3-CTA instance stay
  // exact even if one warp walked every ray
  if (kThreeCtas<SAMPLING, DENSE, VOL> && (uint64_t)p.n_rays * ((p.cfg.n_samples + 31) / 32) * 2 > 0xffffffffull)
    return TIR_ERR_SHAPE;
  // persistent: every resident CTA slot; grid-stride over rays, or (dense) one surface point per CTA at a time
  int64_t blocks = DENSE ? p.n_pts : (p.n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock;
  const int64_t max_blocks = (int64_t)num_sms() * kBlocksPerSM<SAMPLING, DENSE, VOL>;
  if (blocks > max_blocks) blocks = max_blocks;
  march_kernel<16, SAMPLING, WITH_APP, DENSE, VOL><<<(int)blocks, kWarpsPerBlock * 32, 0, stream>>>(p);
  return (int)cudaGetLastError();
}

template <bool WITH_APP, bool DENSE, bool VOL = false>
int launch_march(const MarchParams& p, cudaStream_t stream) {
  if (p.n_rays <= 0) return TIR_OK;
  if (p.f.dC != 16) return TIR_ERR_SHAPE;
  if (p.cfg.n_samples <= 0) return TIR_ERR_CONFIG;
  if (p.cfg.sampling == TIR_SAMPLE_STEP) return launch_instance<TIR_SAMPLE_STEP, WITH_APP, DENSE, VOL>(p, stream);
  if (p.cfg.sampling == TIR_SAMPLE_TABLE) {
    if (!p.cfg.z_table) return TIR_ERR_NULL;
    return launch_instance<TIR_SAMPLE_TABLE, WITH_APP, DENSE, VOL>(p, stream);
  }
  return TIR_ERR_CONFIG;
}

// Density volume builder: D[x,y,z] = sum_k sum_c plane_k[c] * line_k[c] at the grid vertices of the box.  A CTA is a
// 32 (x) x 8 (y) tile of vertices and walks kVolZ consecutive z.  The three factor rows that do not depend on z
// (plane 0 at (x,y), line 1 at y, line 2 at x) stay in registers for the whole walk.  The rows that do (line 0 at z,
// plane 1 at (x,z), plane 2 at (y,z)) are read from global memory once per CTA, all loads in flight together, into
// shared memory, where every warp of the tile finds them: each plane-1 row serves the tile's 8 y.
constexpr int kVolTileX = 32, kVolTileY = 8, kVolZ = 8;
// plane-1 row stride in shared memory: 20 floats, so the 8 lanes of a quarter warp reading 16 B of 8 consecutive rows
// hit 8 distinct 4-bank groups (a 16-float stride would put them on 2)
constexpr int kVolRow = 20;

__device__ __forceinline__ float dot16(const float (&a)[16], const float* b) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 16; c += 4) {           // channel order, like density_feature
    const float4 v = *reinterpret_cast<const float4*>(b + c);
    s = __fadd_rn(s, __fmul_rn(a[c + 0], v.x));
    s = __fadd_rn(s, __fmul_rn(a[c + 1], v.y));
    s = __fadd_rn(s, __fmul_rn(a[c + 2], v.z));
    s = __fadd_rn(s, __fmul_rn(a[c + 3], v.w));
  }
  return s;
}

__device__ __forceinline__ void load16(float (&a)[16], const float* src) {
#pragma unroll
  for (int c = 0; c < 16; c += 4) {
    const float4 v = ldg4(src + c);
    a[c] = v.x; a[c + 1] = v.y; a[c + 2] = v.z; a[c + 3] = v.w;
  }
}

__global__ void __launch_bounds__(kVolTileX * kVolTileY) density_volume_kernel(const TirField f, TirDensityVolume v) {
  __shared__ __align__(16) float s_p1[kVolZ][kVolTileX][kVolRow];
  __shared__ __align__(16) float s_p2[kVolZ][kVolTileY][16];
  __shared__ __align__(16) float s_l0[kVolZ][16];
  const int X = f.grid[0], Y = f.grid[1];
  const int xi0 = blockIdx.x * kVolTileX, yi0 = blockIdx.y * kVolTileY, zi0 = blockIdx.z * kVolZ;
  const int tx = min(kVolTileX, v.n[0] - xi0), ty = min(kVolTileY, v.n[1] - yi0), tz = min(kVolZ, v.n[2] - zi0);
  const int x0 = v.lo[0] + xi0, y0 = v.lo[1] + yi0, z0 = v.lo[2] + zi0;
  const int tid = threadIdx.y * kVolTileX + threadIdx.x;
  // stage the z-dependent rows of the tile, 16 B per load, consecutive threads on consecutive 16 B of a row
  // matMode {0,1},{0,2},{1,2}, vecMode {2,1,0}: plane k is [G[m1]][G[m0]][C], line k is [G[v]][C]
  for (int i = tid; i < kVolZ * kVolTileX * 4; i += kVolTileX * kVolTileY) {
    const int c = (i & 3) * 4, xl = (i >> 2) % kVolTileX, zl = (i >> 2) / kVolTileX;
    if (xl < tx && zl < tz)
      *reinterpret_cast<float4*>(&s_p1[zl][xl][c]) = ldg4(f.dplane[1] + ((size_t)(z0 + zl) * X + x0 + xl) * 16 + c);
  }
  for (int i = tid; i < kVolZ * kVolTileY * 4; i += kVolTileX * kVolTileY) {
    const int c = (i & 3) * 4, yl = (i >> 2) % kVolTileY, zl = (i >> 2) / kVolTileY;
    if (yl < ty && zl < tz)
      *reinterpret_cast<float4*>(&s_p2[zl][yl][c]) = ldg4(f.dplane[2] + ((size_t)(z0 + zl) * Y + y0 + yl) * 16 + c);
  }
  if (tid < kVolZ * 4) {
    const int c = (tid & 3) * 4, zl = tid >> 2;
    if (zl < tz) *reinterpret_cast<float4*>(&s_l0[zl][c]) = ldg4(f.dline[0] + (size_t)(z0 + zl) * 16 + c);
  }
  const bool in_box = (int)threadIdx.x < tx && (int)threadIdx.y < ty;
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  float p0[16], l1[16], l2[16];
  if (in_box) {
    load16(p0, f.dplane[0] + ((size_t)y * X + x) * 16);
    load16(l1, f.dline[1] + (size_t)y * 16);
    load16(l2, f.dline[2] + (size_t)x * 16);
  }
  __syncthreads();
  if (!in_box) return;
  float* out = v.data + ((size_t)zi0 * v.n[1] + yi0 + threadIdx.y) * v.n[0] + xi0 + threadIdx.x;
  const size_t z_stride = (size_t)v.n[1] * v.n[0];
#pragma unroll
  for (int zl = 0; zl < kVolZ; ++zl) {
    if (zl < tz) {
      const float s0 = dot16(p0, s_l0[zl]);
      const float s1 = dot16(l1, s_p1[zl][threadIdx.x]);
      const float s2 = dot16(l2, s_p2[zl][threadIdx.y]);
      out[zl * z_stride] = __fadd_rn(__fadd_rn(s0, s1), s2);
    }
  }
}

// grid vertex index of world coordinate c along `axis`, with the march's normalize_coord / unnormalize arithmetic
int host_floor_index(const TirField& f, int axis, float c) {
  const float n = (c - f.aabb_lo[axis]) * f.inv_aabb[axis] - 1.f;
  const float i = ((n + 1.f) * 0.5f) * (float)(f.grid[axis] - 1);
  const float lim = (float)f.grid[axis] + 2.f;                 // keeps the int conversion in range
  return (int)floorf(fminf(fmaxf(i, -lim), lim));
}

// validate a box handed in by the caller against the field's grid
int check_box(const TirField& f, const TirDensityVolume& v, bool* empty) {
  *empty = false;
  for (int a = 0; a < 3; ++a) {
    if (v.n[a] < 0 || v.lo[a] < 0 || (int64_t)v.lo[a] + v.n[a] > f.grid[a]) return TIR_ERR_SHAPE;
    if (v.n[a] == 0) *empty = true;
  }
  if (!*empty && !v.data) return TIR_ERR_NULL;
  return TIR_OK;
}

}  // namespace

extern "C" int tir_density_volume_extent(const TirField* field, int32_t lo[3], int32_t n[3]) {
  if (!field || !lo || !n) return TIR_ERR_NULL;
  const TirField& f = *field;
  for (int a = 0; a < 3; ++a)
    if (f.grid[a] < 1) return TIR_ERR_SHAPE;
  const bool box = f.amask != nullptr && f.occ_lo[0] <= f.occ_hi[0];
  bool empty = false;
  for (int a = 0; a < 3; ++a) {
    if (!box) { lo[a] = 0; n[a] = f.grid[a]; continue; }
    // taps floor(i) and floor(i)+1 of every coordinate in [occ_lo, occ_hi] (the arithmetic is monotone), plus a
    // one-vertex guard on each side for any host / device rounding difference
    const int i0 = host_floor_index(f, a, f.occ_lo[a]) - 1;
    const int i1 = host_floor_index(f, a, f.occ_hi[a]) + 2;
    const int a0 = i0 < 0 ? 0 : i0, a1 = i1 > f.grid[a] - 1 ? f.grid[a] - 1 : i1;
    lo[a] = a0;
    n[a] = a1 >= a0 ? a1 - a0 + 1 : 0;
    if (n[a] == 0) empty = true;
  }
  if (empty)
    for (int a = 0; a < 3; ++a) { lo[a] = 0; n[a] = 0; }
  return TIR_OK;
}

extern "C" int tir_density_volume_build(const TirField* field, TirDensityVolume* vol, int64_t capacity, void* stream) {
  if (!field || !vol) return TIR_ERR_NULL;
  const TirField& f = *field;
  if (f.dC != 16) return TIR_ERR_SHAPE;
  bool empty = false;
  if (int rc = check_box(f, *vol, &empty)) return rc;
  if (empty) return TIR_OK;
  if ((int64_t)vol->n[0] * vol->n[1] * vol->n[2] > capacity) return TIR_ERR_CAPACITY;
  for (int k = 0; k < 3; ++k)
    if (!f.dplane[k] || !f.dline[k]) return TIR_ERR_NULL;
  const dim3 block(kVolTileX, kVolTileY);
  const dim3 grid((vol->n[0] + kVolTileX - 1) / kVolTileX, (vol->n[1] + kVolTileY - 1) / kVolTileY,
                  (vol->n[2] + kVolZ - 1) / kVolZ);
  density_volume_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(f, *vol);
  return (int)cudaGetLastError();
}

extern "C" int tir_march_density(const TirField* field, const float* rays_o, const float* rays_d, int64_t n_rays,
                                 const TirMarchCfg* cfg, float* t_last, float* acc, float* depth,
                                 uint64_t* counters, void* stream) {
  if (n_rays <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !cfg || !rays_o || !rays_d) return TIR_ERR_NULL;
  MarchParams p{};
  p.f = *field; p.cfg = *cfg; p.rays_o = rays_o; p.rays_d = rays_d; p.n_rays = n_rays;
  p.t_last = t_last; p.acc = acc; p.depth = depth; p.counters = (unsigned long long*)counters;
  return launch_march<false, false>(p, (cudaStream_t)stream);
}

extern "C" int tir_march_radiance(const TirField* field, const TirMlp* mlp, const float* rays_o, const float* rays_d,
                                  const int32_t* light_idx, int64_t n_rays, const TirMarchCfg* cfg,
                                  float* t_last, float* acc, float* depth, float* rgb,
                                  TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                                  uint64_t* counters, void* stream) {
  if (n_rays <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !mlp || !cfg || !rays_o || !rays_d || !rgb || !samples || !sample_count) return TIR_ERR_NULL;
  if (capacity <= 0) return TIR_ERR_CAPACITY;
  MarchParams p{};
  p.f = *field; p.cfg = *cfg; p.rays_o = rays_o; p.rays_d = rays_d; p.n_rays = n_rays;
  p.t_last = t_last; p.acc = acc; p.depth = depth; p.counters = (unsigned long long*)counters;
  p.samples = samples; p.sample_count = sample_count; p.capacity = capacity;
  int rc = launch_march<true, false>(p, (cudaStream_t)stream);
  if (rc) return rc;
  return tir_app_mlp(field, mlp, samples, sample_count, capacity, rays_d, 0, light_idx, rgb, stream);
}

namespace {
// tir_secondary_march(_vol): vol == nullptr selects the factor path
int secondary_march(const TirField* field, const float* surf_xyz, const float* normals, int64_t n_pts,
                    const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg, const TirDensityVolume* vol, float* vis,
                    TirAppSample* samples, uint32_t* sample_count, int64_t capacity, uint64_t* counters,
                    void* stream) {
  if (n_pts <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !cfg || !surf_xyz || !normals || !dirs || !vis || !samples || !sample_count) return TIR_ERR_NULL;
  if (n_dirs <= 0) return TIR_ERR_SHAPE;
  if (capacity <= 0) return TIR_ERR_CAPACITY;
  MarchParams p{};
  p.f = *field; p.cfg = *cfg; p.surf_xyz = surf_xyz; p.normals = normals; p.dirs = dirs; p.n_dirs = n_dirs;
  p.n_pts = n_pts;
  p.n_rays = n_pts * (int64_t)n_dirs;
  p.t_last = vis; p.counters = (unsigned long long*)counters;
  p.samples = samples; p.sample_count = sample_count; p.capacity = capacity;
  if (!vol) return launch_march<true, true, false>(p, (cudaStream_t)stream);
  bool empty = false;
  if (int rc = check_box(*field, *vol, &empty)) return rc;
  p.vol = empty ? nullptr : vol->data;
  for (int a = 0; a < 3; ++a) { p.vlo[a] = vol->lo[a]; p.vn[a] = vol->n[a]; }
  return launch_march<true, true, true>(p, (cudaStream_t)stream);
}
}  // namespace

extern "C" int tir_secondary_march(const TirField* field, const float* surf_xyz, const float* normals,
                                  int64_t n_pts, const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg,
                                  float* vis, TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                                  uint64_t* counters, void* stream) {
  return secondary_march(field, surf_xyz, normals, n_pts, dirs, n_dirs, cfg, nullptr, vis, samples, sample_count,
                         capacity, counters, stream);
}

extern "C" int tir_secondary_march_vol(const TirField* field, const float* surf_xyz, const float* normals,
                                      int64_t n_pts, const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg,
                                      const TirDensityVolume* vol, float* vis, TirAppSample* samples,
                                      uint32_t* sample_count, int64_t capacity, uint64_t* counters, void* stream) {
  if (n_pts > 0 && !vol) return TIR_ERR_NULL;
  return secondary_march(field, surf_xyz, normals, n_pts, dirs, n_dirs, cfg, vol, vis, samples, sample_count,
                         capacity, counters, stream);
}

extern "C" int tir_secondary_radiance(const TirField* field, const TirMlp* mlp, const float* surf_xyz,
                                      const float* normals, const int32_t* light_idx, int64_t n_pts,
                                      const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg, float* vis,
                                      float* indirect, TirAppSample* samples, uint32_t* sample_count,
                                      int64_t capacity, uint64_t* counters, void* stream) {
  if (n_pts <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!mlp || !indirect) return TIR_ERR_NULL;
  int rc = tir_secondary_march(field, surf_xyz, normals, n_pts, dirs, n_dirs, cfg, vis, samples, sample_count,
                               capacity, counters, stream);
  if (rc) return rc;
  return tir_app_mlp(field, mlp, samples, sample_count, capacity, dirs, n_dirs, light_idx, indirect, stream);
}

extern "C" int tir_secondary_radiance_vol(const TirField* field, const TirMlp* mlp, const float* surf_xyz,
                                          const float* normals, const int32_t* light_idx, int64_t n_pts,
                                          const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg,
                                          const TirDensityVolume* vol, float* vis, float* indirect,
                                          TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                                          uint64_t* counters, void* stream) {
  if (n_pts <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!mlp || !indirect) return TIR_ERR_NULL;
  int rc = tir_secondary_march_vol(field, surf_xyz, normals, n_pts, dirs, n_dirs, cfg, vol, vis, samples,
                                   sample_count, capacity, counters, stream);
  if (rc) return rc;
  return tir_app_mlp(field, mlp, samples, sample_count, capacity, dirs, n_dirs, light_idx, indirect, stream);
}
