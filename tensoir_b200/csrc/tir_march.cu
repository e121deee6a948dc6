// Fused ray march: sample generation -> bbox / alpha-mask filter -> VM density gather -> softplus ->
// alpha -> transmittance scan -> compositing (+ compaction of the samples that need appearance).
//
// Mapping: one warp per ray, lanes = consecutive samples along the ray.  Valid samples (in bbox and
// alpha-mask > 0) are compacted into a per-warp shared-memory queue and the expensive gather runs on
// full 32-lane batches; invalid samples have sigma = 0 => alpha = 0 => T factor (1 - 0 + 1e-10) == 1.0f
// in fp32, so dropping them is exact (raw2alpha, tensorBase:21-28).
#include "tir_device.cuh"

using namespace tir;

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kQueue = 64;
constexpr int kBlocksPerSM = 2;

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
  int64_t n_rays;
  float* t_last;
  float* acc;
  float* depth;
  TirAppSample* samples;
  uint32_t* sample_count;
  int64_t capacity;
  unsigned long long* counters;
};

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

template <int C, int SAMPLING, bool WITH_APP, bool DENSE>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kBlocksPerSM) march_kernel(const MarchParams p) {
  __shared__ QEntry queue[kWarpsPerBlock][kQueue];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  QEntry* q = queue[warp];
  const TirField& f = p.f;
  const int N = p.cfg.n_samples;
  const float scale = f.distance_scale;
  const bool need_sums = (p.acc != nullptr) | (p.depth != nullptr);
  unsigned long long c_mask = 0, c_density = 0, c_app = 0, c_rays = 0, c_over = 0;

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
    if (active) sigma = feature_to_sigma(f, density_feature<C>(f, e.x, e.y, e.z));
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
            TirAppSample sm;
            sm.xn[0] = e.x; sm.xn[1] = e.y; sm.xn[2] = e.z; sm.weight = w; sm.ray = e.ray; sm.sample = e.s;
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

  const int64_t warp_stride = (int64_t)gridDim.x * kWarpsPerBlock;
  for (int64_t ray64 = (int64_t)blockIdx.x * kWarpsPerBlock + warp; ray64 < p.n_rays; ray64 += warp_stride) {
    const int ray = (int)ray64;
    float ox, oy, oz, dx, dy, dz;
    if (DENSE) {
      // (point, direction) of the slot; 32-bit division whenever the slot index fits (a 64-bit divide is ~10x the cost)
      int64_t pt;
      int di;
      if (p.n_rays <= 0x7fffffffLL) {
        const uint32_t q = (uint32_t)ray64 / (uint32_t)p.n_dirs;
        pt = (int64_t)q;
        di = (int)((uint32_t)ray64 - q * (uint32_t)p.n_dirs);
      } else {
        pt = ray64 / p.n_dirs;
        di = (int)(ray64 - pt * p.n_dirs);
      }
      dx = __ldg(p.dirs + di * 3 + 0); dy = __ldg(p.dirs + di * 3 + 1); dz = __ldg(p.dirs + di * 3 + 2);
      const float nx = __ldg(p.normals + pt * 3 + 0), ny = __ldg(p.normals + pt * 3 + 1),
                  nz = __ldg(p.normals + pt * 3 + 2);
      // cosine = clamp(einsum(surf2l, normal), 0) > 1e-6 (relight_utils.py:433-435)
      const float cosine = fmaxf(fmaf(dz, nz, fmaf(dy, ny, __fmul_rn(dx, nx))), 0.f);
      if (!(cosine > 1e-6f)) continue;
      ox = __ldg(p.surf_xyz + pt * 3 + 0); oy = __ldg(p.surf_xyz + pt * 3 + 1); oz = __ldg(p.surf_xyz + pt * 3 + 2);
    } else {
      ox = __ldg(p.rays_o + ray64 * 3 + 0); oy = __ldg(p.rays_o + ray64 * 3 + 1); oz = __ldg(p.rays_o + ray64 * 3 + 2);
      dx = __ldg(p.rays_d + ray64 * 3 + 0); dy = __ldg(p.rays_d + ray64 * 3 + 1); dz = __ldg(p.rays_d + ray64 * 3 + 2);
    }
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
            valid = in_occ && alpha_mask_positive(f, px, py, pz);
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
  }
  if (qn > 0) process(qn, -1);

  c_mask = warp_sum_u64(c_mask); c_density = warp_sum_u64(c_density); c_app = warp_sum_u64(c_app);
  c_rays = warp_sum_u64(c_rays); c_over = warp_sum_u64(c_over);
  if (lane == 0 && p.counters) {
    if (c_mask) atomicAdd(p.counters + TIR_CNT_MASK, c_mask);
    if (c_density) atomicAdd(p.counters + TIR_CNT_DENSITY, c_density);
    if (c_app) atomicAdd(p.counters + TIR_CNT_APP, c_app);
    if (c_rays) atomicAdd(p.counters + TIR_CNT_RAYS, c_rays);
    if (c_over) atomicAdd(p.counters + TIR_CNT_OVERFLOW, c_over);
  }
}

template <bool WITH_APP, bool DENSE>
int launch_march(const MarchParams& p, cudaStream_t stream) {
  if (p.n_rays <= 0) return TIR_OK;
  if (p.f.dC != 16) return TIR_ERR_SHAPE;
  if (p.cfg.n_samples <= 0) return TIR_ERR_CONFIG;
  int64_t blocks = (p.n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock;
  const int64_t max_blocks = (int64_t)num_sms() * kBlocksPerSM;   // persistent: every resident CTA slot, grid-stride over rays
  if (blocks > max_blocks) blocks = max_blocks;
  if (p.cfg.sampling == TIR_SAMPLE_STEP) {
    march_kernel<16, TIR_SAMPLE_STEP, WITH_APP, DENSE><<<(int)blocks, kWarpsPerBlock * 32, 0, stream>>>(p);
  } else if (p.cfg.sampling == TIR_SAMPLE_TABLE) {
    if (!p.cfg.z_table) return TIR_ERR_NULL;
    march_kernel<16, TIR_SAMPLE_TABLE, WITH_APP, DENSE><<<(int)blocks, kWarpsPerBlock * 32, 0, stream>>>(p);
  } else {
    return TIR_ERR_CONFIG;
  }
  return (int)cudaGetLastError();
}

}  // namespace

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

extern "C" int tir_secondary_march(const TirField* field, const float* surf_xyz, const float* normals,
                                  int64_t n_pts, const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg,
                                  float* vis, TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                                  uint64_t* counters, void* stream) {
  if (n_pts <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !cfg || !surf_xyz || !normals || !dirs || !vis || !samples || !sample_count) return TIR_ERR_NULL;
  if (n_dirs <= 0) return TIR_ERR_SHAPE;
  if (capacity <= 0) return TIR_ERR_CAPACITY;
  MarchParams p{};
  p.f = *field; p.cfg = *cfg; p.surf_xyz = surf_xyz; p.normals = normals; p.dirs = dirs; p.n_dirs = n_dirs;
  p.n_rays = n_pts * (int64_t)n_dirs;
  p.t_last = vis; p.counters = (unsigned long long*)counters;
  p.samples = samples; p.sample_count = sample_count; p.capacity = capacity;
  return launch_march<true, true>(p, (cudaStream_t)stream);
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
