// One bounce of indirect light for relighting under environment maps (estimator in tir_indirect_body.h), around the
// existing density march and relighting sampler:
//
//   1. tir_indirect_sample    one thread per (ray, slot): cosine-weighted direction, throughput T, and a warp-aggregated
//                             append of (surface point, direction) to the secondary list; pos[] remembers each slot's row;
//   2. tir_march_density      (unchanged) on the list, by the caller, with relight()'s table;
//   3. tir_indirect_hits      one thread per slot, through pos[]: the 1e-3 occlusion cut, then a stable compaction (flags,
//                             CUB exclusive scan, scatter) of the secondary hits in slot order;
//   4. tir_relight_sample     (unchanged) on the hit list, by the caller, and tir_march_density from the hits;
//   5. tir_indirect_radiance  one warp per (map, hit): direct light at the hit, un-toned;
//   6. tir_indirect_shade     one warp per (map, ray): tir_relight_shade's direct sum, the indirect sum over the slots,
//                             tone and composite into the view's maps.
//
// The secondary list's order depends on warp scheduling and it is read only through pos[]; the caller puts it in slot
// order before the march (relighting.slot_order), whose result for a ray can change in its last bits with its
// neighbours.  The hit list is in slot order.  No float atomics: repeated calls give identical bits.
#include <cub/device/device_scan.cuh>

#include "tir_device.cuh"
#include "tir_indirect_body.h"

using namespace tir;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = 8;

struct SampleParams {
  const float* rays; const float* depth; const float* normal; const float* albedo; const float* rough;
  int rough_stride; const float* fresnel; const float* acc;
  int64_t n; int K; float thr; const float* rescale;
  const double* u;
  float* dir; float* T; int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kThreads) indirect_sample_kernel(const __grid_constant__ SampleParams p) {
  const int64_t total = p.n * p.K;
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  bool append = false;
  float o[3], om[3] = {0.f, 0.f, 0.f}, T[3] = {0.f, 0.f, 0.f};
  if (t < total) {
    const int64_t i = t / p.K;
    if (p.acc[i] > p.thr) {
      PointCtx c;
      const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
      rl_point(p.rays + i * 6, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
               p.fresnel + i * 3, resc, c);
      float z;
      ind_direction(p.normal + i * 3, p.u + t * 2, om, z);
      append = ind_throughput(c, om, z, T);
      if (append) rl_surface(p.rays + i * 6, p.depth[i], o);
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, om);
  if (t >= total) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) { p.dir[t * 3 + c] = om[c]; p.T[t * 3 + c] = T[c]; }
  p.pos[t] = slot;
}

struct HitsParams {
  int64_t slots;
  const int32_t* pos; const float* list_o; const float* list_d;
  const float* t_last; const float* acc; const float* depth; int vis_kind;
  float aabb[6];
  float* hit_rays; float* xn; float* w; int32_t* hit;
  int64_t capacity;
  long long* count;
};

__device__ __forceinline__ bool slot_hits(const HitsParams& p, int64_t t, int32_t& q, float& w) {
  q = p.pos[t];
  if (q < 0) return false;
  const float a = p.acc[q];
  w = ind_weight(p.vis_kind, p.t_last[q], a);
  return ind_is_hit(w, a);
}

__global__ void __launch_bounds__(kThreads) indirect_flags_kernel(const __grid_constant__ HitsParams p) {
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (t >= p.slots) return;
  int32_t q;
  float w;
  p.hit[t] = slot_hits(p, t, q, w) ? 1 : 0;
}

// hit[] holds the exclusive scan of the flags on entry and the hit row (or -1) on exit
__global__ void __launch_bounds__(kThreads) indirect_emit_kernel(const __grid_constant__ HitsParams p) {
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (t >= p.slots) return;
  int32_t q;
  float w = 0.f;
  const bool h = slot_hits(p, t, q, w);
  const int64_t row = p.hit[t];
  if (t == p.slots - 1) *p.count = row + (h ? 1 : 0);
  int32_t out = -1;
  if (h && row < p.capacity) {
    float o[3], d[3], x[3], xn[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { o[c] = p.list_o[(int64_t)q * 3 + c]; d[c] = p.list_d[(int64_t)q * 3 + c]; }
    ind_point(o, d, p.depth[q], p.acc[q], p.aabb, x, xn);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      p.hit_rays[row * 6 + c] = x[c];
      p.hit_rays[row * 6 + 3 + c] = d[c];
      p.xn[row * 3 + c] = xn[c];
    }
    p.w[row] = w;
    out = (int32_t)row;
  }
  p.hit[t] = out;
}

cudaError_t scan_temp_bytes(int64_t slots, size_t* bytes) {
  *bytes = 0;
  return cub::DeviceScan::ExclusiveSum(nullptr, *bytes, (int32_t*)nullptr, (int32_t*)nullptr, (int)slots);
}

struct RadianceParams {
  EnvTable env;
  const float* rays; const float* normal; const float* albedo; const float* rough; int rough_stride;
  const float* fresnel;
  int64_t m; int S; const float* rescale;
  const int32_t* bin; const int32_t* pos; const float* vis; int vis_kind;
  float* Lo; int64_t out_rows; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) indirect_radiance_kernel(const __grid_constant__ RadianceParams p, int L) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (w >= (int64_t)L * p.m) return;
  const int l = (int)(w / p.m);
  const int64_t h = w - (int64_t)l * p.m;
  PointCtx c;
  const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
  rl_point(p.rays + h * 6, p.normal + h * 3, p.albedo + h * 3, p.rough + h * p.rough_stride, p.rough_stride,
           p.fresnel + h * 3, resc, c);
  float acc[3] = {0.f, 0.f, 0.f};
  const int64_t k0 = w * p.S;
  rl_direct_lane(p.env.e[l], c, p.bin + k0, p.pos + k0, p.vis, p.vis_kind, p.S, lane, 32, acc);
  float lo[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) lo[ch] = warp_sum(acc[ch]) / (float)p.S;
  if (lane != 0) return;
  const int64_t r = ((int64_t)l * p.out_rows + p.row0 + h) * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) p.Lo[r + ch] = lo[ch];
}

struct ShadeParams {
  EnvTable env;
  const float* rays; const float* normal; const float* albedo; const float* rough; int rough_stride;
  const float* fresnel; const float* acc;
  int64_t n; int S; float thr; const float* rescale;
  const int32_t* bin; const int32_t* pos; const float* vis; int vis_kind;
  int K; const float* T; const int32_t* hit; const float* w; const float* Lo; int64_t m_h;
  float* with_bg; float* without_bg; float* indirect; int64_t out_rows; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) indirect_shade_kernel(const __grid_constant__ ShadeParams p, int L) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (w >= (int64_t)L * p.n) return;
  const int l = (int)(w / p.n);
  const int64_t i = w - (int64_t)l * p.n;
  const TirEnvMap& e = p.env.e[l];
  const float* ray = p.rays + i * 6;
  const float a = p.acc[i];
  float wo[3] = {1.f, 1.f, 1.f}, ind[3] = {0.f, 0.f, 0.f};
  if (a > p.thr) {
    PointCtx c;
    const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
    rl_point(ray, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
             p.fresnel + i * 3, resc, c);
    float acc[3] = {0.f, 0.f, 0.f};
    rl_direct_lane(e, c, p.bin + w * p.S, p.pos + w * p.S, p.vis, p.vis_kind, p.S, lane, 32, acc);
    float ia[3] = {0.f, 0.f, 0.f};
    bool any = false;
    for (int k = lane; k < p.K; k += 32) {
      const int64_t t = i * p.K + k;
      const int h = p.hit[t];
      if (h < 0) continue;
      any = true;
      const float T[3] = {p.T[t * 3], p.T[t * 3 + 1], p.T[t * 3 + 2]};
      const float* lo = p.Lo + ((int64_t)l * p.m_h + h) * 3;
      const float Lo[3] = {lo[0], lo[1], lo[2]};
      ind_add(T, p.w[h], Lo, ia);
    }
    any = __any_sync(0xffffffffu, any);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float d = warp_sum(acc[ch]) / (float)p.S;
      const float s = warp_sum(ia[ch]);
      if (any) ind[ch] = ev_div(s, (float)p.K);
      wo[ch] = tone(any ? ev_add(d, ind[ch]) : d, 1);
    }
  }
  if (lane != 0) return;
  float wb[3];
  rl_composite(e, ray, a, wo, wb);
  const int64_t r = ((int64_t)l * p.out_rows + p.row0 + i) * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    p.without_bg[r + ch] = wo[ch];
    p.with_bg[r + ch] = wb[ch];
    if (p.indirect) p.indirect[r + ch] = ind[ch];
  }
}

void copy_envs(EnvTable& t, const TirEnvMap* envs, int L) {
  for (int l = 0; l < L; ++l) t.e[l] = envs[l];
}

}  // namespace

extern "C" int tir_indirect_sample(const float* rays, const float* depth, const float* normal, const float* albedo,
                                   const float* rough, int32_t rough_stride, const float* fresnel, const float* acc,
                                   int64_t n, int32_t K, float acc_mask_threshold, const float* rescale,
                                   const double* u, float* dir, float* T, int32_t* pos, float* list_o, float* list_d,
                                   int64_t capacity, int64_t* count, void* stream) {
  const int rc = ind_sample_check(rays, depth, normal, albedo, rough, rough_stride, fresnel, acc, n, K, rescale, u, dir,
                                  T, pos, list_o, list_d, capacity, count);
  if (rc <= 0) return rc;
  SampleParams p{};
  p.rays = rays; p.depth = depth; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.acc = acc; p.n = n; p.K = K; p.thr = acc_mask_threshold; p.u = u; p.dir = dir; p.T = T;
  p.pos = pos; p.list_o = list_o; p.list_d = list_d; p.capacity = capacity;
  p.count = reinterpret_cast<unsigned long long*>(count);
  p.rescale = rescale;
  const int64_t total = n * K;
  indirect_sample_kernel<<<(unsigned)((total + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_indirect_hits_work_size(int64_t n, int32_t K, int64_t* bytes) {
  const int rc = ind_hits_work_size_check(n, K, bytes);
  if (rc <= 0) return rc;
  size_t b = 0;
  const cudaError_t e = scan_temp_bytes(n * K, &b);
  if (e != cudaSuccess) return (int)e;
  *bytes = (int64_t)b;
  return TIR_OK;
}

extern "C" int tir_indirect_hits(int64_t n, int32_t K, const int32_t* pos, const float* list_o, const float* list_d,
                                 const float* t_last, const float* acc, const float* depth, int32_t vis_kind,
                                 const float* aabb, float* hit_rays, float* xn, float* w, int32_t* hit,
                                 int64_t capacity, int64_t* count, void* work, int64_t work_bytes, void* stream) {
  const int rc = ind_hits_check(n, K, pos, list_o, list_d, t_last, acc, depth, vis_kind, aabb, hit_rays, xn, w, hit,
                                capacity, count);
  if (rc < 0) return rc;
  if (rc == 0) return (int)cudaMemsetAsync(count, 0, sizeof(int64_t), (cudaStream_t)stream);
  const int64_t slots = n * K;
  size_t temp = 0;
  cudaError_t e = scan_temp_bytes(slots, &temp);
  if (e != cudaSuccess) return (int)e;
  if (!work && temp > 0) return TIR_ERR_NULL;
  if (work_bytes < (int64_t)temp) return TIR_ERR_CAPACITY;
  HitsParams p{};
  p.slots = slots; p.pos = pos; p.list_o = list_o; p.list_d = list_d; p.t_last = t_last; p.acc = acc; p.depth = depth;
  p.vis_kind = vis_kind; p.hit_rays = hit_rays; p.xn = xn; p.w = w; p.hit = hit; p.capacity = capacity;
  p.count = reinterpret_cast<long long*>(count);
  for (int c = 0; c < 6; ++c) p.aabb[c] = aabb[c];
  const cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((slots + kThreads - 1) / kThreads);
  indirect_flags_kernel<<<blocks, kThreads, 0, s>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  e = cub::DeviceScan::ExclusiveSum(work, temp, hit, hit, (int)slots, s);
  if (e != cudaSuccess) return (int)e;
  indirect_emit_kernel<<<blocks, kThreads, 0, s>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_indirect_radiance(const TirEnvMap* envs, int32_t n_lights, const float* hit_rays,
                                     const float* normal, const float* albedo, const float* rough,
                                     int32_t rough_stride, const float* fresnel, int64_t m, int32_t n_samples,
                                     const float* rescale, const int32_t* bin, const int32_t* pos,
                                     const float* vis_list, int32_t vis_kind, float* Lo, int64_t out_rows,
                                     int64_t row0, void* stream) {
  const int rc = ind_radiance_check(envs, n_lights, hit_rays, normal, albedo, rough, rough_stride, fresnel, m,
                                    n_samples, rescale, bin, pos, vis_list, vis_kind, Lo, out_rows, row0);
  if (rc <= 0) return rc;
  RadianceParams p{};
  copy_envs(p.env, envs, n_lights);
  p.rays = hit_rays; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.m = m; p.S = n_samples; p.bin = bin; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind;
  p.Lo = Lo; p.out_rows = out_rows; p.row0 = row0;
  p.rescale = rescale;
  const int64_t warps = (int64_t)n_lights * m;
  indirect_radiance_kernel<<<(unsigned)((warps + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(
      p, n_lights);
  return (int)cudaGetLastError();
}

extern "C" int tir_indirect_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                                  const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                                  const float* acc, int64_t n, int32_t n_samples, float acc_mask_threshold,
                                  const float* rescale, const int32_t* bin, const int32_t* pos, const float* vis_list,
                                  int32_t vis_kind, int32_t K, const float* T, const int32_t* hit, const float* w,
                                  const float* Lo, int64_t m_h, float* with_bg, float* without_bg, float* indirect,
                                  int64_t out_rows, int64_t row0, void* stream) {
  const int rc = ind_shade_check(envs, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, n_samples,
                                 rescale, bin, pos, vis_kind, K, T, hit, w, Lo, m_h, with_bg, without_bg, out_rows,
                                 row0);
  if (rc <= 0) return rc;
  ShadeParams p{};
  copy_envs(p.env, envs, n_lights);
  p.rays = rays; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.acc = acc; p.n = n; p.S = n_samples; p.thr = acc_mask_threshold; p.bin = bin; p.pos = pos;
  p.vis = vis_list; p.vis_kind = vis_kind; p.K = K; p.T = T; p.hit = hit; p.w = w; p.Lo = Lo; p.m_h = m_h;
  p.with_bg = with_bg; p.without_bg = without_bg; p.indirect = indirect; p.out_rows = out_rows; p.row0 = row0;
  p.rescale = rescale;
  const int64_t warps = (int64_t)n_lights * n;
  indirect_shade_kernel<<<(unsigned)((warps + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(
      p, n_lights);
  return (int)cudaGetLastError();
}
