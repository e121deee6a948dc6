// Relighting of one chunk of primary rays under L environment maps (scripts/relight_importance.py:99-181), around the
// existing density march:
//
//   1. tir_relight_sample  one thread per (map, ray, sample): inverse-CDF bin of the caller's uniform draw, the raw-normal
//                          cosine test, and a warp-aggregated append of (surface point, direction) to the visibility
//                          list; the slot map pos[] remembers where each sample went;
//   2. tir_march_density   (unchanged) on the list, by the caller, sized by the list length read back once per chunk;
//   3. tir_relight_shade   one warp per (map, ray), lanes stride over the samples: GGX + Lambert, visibility, light and
//                          pdf weighting, fixed-order mean, clamp, sRGB, background lookup and compositing, written
//                          straight into the view's maps.
//
// This replaces the ~70 element-wise / gather / compaction launches per map of the eager chunk body.  The list order
// depends on warp scheduling, but every sample reads its own row back through pos[], so the outputs do not.
#include "tir_device.cuh"
#include "tir_relight_body.h"

using namespace tir;

namespace {

constexpr int kSampleThreads = 256;
constexpr int kWarps = 8;

struct SampleParams {
  EnvTable env;
  const float* rays; const float* depth; const float* normal; const float* acc;
  int64_t n; int S; float thr;
  const double* u;
  int32_t* bin; int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kSampleThreads) relight_sample_kernel(const SampleParams p, int L) {
  const int64_t total = (int64_t)L * p.n * p.S;
  const int64_t t = (int64_t)blockIdx.x * kSampleThreads + threadIdx.x;
  bool append = false;
  float o[3], L3[3];
  int b = 0;
  if (t < total) {
    const int64_t li = t / p.S;            // (map, ray)
    const int l = (int)(li / p.n);
    const int64_t i = li - (int64_t)l * p.n;
    if (p.acc[i] > p.thr) {
      const TirEnvMap& e = p.env.e[l];
      b = rl_bin(e.cdf, e.H * e.W, p.u[t]);
      float nrm[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) { L3[c] = __ldg(e.dir + (int64_t)b * 3 + c); nrm[c] = p.normal[i * 3 + c]; }
      append = rl_cosine(L3, nrm) > 1e-6f;
      if (append) rl_surface(p.rays + i * 6, p.depth[i], o);
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, L3);
  if (t >= total) return;
  p.bin[t] = b;
  p.pos[t] = slot;
}

struct ShadeParams {
  EnvTable env;
  const float* rays; const float* normal; const float* albedo; const float* rough; int rough_stride;
  const float* fresnel; const float* acc;
  int64_t n; int S; float thr;
  const float* rescale;
  const int32_t* bin; const int32_t* pos; const float* vis; int vis_kind;
  float* with_bg; float* without_bg; int64_t out_rows; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) relight_shade_kernel(const ShadeParams p, int L) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (w >= (int64_t)L * p.n) return;
  const int l = (int)(w / p.n);
  const int64_t i = w - (int64_t)l * p.n;
  const TirEnvMap& e = p.env.e[l];
  const float* ray = p.rays + i * 6;
  const float a = p.acc[i];
  float wo[3] = {1.f, 1.f, 1.f};
  if (a > p.thr) {
    PointCtx c;
    const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
    rl_point(ray, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
             p.fresnel + i * 3, resc, c);
    float acc[3] = {0.f, 0.f, 0.f};
    const int64_t k0 = w * p.S;
    rl_direct_lane(e, c, p.bin + k0, p.pos + k0, p.vis, p.vis_kind, p.S, lane, 32, acc);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) wo[ch] = tone(warp_sum(acc[ch]) / (float)p.S, 1);
  }
  if (lane != 0) return;
  float wb[3];
  rl_composite(e, ray, a, wo, wb);
  const int64_t r = ((int64_t)l * p.out_rows + p.row0 + i) * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) { p.without_bg[r + ch] = wo[ch]; p.with_bg[r + ch] = wb[ch]; }
}

}  // namespace

extern "C" int tir_relight_sample(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* depth,
                                  const float* normal, const float* acc, int64_t n, int32_t n_samples,
                                  float acc_mask_threshold, const double* u, int32_t* bin, int32_t* pos,
                                  float* list_o, float* list_d, int64_t capacity, int64_t* count, void* stream) {
  const int rc = rl_sample_check(envs, n_lights, rays, depth, normal, acc, n, n_samples, u, bin, pos, list_o, list_d,
                                 capacity, count);
  if (rc <= 0) return rc;
  SampleParams p{};
  for (int l = 0; l < n_lights; ++l) p.env.e[l] = envs[l];
  p.rays = rays; p.depth = depth; p.normal = normal; p.acc = acc; p.n = n; p.S = n_samples;
  p.thr = acc_mask_threshold; p.u = u; p.bin = bin; p.pos = pos; p.list_o = list_o; p.list_d = list_d;
  p.capacity = capacity; p.count = reinterpret_cast<unsigned long long*>(count);
  const int64_t total = (int64_t)n_lights * n * n_samples;
  relight_sample_kernel<<<(unsigned)((total + kSampleThreads - 1) / kSampleThreads), kSampleThreads, 0,
                          (cudaStream_t)stream>>>(p, n_lights);
  return (int)cudaGetLastError();
}

extern "C" int tir_relight_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                                 const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                                 const float* acc, int64_t n, int32_t n_samples, float acc_mask_threshold,
                                 const float* rescale, const int32_t* bin, const int32_t* pos, const float* vis_list,
                                 int32_t vis_kind, float* with_bg, float* without_bg, int64_t out_rows, int64_t row0,
                                 void* stream) {
  const int rc = rl_shade_check(envs, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, n_samples,
                                rescale, bin, pos, vis_kind, with_bg, without_bg, out_rows, row0);
  if (rc <= 0) return rc;
  ShadeParams p{};
  for (int l = 0; l < n_lights; ++l) p.env.e[l] = envs[l];
  p.rays = rays; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.acc = acc; p.n = n; p.S = n_samples; p.thr = acc_mask_threshold; p.rescale = rescale;
  p.bin = bin; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind; p.with_bg = with_bg; p.without_bg = without_bg;
  p.out_rows = out_rows; p.row0 = row0;
  const int64_t warps = (int64_t)n_lights * n;
  relight_shade_kernel<<<(unsigned)((warps + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p, n_lights);
  return (int)cudaGetLastError();
}
