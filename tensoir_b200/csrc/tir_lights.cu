// Relighting of one chunk of primary rays under one setup of analytic lights (directional, point, spot), around the
// existing density march, in the shape of tir_relight.cu:
//
//   1. tir_lights_sample  one thread per slot (light, ray, area sample): the direction and falloff of the light sample
//                         seen from the surface point, the raw-normal cosine test, and a warp-aggregated append of
//                         (surface point, direction) to the shadow-ray list; pos[] remembers where each slot went;
//   2. tir_march_density  (unchanged) on the list, by the caller, sized by the list length read back once per chunk;
//   3. tir_lights_shade   one warp per ray: per light, lanes stride over its slots (GGX + Lambert, visibility, falloff,
//                         cosine), a fixed-order butterfly sums them, the lights add up in order; clamp, sRGB and
//                         compositing over the setup's background colour, written straight into the view's maps.
//
// A hard-shadowed light is one slot and one shadow ray per hit.  The list order depends on warp scheduling, but every
// slot reads its own row back through pos[], so the outputs do not.
#include "tir_device.cuh"
#include "tir_lights_body.h"

using namespace tir;

namespace {

constexpr int kSampleThreads = 256;
constexpr int kWarps = 8;

struct LightsSampleParams {
  LightTable lt;
  int n_lights;
  const float* rays; const float* depth; const float* normal; const float* acc;
  int64_t n; float thr;
  const double* u;
  float* L; float* falloff; int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kSampleThreads) lights_sample_kernel(const __grid_constant__ LightsSampleParams p) {
  const int64_t total = p.n * p.lt.prefix[p.n_lights];
  const int64_t t = (int64_t)blockIdx.x * kSampleThreads + threadIdx.x;
  bool append = false;
  float o[3], L3[3] = {0.f, 0.f, 0.f}, fall = 0.f;
  if (t < total) {
    int j = 0;
    while (j + 1 < p.n_lights && t >= p.n * p.lt.prefix[j + 1]) ++j;
    const int64_t i = (t - p.n * p.lt.prefix[j]) / p.lt.l[j].n_samples;
    if (p.acc[i] > p.thr) {
      rl_surface(p.rays + i * 6, p.depth[i], o);
      lt_sample(p.lt.l[j], o, p.u + t * 2, L3, fall);
      float nrm[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) nrm[c] = p.normal[i * 3 + c];
      append = rl_cosine(L3, nrm) > 1e-6f && fall > 0.f;
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, L3);
  if (t >= total) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) p.L[t * 3 + c] = L3[c];
  p.falloff[t] = fall;
  p.pos[t] = slot;
}

struct LightsShadeParams {
  LightTable lt;
  int n_lights;
  const float* rays; const float* normal; const float* albedo; const float* rough; int rough_stride;
  const float* fresnel; const float* acc;
  int64_t n; float thr;
  const float* rescale; const float* background;
  const float* L; const float* falloff; const int32_t* pos; const float* vis; int vis_kind;
  float* with_bg; float* without_bg; float* linear; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) lights_shade_kernel(const __grid_constant__ LightsShadeParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (i >= p.n) return;
  const float a = p.acc[i];
  const bool hit = a > p.thr;
  float lin[3] = {0.f, 0.f, 0.f};
  if (hit) {
    PointCtx c;
    const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
    rl_point(p.rays + i * 6, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
             p.fresnel + i * 3, resc, c);
    for (int j = 0; j < p.n_lights; ++j) {
      const int K = p.lt.l[j].n_samples;
      const int64_t k0 = p.n * p.lt.prefix[j] + i * K;
      float acc[3] = {0.f, 0.f, 0.f};
      for (int s = lane; s < K; s += 32) {
        const int q = p.pos[k0 + s];
        if (q < 0) continue;
        const float vis = rl_vis(p.vis, p.vis_kind, q);
        const float Ld[3] = {p.L[(k0 + s) * 3], p.L[(k0 + s) * 3 + 1], p.L[(k0 + s) * 3 + 2]};
        lt_contrib(c, Ld, p.falloff[k0 + s], vis, acc);
      }
#pragma unroll
      for (int ch = 0; ch < 3; ++ch)
        lin[ch] = ev_add(lin[ch], ev_mul(p.lt.l[j].power[ch], warp_sum(acc[ch]) / (float)K));
    }
  }
  if (lane != 0) return;
  float wo[3], wb[3];
  lt_finish(hit, a, lin, p.background, wo, wb);
  const int64_t r = (p.row0 + i) * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    p.without_bg[r + ch] = wo[ch];
    p.with_bg[r + ch] = wb[ch];
    if (p.linear) p.linear[r + ch] = lin[ch];
  }
}

}  // namespace

extern "C" int tir_lights_sample(const TirLight* lights, int32_t n_lights, const float* rays, const float* depth,
                                 const float* normal, const float* acc, int64_t n, float acc_mask_threshold,
                                 const double* u, float* L, float* falloff, int32_t* pos, float* list_o, float* list_d,
                                 int64_t capacity, int64_t* count, void* stream) {
  LightsSampleParams p{};
  const int rc = lt_sample_check(lights, n_lights, rays, depth, normal, acc, n, u, L, falloff, pos, list_o, list_d,
                                 capacity, count, p.lt);
  if (rc <= 0) return rc;
  p.n_lights = n_lights;
  p.rays = rays; p.depth = depth; p.normal = normal; p.acc = acc; p.n = n; p.thr = acc_mask_threshold; p.u = u;
  p.L = L; p.falloff = falloff; p.pos = pos; p.list_o = list_o; p.list_d = list_d; p.capacity = capacity;
  p.count = reinterpret_cast<unsigned long long*>(count);
  const int64_t total = n * p.lt.prefix[n_lights];
  lights_sample_kernel<<<(unsigned)((total + kSampleThreads - 1) / kSampleThreads), kSampleThreads, 0,
                         (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_lights_shade(const TirLight* lights, int32_t n_lights, const float* rays, const float* normal,
                                const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                                const float* acc, int64_t n, float acc_mask_threshold, const float* rescale,
                                const float* background, const float* L, const float* falloff, const int32_t* pos,
                                const float* vis_list, int32_t vis_kind, float* with_bg, float* without_bg,
                                float* linear, int64_t out_rows, int64_t row0, void* stream) {
  LightsShadeParams p{};
  const int rc = lt_shade_check(lights, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, rescale,
                                background, L, falloff, pos, vis_list, vis_kind, with_bg, without_bg, out_rows, row0,
                                p.lt);
  if (rc <= 0) return rc;
  p.n_lights = n_lights;
  p.rays = rays; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.acc = acc; p.n = n; p.thr = acc_mask_threshold; p.rescale = rescale;
  p.background = background; p.L = L; p.falloff = falloff; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind;
  p.with_bg = with_bg; p.without_bg = without_bg; p.linear = linear; p.row0 = row0;
  lights_shade_kernel<<<(unsigned)((n + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}
