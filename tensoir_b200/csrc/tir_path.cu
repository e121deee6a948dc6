// Camera-path frames under rotated environment maps with a shadow-catching ground plane, around the existing relighting
// calls (the object is shaded by tir_relight_sample / tir_march_density / tir_relight_shade with the maps' direction
// tables rotated on the host):
//
//   1. tir_ground_sample   one thread per (map, ray, slot) of a ray that meets the ground: inverse-CDF bin of the
//                          caller's uniform draw, the horizon test, the slab test of the shadow ray against the model's
//                          occupied box, and a warp-aggregated append of the rays that meet it to a visibility list;
//                          pos[] remembers where each slot went (-1 nowhere, -2 unoccluded);
//   2. tir_march_density   (unchanged) on the list, by the caller;
//   3. tir_path_composite  one warp per (map, pixel), lanes stride over the ground slots: the shadow ratio of the ground
//                          point, the background at the rotated direction, and the composite under the object, written
//                          straight into the frame's map.
//
// Under a setup of analytic lights (the object shaded by tir_lights_sample / tir_march_density / tir_lights_shade), the
// same three steps with the lights' samples in place of the map's texels:
//
//   1. tir_ground_lights_sample   one thread per (light, ray, area sample) slot, laid out as tir_lights_sample's: the
//                                 light sample seen from the ground point, its weight falloff * L.z, the horizon test,
//                                 the slab test and, for a point or spot light, the distance cull; append as above;
//   3. tir_path_lights_composite  one warp per pixel: per light, lanes stride over its slots, the butterfly sums them,
//                                 the lights add up in order; the setup's background, darkened in linear light by the
//                                 ratio, under the object.
//
// An infinite plane costs march work only where the object can shadow it: a shadow ray that misses the box needs no
// march.  The list order depends on warp scheduling, but every slot reads its own row back through pos[], so the
// outputs do not.
#include "tir_device.cuh"
#include "tir_path_body.h"

using namespace tir;

namespace {

constexpr int kSampleThreads = 256;
constexpr int kWarps = 8;

struct GroundParams {
  EnvTable env;
  const float* rays;
  int64_t n; int S; float ground_z;
  float lo[3], hi[3];
  const double* u;
  int32_t* bin; int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kSampleThreads) ground_sample_kernel(const __grid_constant__ GroundParams p, int L) {
  const int64_t total = (int64_t)L * p.n * p.S;
  const int64_t t = (int64_t)blockIdx.x * kSampleThreads + threadIdx.x;
  bool append = false;
  float o[3], w[3];
  int b = 0, q = -1;
  if (t < total) {
    const int64_t li = t / p.S;            // (map, ray)
    const int l = (int)(li / p.n);
    const int64_t i = li - (int64_t)l * p.n;
    float g[3];
    if (pt_ground(p.rays + i * 6, p.ground_z, g)) {
      const TirEnvMap& e = p.env.e[l];
      b = rl_bin(e.cdf, e.H * e.W, p.u[t]);
#pragma unroll
      for (int c = 0; c < 3; ++c) w[c] = __ldg(e.dir + (int64_t)b * 3 + c);
      q = pt_ground_slot(g, w, p.lo, p.hi, o);
      append = q == 0;
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, w);
  if (t >= total) return;
  p.bin[t] = b;
  p.pos[t] = append ? slot : q;
}

struct CompositeParams {
  EnvTable env;
  const float* rays; const float* acc;
  int64_t n; float rot[9]; float ground_z;
  const int32_t* bin; const int32_t* pos; const float* vis; int vis_kind; int S;
  const float* without_bg; float* with_bg; float* shadow; int64_t out_rows; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) path_composite_kernel(const __grid_constant__ CompositeParams p, int L) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (w >= (int64_t)L * p.n) return;
  const int l = (int)(w / p.n);
  const int64_t i = w - (int64_t)l * p.n;
  const TirEnvMap& e = p.env.e[l];
  const float* ray = p.rays + i * 6;
  float r[3] = {1.f, 1.f, 1.f};
  float g[3];
  if (pt_ground(ray, p.ground_z, g)) {
    float num[3] = {0.f, 0.f, 0.f}, den[3] = {0.f, 0.f, 0.f};
    const int64_t k0 = w * p.S;
    pt_shadow_lane(e, p.bin + k0, p.pos + k0, p.vis, p.vis_kind, p.S, lane, 32, num, den);
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = pt_ratio(warp_sum(num[c]), warp_sum(den[c]));
  }
  if (lane != 0) return;
  const int64_t row = ((int64_t)l * p.out_rows + p.row0 + i) * 3;
  const float wo[3] = {p.without_bg[row], p.without_bg[row + 1], p.without_bg[row + 2]};
  float wb[3];
  pt_composite(e, ray, p.rot, p.acc[i], wo, r, wb);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p.with_bg[row + c] = wb[c];
    if (p.shadow) p.shadow[row + c] = r[c];
  }
}

struct GroundLightsParams {
  LightTable lt;
  int n_lights;
  const float* rays;
  int64_t n; float ground_z;
  float lo[3], hi[3];
  const double* u;
  float* g; int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kSampleThreads) ground_lights_sample_kernel(
    const __grid_constant__ GroundLightsParams p) {
  const int64_t total = p.n * p.lt.prefix[p.n_lights];
  const int64_t t = (int64_t)blockIdx.x * kSampleThreads + threadIdx.x;
  bool append = false;
  float o[3], L3[3] = {0.f, 0.f, 0.f}, gw = 0.f;
  int q = -1;
  if (t < total) {
    int j = 0;
    while (j + 1 < p.n_lights && t >= p.n * p.lt.prefix[j + 1]) ++j;
    const int64_t i = (t - p.n * p.lt.prefix[j]) / p.lt.l[j].n_samples;
    float gp[3];
    if (pt_ground(p.rays + i * 6, p.ground_z, gp)) {
      float fall, d2 = INFINITY;
      lt_sample(p.lt.l[j], gp, p.u + t * 2, L3, fall, &d2);
      gw = ev_mul(fall, L3[2]);
      q = pt_light_slot(p.lt.l[j], gp, L3, gw, d2, p.lo, p.hi, o);
      append = q == 0;
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, L3);
  if (t >= total) return;
  p.g[t] = gw;
  p.pos[t] = append ? slot : q;
}

struct LightsCompositeParams {
  LightTable lt;
  int n_lights;
  const float* rays; const float* acc;
  int64_t n; float ground_z;
  float bg[3], bg_lin[3];
  const float* g; const int32_t* pos; const float* vis; int vis_kind;
  const float* without_bg; float* with_bg; float* shadow; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) path_lights_composite_kernel(
    const __grid_constant__ LightsCompositeParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (i >= p.n) return;
  const float* ray = p.rays + i * 6;
  float r[3] = {1.f, 1.f, 1.f};
  float gp[3];
  if (pt_ground(ray, p.ground_z, gp)) {
    float num[3] = {0.f, 0.f, 0.f}, den[3] = {0.f, 0.f, 0.f};
    for (int j = 0; j < p.n_lights; ++j) {
      const int K = p.lt.l[j].n_samples;
      const int64_t k0 = p.n * p.lt.prefix[j] + i * K;
      float sn = 0.f, sd = 0.f;
      pt_light_lane(p.g + k0, p.pos + k0, p.vis, p.vis_kind, K, lane, 32, sn, sd);
      pt_light_add(p.lt.l[j], K, warp_sum(sn), warp_sum(sd), num, den);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = pt_ratio(num[c], den[c]);
  }
  if (lane != 0) return;
  const int64_t row = (p.row0 + i) * 3;
  const float wo[3] = {p.without_bg[row], p.without_bg[row + 1], p.without_bg[row + 2]};
  float wb[3];
  pt_lights_composite(p.bg, p.bg_lin, p.acc[i], wo, r, wb);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    p.with_bg[row + c] = wb[c];
    if (p.shadow) p.shadow[row + c] = r[c];
  }
}

}  // namespace

extern "C" int tir_ground_lights_sample(const TirLight* lights, int32_t n_lights, const float* rays, int64_t n,
                                        float ground_z, const float* box_lo, const float* box_hi, const double* u,
                                        float* g, int32_t* pos, float* list_o, float* list_d, int64_t capacity,
                                        int64_t* count, void* stream) {
  GroundLightsParams p{};
  const int rc = pt_lights_sample_check(lights, n_lights, rays, n, box_lo, box_hi, u, g, pos, list_o, list_d, capacity,
                                        count, p.lt);
  if (rc <= 0) return rc;
  p.n_lights = n_lights;
  p.rays = rays; p.n = n; p.ground_z = ground_z;
  for (int c = 0; c < 3; ++c) { p.lo[c] = box_lo[c]; p.hi[c] = box_hi[c]; }
  p.u = u; p.g = g; p.pos = pos; p.list_o = list_o; p.list_d = list_d; p.capacity = capacity;
  p.count = reinterpret_cast<unsigned long long*>(count);
  const int64_t total = n * p.lt.prefix[n_lights];
  ground_lights_sample_kernel<<<(unsigned)((total + kSampleThreads - 1) / kSampleThreads), kSampleThreads, 0,
                                (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_path_lights_composite(const TirLight* lights, int32_t n_lights, const float* rays,
                                         const float* acc, int64_t n, float ground_z, const float* background,
                                         const float* background_linear, const float* g, const int32_t* pos,
                                         const float* vis_list, int32_t vis_kind, const float* without_bg,
                                         float* with_bg, float* shadow, int64_t out_rows, int64_t row0, void* stream) {
  LightsCompositeParams p{};
  const int rc = pt_lights_composite_check(lights, n_lights, rays, acc, n, ground_z, background, background_linear, g,
                                           pos, vis_list, vis_kind, without_bg, with_bg, out_rows, row0, p.lt);
  if (rc <= 0) return rc;
  p.n_lights = n_lights;
  p.rays = rays; p.acc = acc; p.n = n; p.ground_z = ground_z;
  for (int c = 0; c < 3; ++c) { p.bg[c] = background[c]; p.bg_lin[c] = background_linear[c]; }
  p.g = g; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind;
  p.without_bg = without_bg; p.with_bg = with_bg; p.shadow = shadow; p.row0 = row0;
  path_lights_composite_kernel<<<(unsigned)((n + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_ground_sample(const TirEnvMap* envs, int32_t n_lights, const float* rays, int64_t n,
                                 float ground_z, const float* box_lo, const float* box_hi, int32_t n_samples,
                                 const double* u, int32_t* bin, int32_t* pos, float* list_o, float* list_d,
                                 int64_t capacity, int64_t* count, void* stream) {
  const int rc = pt_sample_check(envs, n_lights, rays, n, box_lo, box_hi, n_samples, u, bin, pos, list_o, list_d,
                                 capacity, count);
  if (rc <= 0) return rc;
  GroundParams p{};
  for (int l = 0; l < n_lights; ++l) p.env.e[l] = envs[l];
  p.rays = rays; p.n = n; p.S = n_samples; p.ground_z = ground_z;
  for (int c = 0; c < 3; ++c) { p.lo[c] = box_lo[c]; p.hi[c] = box_hi[c]; }
  p.u = u; p.bin = bin; p.pos = pos; p.list_o = list_o; p.list_d = list_d; p.capacity = capacity;
  p.count = reinterpret_cast<unsigned long long*>(count);
  const int64_t total = (int64_t)n_lights * n * n_samples;
  ground_sample_kernel<<<(unsigned)((total + kSampleThreads - 1) / kSampleThreads), kSampleThreads, 0,
                         (cudaStream_t)stream>>>(p, n_lights);
  return (int)cudaGetLastError();
}

extern "C" int tir_path_composite(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* acc,
                                  int64_t n, const float* rot, float ground_z, const int32_t* bin, const int32_t* pos,
                                  const float* vis_list, int32_t vis_kind, int32_t n_samples, const float* without_bg,
                                  float* with_bg, float* shadow, int64_t out_rows, int64_t row0, void* stream) {
  const int rc = pt_composite_check(envs, n_lights, rays, acc, n, rot, ground_z, bin, pos, vis_list, vis_kind,
                                    n_samples, without_bg, with_bg, out_rows, row0);
  if (rc <= 0) return rc;
  CompositeParams p{};
  for (int l = 0; l < n_lights; ++l) p.env.e[l] = envs[l];
  p.rays = rays; p.acc = acc; p.n = n; p.ground_z = ground_z;
  for (int k = 0; k < 9; ++k) p.rot[k] = rot[k];
  p.bin = bin; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind; p.S = isnan(ground_z) ? 0 : n_samples;
  p.without_bg = without_bg; p.with_bg = with_bg; p.shadow = shadow; p.out_rows = out_rows; p.row0 = row0;
  const int64_t warps = (int64_t)n_lights * n;
  path_composite_kernel<<<(unsigned)((warps + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(
      p, n_lights);
  return (int)cudaGetLastError();
}
