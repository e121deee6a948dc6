// Relighting of one chunk of primary rays under L environment maps with multiple importance sampling (estimator in
// tir_mis_body.h), around the existing density march:
//
//   1. tir_relight_mis_sample  one thread per slot: the L*n*S_l light slots (texel from the CDF, a point uniform in its
//                              solid angle) and then the n*S_b BRDF slots shared by every map (GGX visible normals or
//                              cosine); the raw-normal cosine test and a warp-aggregated append of (surface point,
//                              direction) to the visibility list; pos[] remembers each slot's row;
//   2. tir_march_density       (unchanged) on the list, by the caller, in slot order (relighting.slot_order);
//   3. tir_relight_mis_shade   one warp per (map, ray), lanes stride over the map's light slots and then the ray's BRDF
//                              slots: texel lookup, both densities, BRDF, visibility, fixed-order sum, clamp, sRGB and
//                              compositing into the view's maps.
//
// The list order depends on warp scheduling, but every slot reads its own row back through pos[]; no float atomics.
#include "tir_device.cuh"
#include "tir_mis_body.h"

using namespace tir;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = 8;

struct SampleParams {
  EnvTable env;
  const float* rays; const float* depth; const float* normal; const float* albedo; const float* rough;
  int rough_stride; const float* fresnel; const float* acc;
  int64_t n; int S_l, S_b; float thr;
  const double* u_light; const double* u_brdf;
  float* dir; int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kThreads) mis_sample_kernel(const __grid_constant__ SampleParams p, int L) {
  const int64_t n_light = (int64_t)L * p.n * p.S_l;
  const int64_t total = n_light + p.n * p.S_b;
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  bool append = false;
  float o[3], w[3] = {0.f, 0.f, 0.f};
  if (t < total) {
    const bool light = t < n_light;
    const int64_t i = light ? (t / p.S_l) % p.n : (t - n_light) / p.S_b;
    if (p.acc[i] > p.thr) {
      if (light) {
        const TirEnvMap& e = p.env.e[(int)(t / p.S_l / p.n)];
        const double* u = p.u_light + t * 3;
        mis_light_dir(e, rl_bin(e.cdf, e.H * e.W, u[0]), u + 1, w);
      } else {
        PointCtx c;
        const float one[3] = {1.f, 1.f, 1.f};
        rl_point(p.rays + i * 6, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
                 p.fresnel + i * 3, one, c);
        MisPoint m;
        mis_point(c, m);
        mis_brdf_dir(c, m, p.u_brdf + (t - n_light) * 3, w);
      }
      append = rl_cosine(w, p.normal + i * 3) > 1e-6f;
      if (append) rl_surface(p.rays + i * 6, p.depth[i], o);
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, w);
  if (t >= total) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) p.dir[t * 3 + c] = w[c];
  p.pos[t] = slot;
}

struct ShadeParams {
  EnvTable env;
  const float* rays; const float* normal; const float* albedo; const float* rough; int rough_stride;
  const float* fresnel; const float* acc;
  int64_t n; int S_l, S_b; float thr;
  const float* rescale;
  const float* dir; const int32_t* pos; const float* vis; int vis_kind;
  float* with_bg; float* without_bg; float* linear; int64_t out_rows; int64_t row0;
};

__global__ void __launch_bounds__(kWarps * 32) mis_shade_kernel(const __grid_constant__ ShadeParams p, int L) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (w >= (int64_t)L * p.n) return;
  const int l = (int)(w / p.n);
  const int64_t i = w - (int64_t)l * p.n;
  const TirEnvMap& e = p.env.e[l];
  const float* ray = p.rays + i * 6;
  const float a = p.acc[i];
  float wo[3] = {1.f, 1.f, 1.f}, lin[3] = {0.f, 0.f, 0.f};
  if (a > p.thr) {
    PointCtx c;
    const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
    rl_point(ray, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
             p.fresnel + i * 3, resc, c);
    MisPoint m;
    mis_point(c, m);
    float acc[3] = {0.f, 0.f, 0.f};
    const int64_t kl = w * p.S_l, kb = (int64_t)L * p.n * p.S_l + i * p.S_b;
    mis_lane(e, c, m, p.dir + kl * 3, p.pos + kl, p.S_l, p.dir + kb * 3, p.pos + kb, p.S_b, p.vis, p.vis_kind, lane,
             32, acc);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      lin[ch] = warp_sum(acc[ch]);
      wo[ch] = tone(lin[ch], 1);
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
    if (p.linear) p.linear[r + ch] = lin[ch];
  }
}

}  // namespace

extern "C" int tir_relight_mis_sample(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* depth,
                                      const float* normal, const float* albedo, const float* rough,
                                      int32_t rough_stride, const float* fresnel, const float* acc, int64_t n,
                                      int32_t S_l, int32_t S_b, float acc_mask_threshold, const double* u_light,
                                      const double* u_brdf, float* dir, int32_t* pos, float* list_o, float* list_d,
                                      int64_t capacity, int64_t* count, void* stream) {
  const int rc = mis_sample_check(envs, n_lights, rays, depth, normal, albedo, rough, rough_stride, fresnel, acc, n,
                                  S_l, S_b, u_light, u_brdf, dir, pos, list_o, list_d, capacity, count);
  if (rc <= 0) return rc;
  SampleParams p{};
  for (int l = 0; l < n_lights; ++l) p.env.e[l] = envs[l];
  p.rays = rays; p.depth = depth; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.acc = acc; p.n = n; p.S_l = S_l; p.S_b = S_b; p.thr = acc_mask_threshold;
  p.u_light = u_light; p.u_brdf = u_brdf; p.dir = dir; p.pos = pos; p.list_o = list_o; p.list_d = list_d;
  p.capacity = capacity; p.count = reinterpret_cast<unsigned long long*>(count);
  const int64_t total = (int64_t)n_lights * n * S_l + n * S_b;
  mis_sample_kernel<<<(unsigned)((total + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(p, n_lights);
  return (int)cudaGetLastError();
}

extern "C" int tir_relight_mis_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                                     const float* albedo, const float* rough, int32_t rough_stride,
                                     const float* fresnel, const float* acc, int64_t n, int32_t S_l, int32_t S_b,
                                     float acc_mask_threshold, const float* rescale, const float* dir,
                                     const int32_t* pos, const float* vis_list, int32_t vis_kind, float* with_bg,
                                     float* without_bg, float* linear_out, int64_t out_rows, int64_t row0,
                                     void* stream) {
  const int rc = mis_shade_check(envs, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, S_l, S_b,
                                 rescale, dir, pos, vis_list, vis_kind, with_bg, without_bg, out_rows, row0);
  if (rc <= 0) return rc;
  ShadeParams p{};
  for (int l = 0; l < n_lights; ++l) p.env.e[l] = envs[l];
  p.rays = rays; p.normal = normal; p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride;
  p.fresnel = fresnel; p.acc = acc; p.n = n; p.S_l = S_l; p.S_b = S_b; p.thr = acc_mask_threshold;
  p.rescale = rescale; p.dir = dir; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind; p.with_bg = with_bg;
  p.without_bg = without_bg; p.linear = linear_out; p.out_rows = out_rows; p.row0 = row0;
  const int64_t warps = (int64_t)n_lights * n;
  mis_shade_kernel<<<(unsigned)((warps + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p, n_lights);
  return (int)cudaGetLastError();
}
