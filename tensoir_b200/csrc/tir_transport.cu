// Light transport of one chunk of primary rays to the K texels of an environment map, around the existing density
// march, in the shape of tir_relight.cu:
//
//   1. tir_transport_sample  one thread per (ray, texel): the raw-normal cosine test of the texel's direction and a
//                            warp-aggregated append of (surface point, direction) to the visibility list; pos[] remembers
//                            where each (ray, texel) went;
//   2. tir_march_density     (unchanged) on the list, by the caller, sized by the list length read back once per chunk;
//   3. tir_transport_build   one warp per ray, lanes stride over the texels: GGX + Lambert, visibility, cosine and solid
//                            angle, written channel-major into T[3, n, K], so each channel is one GEMM operand.
//
// The list order depends on warp scheduling, but every (ray, texel) reads its own row back through pos[], so T does not.
#include "tir_device.cuh"
#include "tir_transport_body.h"

using namespace tir;

namespace {

constexpr int kSampleThreads = 256;
constexpr int kWarps = 8;

struct TransportSampleParams {
  const float* dirs; int K;
  const float* rays; const float* depth; const float* normal; const float* acc;
  int64_t n; float thr;
  int32_t* pos;
  float* list_o; float* list_d;
  int64_t capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kSampleThreads) transport_sample_kernel(const __grid_constant__ TransportSampleParams p) {
  const int64_t total = p.n * p.K;
  const int64_t t = (int64_t)blockIdx.x * kSampleThreads + threadIdx.x;
  bool append = false;
  float o[3], L3[3];
  if (t < total) {
    const int64_t i = t / p.K;
    const int k = (int)(t - i * p.K);
    if (p.acc[i] > p.thr) {
      float nrm[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) { L3[c] = __ldg(p.dirs + (int64_t)k * 3 + c); nrm[c] = p.normal[i * 3 + c]; }
      append = rl_cosine(L3, nrm) > 1e-6f;
      if (append) rl_surface(p.rays + i * 6, p.depth[i], o);
    }
  }
  const int32_t slot = list_append(p.list_o, p.list_d, p.capacity, p.count, append, o, L3);
  if (t >= total) return;
  p.pos[t] = slot;
}

struct TransportBuildParams {
  const float* dirs; const float* domega; int K;
  const float* rays; const float* normal; const float* albedo; const float* rough; int rough_stride;
  const float* fresnel; const float* acc;
  int64_t n; float thr;
  const float* rescale;
  const int32_t* pos; const float* vis; int vis_kind;
  float* T;
};

__global__ void __launch_bounds__(kWarps * 32) transport_build_kernel(const __grid_constant__ TransportBuildParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (i >= p.n) return;
  const int64_t plane = p.n * p.K;
  float* row = p.T + i * p.K;
  if (!(p.acc[i] > p.thr)) {
    for (int k = lane; k < p.K; k += 32) row[k] = row[plane + k] = row[2 * plane + k] = 0.f;
    return;
  }
  PointCtx c;
  const float resc[3] = {p.rescale[0], p.rescale[1], p.rescale[2]};
  rl_point(p.rays + i * 6, p.normal + i * 3, p.albedo + i * 3, p.rough + i * p.rough_stride, p.rough_stride,
           p.fresnel + i * 3, resc, c);
  const int32_t* pos = p.pos + i * p.K;
  for (int k = lane; k < p.K; k += 32) {
    const int q = pos[k];
    float t[3] = {0.f, 0.f, 0.f};
    if (q >= 0) {
      const float vis = rl_vis(p.vis, p.vis_kind, q);
      const float L[3] = {__ldg(p.dirs + (int64_t)k * 3), __ldg(p.dirs + (int64_t)k * 3 + 1),
                          __ldg(p.dirs + (int64_t)k * 3 + 2)};
      tt_contrib(c, L, __ldg(p.domega + k), vis, t);
    }
    row[k] = t[0];
    row[plane + k] = t[1];
    row[2 * plane + k] = t[2];
  }
}

}  // namespace

extern "C" int tir_transport_sample(const float* dirs, int32_t K, const float* rays, const float* depth,
                                    const float* normal, const float* acc, int64_t n, float acc_mask_threshold,
                                    int32_t* pos, float* list_o, float* list_d, int64_t capacity, int64_t* count,
                                    void* stream) {
  const int rc = tt_sample_check(dirs, K, rays, depth, normal, acc, n, pos, list_o, list_d, capacity, count);
  if (rc <= 0) return rc;
  TransportSampleParams p{};
  p.dirs = dirs; p.K = K; p.rays = rays; p.depth = depth; p.normal = normal; p.acc = acc; p.n = n;
  p.thr = acc_mask_threshold; p.pos = pos; p.list_o = list_o; p.list_d = list_d; p.capacity = capacity;
  p.count = reinterpret_cast<unsigned long long*>(count);
  const int64_t total = n * K;
  transport_sample_kernel<<<(unsigned)((total + kSampleThreads - 1) / kSampleThreads), kSampleThreads, 0,
                            (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_transport_build(const float* dirs, const float* domega, int32_t K, const float* rays,
                                   const float* normal, const float* albedo, const float* rough, int32_t rough_stride,
                                   const float* fresnel, const float* acc, int64_t n, float acc_mask_threshold,
                                   const float* rescale, const int32_t* pos, const float* vis_list, int32_t vis_kind,
                                   float* T, void* stream) {
  const int rc = tt_build_check(dirs, domega, K, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, rescale,
                                pos, vis_list, vis_kind, T);
  if (rc <= 0) return rc;
  TransportBuildParams p{};
  p.dirs = dirs; p.domega = domega; p.K = K; p.rays = rays; p.normal = normal; p.albedo = albedo; p.rough = rough;
  p.rough_stride = rough_stride; p.fresnel = fresnel; p.acc = acc; p.n = n; p.thr = acc_mask_threshold;
  p.rescale = rescale; p.pos = pos; p.vis = vis_list; p.vis_kind = vis_kind; p.T = T;
  transport_build_kernel<<<(unsigned)((n + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}
