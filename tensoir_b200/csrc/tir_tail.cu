// Fused end of the primary march: (i) per appearance sample, everything between the heads and the per-ray sums
// (BRDF split, relative-smoothness costs, normal losses, weighting; tensorBase_rotated_lights.py:930-975), (ii) per ray,
// the epilogue of TensorBase.forward (background compositing, clamps, linear->sRGB, normal normalisation, the two scalar
// smoothness means, acc_mask; :977-1036).  Forward and analytic backward; the per-item math lives in tir_tail_body.h /
// tir_epilogue_body.h, which a host build checks against torch autograd (experiments/primary_tail, primary_epilogue).
#include <cuda_runtime.h>

#include "../../include/tensoir_b200.h"
#include "tir_device.cuh"
#include "tir_epilogue_body.h"
#include "tir_tail_body.h"

namespace {

__device__ __forceinline__ TailSample load_sample(int64_t i, const float* __restrict__ w, const int64_t* __restrict__ ray,
                                                  const float* __restrict__ rgb, const float* __restrict__ brdf,
                                                  const float* __restrict__ brdfj, const float* __restrict__ vn,
                                                  const float* __restrict__ dn, const float* __restrict__ viewdirs) {
  TailSample s;
  s.w = w[i];
  const int64_t r = ray[i];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    s.rgb[c] = rgb[i * 3 + c];
    s.vn[c] = vn[i * 3 + c];
    s.dn[c] = dn ? dn[i * 3 + c] : 0.f;
    s.vd[c] = __ldg(viewdirs + r * 3 + c);
  }
  const float4 b = *reinterpret_cast<const float4*>(brdf + i * 4), bj = *reinterpret_cast<const float4*>(brdfj + i * 4);
  s.brdf[0] = b.x; s.brdf[1] = b.y; s.brdf[2] = b.z; s.brdf[3] = b.w;
  s.brdfj[0] = bj.x; s.brdfj[1] = bj.y; s.brdfj[2] = bj.z; s.brdfj[3] = bj.w;
  return s;
}

__global__ void tail_fwd_kernel(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                                const float* brdfj, const float* vn, const float* dn, const float* viewdirs,
                                float* __restrict__ packed) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const TailSample s = load_sample(i, w, ray, rgb, brdf, brdfj, vn, dn, viewdirs);
    if (s.w == 0.f) continue;                      // padding rows of a static-capacity list contribute nothing
    float v[TAIL_CH];
    tail_channels(s, dn != nullptr, v);
    float* dst = packed + ray[i] * TAIL_CH;
#pragma unroll
    for (int k = 0; k < TAIL_CH; ++k) atomicAdd(dst + k, s.w * v[k]);
  }
}

__global__ void tail_bwd_kernel(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                                const float* brdfj, const float* vn, const float* dn, const float* viewdirs,
                                const float* __restrict__ g_packed, float* g_w, float* g_rgb, float* g_brdf,
                                float* g_brdfj, float* g_vn, float* g_dn) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const TailSample s = load_sample(i, w, ray, rgb, brdf, brdfj, vn, dn, viewdirs);
    float G[TAIL_CH];
    const float* src = g_packed + ray[i] * TAIL_CH;
#pragma unroll
    for (int k = 0; k < TAIL_CH; ++k) G[k] = __ldg(src + k);
    TailGrad g;
    tail_backward_sample(s, dn != nullptr, G, g);
    g_w[i] = g.w;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      g_rgb[i * 3 + c] = g.rgb[c];
      g_vn[i * 3 + c] = g.vn[c];
      if (g_dn) g_dn[i * 3 + c] = g.dn[c];
    }
    *reinterpret_cast<float4*>(g_brdf + i * 4) = make_float4(g.brdf[0], g.brdf[1], g.brdf[2], g.brdf[3]);
    *reinterpret_cast<float4*>(g_brdfj + i * 4) = make_float4(g.brdfj[0], g.brdfj[1], g.brdfj[2], g.brdfj[3]);
  }
}

__device__ __forceinline__ EpiIn load_ray(int64_t r, const float* __restrict__ packed, const float* __restrict__ acc,
                                          const float* __restrict__ depth, const float* __restrict__ rays, float fresnel0,
                                          int bg) {
  EpiIn in;
#pragma unroll
  for (int k = 0; k < 14; ++k) in.P[k] = packed[r * 14 + k];
  in.acc = acc[r]; in.depth = depth[r]; in.dz = rays[r * 6 + 5]; in.fresnel0 = fresnel0; in.bg = bg;
  return in;
}

__global__ void epilogue_fwd_kernel(int64_t n, const float* packed, const float* acc, const float* depth,
                                    const float* rays, float fresnel0, int bg, TirRayMaps o,
                                    uint8_t* __restrict__ acc_mask, float* __restrict__ losses) {
  float s_ac = 0.f, s_rc = 0.f;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const EpiIn in = load_ray(r, packed, acc, depth, rays, fresnel0, bg);
    EpiOut e;
    epi_forward(in, e);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      o.rgb[r * 3 + c] = e.rgb[c];
      o.normal[r * 3 + c] = e.normal[c];
      o.albedo[r * 3 + c] = e.albedo[c];
      o.fresnel[r * 3 + c] = e.fresnel[c];
    }
    o.depth[r] = e.depth; o.rough[r] = e.rough; o.nd[r] = e.nd; o.no[r] = e.no;
    acc_mask[r] = in.acc > 0.5f ? 1 : 0;
    s_ac += e.ac; s_rc += e.rc;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s_ac += __shfl_xor_sync(0xffffffffu, s_ac, off);
    s_rc += __shfl_xor_sync(0xffffffffu, s_rc, off);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(losses + 0, s_ac / (float)n);
    atomicAdd(losses + 1, s_rc / (float)n);
  }
}

// every gradient pointer of `g` may be NULL (that output did not take part in the loss)
__global__ void epilogue_bwd_kernel(int64_t n, const float* packed, const float* acc, const float* depth,
                                    const float* rays, float fresnel0, int bg, TirRayMaps g,
                                    const float* __restrict__ g_loss_albedo, const float* __restrict__ g_loss_rough,
                                    float* __restrict__ g_packed, float* __restrict__ g_acc,
                                    float* __restrict__ g_depth) {
  const float g_ac = g_loss_albedo ? g_loss_albedo[0] / (float)n : 0.f;
  const float g_rc = g_loss_rough ? g_loss_rough[0] / (float)n : 0.f;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const EpiIn in = load_ray(r, packed, acc, depth, rays, fresnel0, bg);
    EpiOut e;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      e.rgb[c] = g.rgb ? g.rgb[r * 3 + c] : 0.f;
      e.normal[c] = g.normal ? g.normal[r * 3 + c] : 0.f;
      e.albedo[c] = g.albedo ? g.albedo[r * 3 + c] : 0.f;
      e.fresnel[c] = g.fresnel ? g.fresnel[r * 3 + c] : 0.f;
    }
    e.depth = g.depth ? g.depth[r] : 0.f;
    e.rough = g.rough ? g.rough[r] : 0.f;
    e.nd = g.nd ? g.nd[r] : 0.f;
    e.no = g.no ? g.no[r] : 0.f;
    e.ac = g_ac; e.rc = g_rc;
    float gP[14], ga, gd;
    epi_backward(in, e, gP, &ga, &gd);
#pragma unroll
    for (int k = 0; k < 14; ++k) g_packed[r * 14 + k] = gP[k];
    g_acc[r] = ga;
    g_depth[r] = gd;
  }
}

inline int blocks_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)tir::num_sms() * 8;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace

extern "C" int tir_tail_fwd(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                            const float* brdfj, const float* vn, const float* dn, const float* viewdirs, float* packed,
                            void* stream) {
  if (n <= 0) return TIR_OK;
  if (!w || !ray || !rgb || !brdf || !brdfj || !vn || !viewdirs || !packed) return TIR_ERR_NULL;
  tail_fwd_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(n, w, ray, rgb, brdf, brdfj, vn, dn, viewdirs,
                                                                        packed);
  return (int)cudaGetLastError();
}

extern "C" int tir_tail_bwd(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                            const float* brdfj, const float* vn, const float* dn, const float* viewdirs,
                            const float* g_packed, float* g_w, float* g_rgb, float* g_brdf, float* g_brdfj, float* g_vn,
                            float* g_dn, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!w || !ray || !rgb || !brdf || !brdfj || !vn || !viewdirs || !g_packed || !g_w || !g_rgb || !g_brdf || !g_brdfj ||
      !g_vn)
    return TIR_ERR_NULL;
  tail_bwd_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(n, w, ray, rgb, brdf, brdfj, vn, dn, viewdirs,
                                                                        g_packed, g_w, g_rgb, g_brdf, g_brdfj, g_vn, g_dn);
  return (int)cudaGetLastError();
}

extern "C" int tir_epilogue_fwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                                float fresnel0, int32_t bg, const TirRayMaps* out, uint8_t* acc_mask, float* losses,
                                void* stream) {
  if (n <= 0) return TIR_OK;
  if (!packed || !acc || !depth || !rays || !out || !acc_mask || !losses) return TIR_ERR_NULL;
  if (!out->rgb || !out->depth || !out->normal || !out->albedo || !out->rough || !out->fresnel || !out->nd || !out->no)
    return TIR_ERR_NULL;
  epilogue_fwd_kernel<<<blocks_for(n, 128), 128, 0, (cudaStream_t)stream>>>(n, packed, acc, depth, rays, fresnel0, bg,
                                                                            *out, acc_mask, losses);
  return (int)cudaGetLastError();
}

extern "C" int tir_epilogue_bwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                                float fresnel0, int32_t bg, const TirRayMaps* g_out, const float* g_loss_albedo,
                                const float* g_loss_rough, float* g_packed, float* g_acc, float* g_depth, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!packed || !acc || !depth || !rays || !g_out || !g_packed || !g_acc || !g_depth) return TIR_ERR_NULL;
  epilogue_bwd_kernel<<<blocks_for(n, 128), 128, 0, (cudaStream_t)stream>>>(n, packed, acc, depth, rays, fresnel0, bg,
                                                                            *g_out, g_loss_albedo, g_loss_rough, g_packed,
                                                                            g_acc, g_depth);
  return (int)cudaGetLastError();
}
