// Shading epilogue of render_with_BRDF (models/relight_utils.py:452-475): GGX specular (:17-50) + Lambert, times
// (visibility * direct SG light + indirect), cosine and solid-angle weight, summed over the incident directions.
// Forward and analytic backward (w.r.t. normal, albedo, roughness, fresnel and the direct light table) in one kernel
// each: one warp per surface point, lanes stride over the directions.  Replaces ~60 forward + ~120 backward
// element-wise / reduction launches on [bs, n_dirs, 3] tensors.
#include "tir_device.cuh"
#include "tir_ggx.h"

using namespace tir;

namespace {

constexpr int kWarps = 8;

struct ShadeParams {
  const float* normal;    // [bs,3]
  const float* albedo;    // [bs,3]
  const float* rough;     // [bs,3]
  const float* fresnel;   // [bs,3]
  const float* view;      // [bs,3]  surf2c (unit)
  const int32_t* light;   // [bs]
  const float* dirs;      // [nl,3]
  const float* weight;    // [nl]
  const float* direct;    // [n_lights, nl, 3]
  const float* vis;       // [bs,nl]
  const float* ind;       // [bs,nl,3]
  int64_t bs;
  int nl;
  int n_lights;
  float* rgb;             // [bs,3] forward output (linear, before clamp / sRGB)
  // backward
  const float* g_rgb;     // [bs,3]
  float* g_normal;
  float* g_albedo;
  float* g_rough;
  float* g_fresnel;
  float* g_direct;        // [n_lights, nl, 3] accumulated with atomics
  // "hits" form (tir_shade_hits_*): every ray of the batch is a row, non-hit rays (mask == 0) shade to white
  const uint8_t* mask;    // [bs] acc_mask, or NULL (every row is a surface point)
  const float* rays;      // [bs,6] origin | direction: view = -direction (p.view is NULL then)
  int rough_stride;       // 3: rough is [bs,3];  1: roughness_map [bs,1] broadcast over the channels
  int srgb;               // hits form: clamp to [0,1] (+ linear -> sRGB when 1) folded into the kernel
  float* lin;             // [bs,3] linear value before clamp / sRGB (saved by the forward, read by the backward)
};

__device__ __forceinline__ float tone_grad(float x, int srgb) {
  if (!(x >= 0.f && x <= 1.f)) return 0.f;          // torch.clamp passes the gradient on [min, max]
  if (!srgb) return 1.f;
  return x <= 0.0031308f ? 12.92f : 1.055f / 2.4f * powf(x + 1e-6f, 1.f / 2.4f - 1.f);
}

// PointCtx / DirCtx and their arithmetic live in tir_ggx.h (shared with the relighting kernel); these load the inputs
__device__ __forceinline__ void load_point(const ShadeParams& p, int64_t i, PointCtx& c) {
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    c.n[d] = p.normal[i * 3 + d]; c.V[d] = p.rays ? -p.rays[i * 6 + 3 + d] : p.view[i * 3 + d];
    c.a[d] = p.albedo[i * 3 + d]; c.F0[d] = p.fresnel[i * 3 + d];
    c.r[d] = p.rough_stride == 1 ? p.rough[i] : p.rough[i * 3 + d];
  }
  ggx_point(c);
}

__device__ __forceinline__ void load_dir(const ShadeParams& p, const PointCtx& c, int l, DirCtx& d) {
#pragma unroll
  for (int e = 0; e < 3; ++e) d.L[e] = __ldg(p.dirs + l * 3 + e);
  ggx_dir(c, d);
}

__global__ void __launch_bounds__(kWarps * 32) shade_fwd_kernel(const ShadeParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (i >= p.bs) return;
  if (p.mask && !p.mask[i]) {          // rgb_with_brdf = ones; rgb_with_brdf[acc_mask] = ... (renderer.py:105-106)
    if (lane < 3) { p.rgb[i * 3 + lane] = 1.f; if (p.lin) p.lin[i * 3 + lane] = 2.f; }
    return;
  }
  PointCtx c;
  load_point(p, i, c);
  const float* D = p.direct + (size_t)__ldg(p.light + i) * p.nl * 3;
  float acc[3] = {0.f, 0.f, 0.f};
  for (int l = lane; l < p.nl; l += 32) {
    DirCtx d;
    load_dir(p, c, l, d);
    const float v = p.vis[i * p.nl + l];
    const float cw = d.cosv * __ldg(p.weight + l);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      float frac, nom;
      ggx_terms(c, d, ch, frac, nom);
      const float brdf = c.a[ch] / kPi + frac / nom;
      const float light = v * __ldg(D + l * 3 + ch) + p.ind[(i * p.nl + l) * 3 + ch];
      acc[ch] += brdf * light * cw;
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float s = warp_sum(acc[ch]);
    if (lane == 0) {
      if (p.lin) { p.lin[i * 3 + ch] = s; p.rgb[i * 3 + ch] = tone(s, p.srgb); }
      else p.rgb[i * 3 + ch] = s;
    }
  }
}

__global__ void __launch_bounds__(kWarps * 32) shade_bwd_kernel(const ShadeParams p) {
  extern __shared__ float s_gd[];            // [n_lights][nl][3] per-CTA accumulator of the direct-light gradient
  const int table = p.n_lights * p.nl * 3;
  for (int t = threadIdx.x; t < table; t += blockDim.x) s_gd[t] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  for (int64_t i = (int64_t)blockIdx.x * kWarps + warp; i < p.bs; i += (int64_t)gridDim.x * kWarps) {
    if (p.mask && !p.mask[i]) {        // a non-hit ray shades to the constant 1: no gradient
      if (lane < 3) {
        p.g_normal[i * 3 + lane] = 0.f; p.g_albedo[i * 3 + lane] = 0.f; p.g_fresnel[i * 3 + lane] = 0.f;
        if (p.rough_stride == 3) p.g_rough[i * 3 + lane] = 0.f;
      }
      if (lane == 0 && p.rough_stride == 1) p.g_rough[i] = 0.f;
      continue;
    }
    PointCtx c;
    load_point(p, i, c);
    const int li = __ldg(p.light + i);
    const float* D = p.direct + (size_t)li * p.nl * 3;
    float go[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
      go[ch] = p.g_rgb[i * 3 + ch] * (p.lin ? tone_grad(p.lin[i * 3 + ch], p.srgb) : 1.f);
    float gNp[3] = {0.f, 0.f, 0.f}, gn[3] = {0.f, 0.f, 0.f}, ga[3] = {0.f, 0.f, 0.f}, gF0[3] = {0.f, 0.f, 0.f},
          gal2[3] = {0.f, 0.f, 0.f}, gk[3] = {0.f, 0.f, 0.f};
    float gNoV = 0.f;
    for (int l = lane; l < p.nl; l += 32) {
      DirCtx d;
      load_dir(p, c, l, d);
      const float v = p.vis[i * p.nl + l];
      const float w = __ldg(p.weight + l);
      float g_cos = 0.f, g_NoL = 0.f, g_NoH = 0.f;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float frac0 = c.F0[ch] + (1.f - c.F0[ch]) * d.p2;
        const float frac = frac0 * c.alpha2[ch];
        const float nom0 = d.NoH * d.NoH * (c.alpha2[ch] - 1.f) + 1.f;
        const float nom2 = d.NoL * (1.f - c.k[ch]) + c.k[ch];
        const float nomr = 4.f * kPi * nom0 * nom0 * c.nom1[ch] * nom2;
        const float nom = fminf(fmaxf(nomr, 1e-6f), 4.f * kPi);
        const float spec = frac / nom;
        const float brdf = c.a[ch] / kPi + spec;
        const float dl = __ldg(D + l * 3 + ch);
        const float light = v * dl + p.ind[(i * p.nl + l) * 3 + ch];
        const float gc = go[ch] * w;
        const float g_brdf = gc * light * d.cosv;
        g_cos += gc * brdf * light;
        atomicAdd(&s_gd[(li * p.nl + l) * 3 + ch], gc * brdf * d.cosv * v);
        ga[ch] += g_brdf / kPi;
        const float g_frac = g_brdf / nom;
        const float g_nom = ((nomr >= 1e-6f) & (nomr <= 4.f * kPi)) ? -g_brdf * spec / nom : 0.f;
        const float base = g_nom * 4.f * kPi;
        const float g_nom0 = base * 2.f * nom0 * c.nom1[ch] * nom2;
        const float g_nom1 = base * nom0 * nom0 * nom2;
        const float g_nom2 = base * nom0 * nom0 * c.nom1[ch];
        gal2[ch] += g_frac * frac0 + g_nom0 * d.NoH * d.NoH;
        gF0[ch] += g_frac * c.alpha2[ch] * (1.f - d.p2);
        g_NoH += g_nom0 * 2.f * d.NoH * (c.alpha2[ch] - 1.f);
        g_NoL += g_nom2 * (1.f - c.k[ch]);
        gk[ch] += g_nom2 * (1.f - d.NoL) + g_nom1 * (1.f - c.NoV);
        gNoV += g_nom1 * (1.f - c.k[ch]);
      }
      // H and VoH depend only on the (gradient-free) light and view directions; N' enters through NoL and NoH
      if (!in_clamp(d.NoL_raw)) g_NoL = 0.f;
      if (!in_clamp(d.NoH_raw)) g_NoH = 0.f;
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        gNp[e] += g_NoL * d.L[e] + g_NoH * d.H[e];
        // cosine = clamp(L_raw . n, min=0): direction as stored (cosr used the un-normalised vector)
        if (d.cosr > 0.f) gn[e] += g_cos * __ldg(p.dirs + l * 3 + e);
      }
    }
    if (!in_clamp(c.NoV_raw)) gNoV = 0.f;
    float red[19];
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      red[e] = gNp[e]; red[3 + e] = gn[e]; red[6 + e] = ga[e]; red[9 + e] = gF0[e]; red[12 + e] = gal2[e];
      red[15 + e] = gk[e];
    }
    red[18] = gNoV;
#pragma unroll
    for (int t = 0; t < 19; ++t) red[t] = warp_sum(red[t]);
    if (lane == 0) {
      float gNpt[3], gNn[3], dot = 0.f;
#pragma unroll
      for (int e = 0; e < 3; ++e) { gNpt[e] = red[e] + red[18] * c.V[e]; gNn[e] = gNpt[e] * c.sgn; }
      float Nn[3];
#pragma unroll
      for (int e = 0; e < 3; ++e) { Nn[e] = c.n[e] * c.inv_nn; dot += Nn[e] * gNn[e]; }
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        p.g_normal[i * 3 + e] = red[3 + e] + (gNn[e] - Nn[e] * dot) * c.inv_nn;
        p.g_albedo[i * 3 + e] = red[6 + e];
        p.g_fresnel[i * 3 + e] = red[9 + e];
      }
      float gr[3];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const float r = c.r[e];
        gr[e] = red[12 + e] * 4.f * r * r * r + red[15 + e] * (2.f * r + 2.f) / 8.f;
      }
      if (p.rough_stride == 1) p.g_rough[i] = gr[0] + gr[1] + gr[2];       // backward of .repeat(1, 3)
      else { p.g_rough[i * 3] = gr[0]; p.g_rough[i * 3 + 1] = gr[1]; p.g_rough[i * 3 + 2] = gr[2]; }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < table; t += blockDim.x)
    if (s_gd[t] != 0.f) atomicAdd(p.g_direct + t, s_gd[t]);
}

}  // namespace

extern "C" int tir_shade_fwd(const float* normal, const float* albedo, const float* rough, const float* fresnel,
                             const float* view, const int32_t* light_idx, int64_t bs, const float* dirs,
                             const float* weight, int32_t n_dirs, const float* direct, int32_t n_lights,
                             const float* vis, const float* indirect, float* rgb, void* stream) {
  if (bs <= 0) return TIR_OK;
  if (!normal || !albedo || !rough || !fresnel || !view || !light_idx || !dirs || !weight || !direct || !vis ||
      !indirect || !rgb)
    return TIR_ERR_NULL;
  ShadeParams p{};
  p.normal = normal; p.albedo = albedo; p.rough = rough; p.fresnel = fresnel; p.view = view; p.light = light_idx;
  p.dirs = dirs; p.weight = weight; p.direct = direct; p.vis = vis; p.ind = indirect; p.bs = bs; p.nl = n_dirs;
  p.n_lights = n_lights; p.rgb = rgb; p.rough_stride = 3;
  shade_fwd_kernel<<<(unsigned)((bs + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_shade_bwd(const float* normal, const float* albedo, const float* rough, const float* fresnel,
                             const float* view, const int32_t* light_idx, int64_t bs, const float* dirs,
                             const float* weight, int32_t n_dirs, const float* direct, int32_t n_lights,
                             const float* vis, const float* indirect, const float* g_rgb, float* g_normal,
                             float* g_albedo, float* g_rough, float* g_fresnel, float* g_direct, void* stream) {
  if (bs <= 0) return TIR_OK;
  if (!normal || !albedo || !rough || !fresnel || !view || !light_idx || !dirs || !weight || !direct || !vis ||
      !indirect || !g_rgb || !g_normal || !g_albedo || !g_rough || !g_fresnel || !g_direct)
    return TIR_ERR_NULL;
  const size_t smem = (size_t)n_lights * n_dirs * 3 * sizeof(float);
  if (smem > 200 * 1024) return TIR_ERR_SHAPE;
  ShadeParams p{};
  p.normal = normal; p.albedo = albedo; p.rough = rough; p.fresnel = fresnel; p.view = view; p.light = light_idx;
  p.dirs = dirs; p.weight = weight; p.direct = direct; p.vis = vis; p.ind = indirect; p.bs = bs; p.nl = n_dirs;
  p.n_lights = n_lights; p.g_rgb = g_rgb; p.g_normal = g_normal; p.g_albedo = g_albedo; p.g_rough = g_rough;
  p.g_fresnel = g_fresnel; p.g_direct = g_direct; p.rough_stride = 3;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(shade_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  int64_t blocks = (bs + kWarps - 1) / kWarps;
  if (blocks > 2 * num_sms()) blocks = 2 * num_sms();
  shade_bwd_kernel<<<(unsigned)blocks, kWarps * 32, smem, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

// ---- "hits" form: the whole ray batch, masked by acc_mask (no compaction of the surface hits at all) -------------------
namespace {
__global__ void hits_prepare_kernel(const float* __restrict__ rays, const float* __restrict__ depth,
                                    const float* __restrict__ normal, const uint8_t* __restrict__ mask, int64_t n,
                                    float* __restrict__ surf, float* __restrict__ nrm) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 3) return;
  const int64_t i = t / 3;
  const int c = (int)(t - i * 3);
  // surface_xyz = rays_o + depth * rays_d (relight_utils.py:412); a zero normal fails the secondary march's cosine
  // test for every direction, which is how non-hit rays are skipped without building a list of hits
  surf[t] = rays[i * 6 + c] + depth[i] * rays[i * 6 + 3 + c];
  nrm[t] = mask[i] ? normal[t] : 0.f;
}
}  // namespace

extern "C" int tir_hits_prepare(const float* rays, const float* depth, const float* normal, const uint8_t* mask,
                                int64_t n, float* surf_xyz, float* normal_masked, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!rays || !depth || !normal || !mask || !surf_xyz || !normal_masked) return TIR_ERR_NULL;
  hits_prepare_kernel<<<(unsigned)((n * 3 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rays, depth, normal, mask, n,
                                                                                         surf_xyz, normal_masked);
  return (int)cudaGetLastError();
}

extern "C" int tir_shade_hits_fwd(const float* rays, const uint8_t* mask, const float* normal, const float* albedo,
                                  const float* rough1, const float* fresnel, const int32_t* light_idx, int64_t n,
                                  const float* dirs, const float* weight, int32_t n_dirs, const float* direct,
                                  int32_t n_lights, const float* vis, const float* indirect, int32_t srgb, float* rgb,
                                  float* lin, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!rays || !mask || !normal || !albedo || !rough1 || !fresnel || !light_idx || !dirs || !weight || !direct || !vis ||
      !indirect || !rgb || !lin)
    return TIR_ERR_NULL;
  ShadeParams p{};
  p.normal = normal; p.albedo = albedo; p.rough = rough1; p.fresnel = fresnel; p.rays = rays; p.light = light_idx;
  p.dirs = dirs; p.weight = weight; p.direct = direct; p.vis = vis; p.ind = indirect; p.bs = n; p.nl = n_dirs;
  p.n_lights = n_lights; p.rgb = rgb; p.lin = lin; p.mask = mask; p.rough_stride = 1; p.srgb = srgb;
  shade_fwd_kernel<<<(unsigned)((n + kWarps - 1) / kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int tir_shade_hits_bwd(const float* rays, const uint8_t* mask, const float* normal, const float* albedo,
                                  const float* rough1, const float* fresnel, const int32_t* light_idx, int64_t n,
                                  const float* dirs, const float* weight, int32_t n_dirs, const float* direct,
                                  int32_t n_lights, const float* vis, const float* indirect, int32_t srgb,
                                  const float* lin, const float* g_rgb, float* g_normal, float* g_albedo,
                                  float* g_rough1, float* g_fresnel, float* g_direct, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!rays || !mask || !normal || !albedo || !rough1 || !fresnel || !light_idx || !dirs || !weight || !direct || !vis ||
      !indirect || !lin || !g_rgb || !g_normal || !g_albedo || !g_rough1 || !g_fresnel || !g_direct)
    return TIR_ERR_NULL;
  const size_t smem = (size_t)n_lights * n_dirs * 3 * sizeof(float);
  if (smem > 200 * 1024) return TIR_ERR_SHAPE;
  ShadeParams p{};
  p.normal = normal; p.albedo = albedo; p.rough = rough1; p.fresnel = fresnel; p.rays = rays; p.light = light_idx;
  p.dirs = dirs; p.weight = weight; p.direct = direct; p.vis = vis; p.ind = indirect; p.bs = n; p.nl = n_dirs;
  p.n_lights = n_lights; p.g_rgb = g_rgb; p.g_normal = g_normal; p.g_albedo = g_albedo; p.g_rough = g_rough1;
  p.g_fresnel = g_fresnel; p.g_direct = g_direct; p.lin = const_cast<float*>(lin); p.mask = mask; p.rough_stride = 1;
  p.srgb = srgb;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(shade_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  int64_t blocks = (n + kWarps - 1) / kWarps;
  if (blocks > 2 * num_sms()) blocks = 2 * num_sms();
  shade_bwd_kernel<<<(unsigned)blocks, kWarps * 32, smem, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}
