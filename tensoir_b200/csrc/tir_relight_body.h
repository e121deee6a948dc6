// Per-sample and per-ray math of the relighting pass (scripts/relight_importance.py:99-181, Environment_Light of
// models/relight_utils.py:150-205).  Shared by the CUDA kernels (tir_relight.cu) and by a host build
// (tests/host_relight.cpp) that the CPU tests drive through the ctypes wrapper and compare with the oracle.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"
#include "tir_eval_body.h"
#include "tir_ggx.h"

#if defined(__CUDACC__)
#define RL_HD __host__ __device__ __forceinline__
#else
#define RL_HD inline
#endif

// torch.searchsorted(cdf, u, right=True).clamp(max=n-1): the first i with cdf[i] > u
RL_HD int rl_bin(const double* cdf, int n, double u) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] <= u) lo = mid + 1;
    else hi = mid;
  }
  return lo < n - 1 ? lo : n - 1;
}

// Environment_Light.get_light (relight_utils.py:193-205): phi = acos(d.z) - 1e-6, theta = atan2(d.y, d.x), grid
// (-theta/pi, 2 phi/pi - 1) into F.grid_sample(bilinear, zeros, align_corners=True) of the [3,H,W] map.
RL_HD void rl_background(const TirEnvMap& e, const float d[3], float out[3]) {
  const float pi = (float)3.14159265358979323846;
  const float phi = ev_sub(acosf(d[2]), 1e-6f);
  const float theta = atan2f(d[1], d[0]);
  const float qy = ev_sub(ev_mul(ev_div(phi, pi), 2.f), 1.f);
  const float qx = ev_div(-theta, pi);
  const float ix = ev_mul(ev_div(ev_add(qx, 1.f), 2.f), (float)(e.W - 1));
  const float iy = ev_mul(ev_div(ev_add(qy, 1.f), 2.f), (float)(e.H - 1));
  const float x0 = floorf(ix), y0 = floorf(iy);
  const int xi = (int)x0, yi = (int)y0;
  const float wx1 = ev_sub(ix, x0), wx0 = ev_sub(ev_add(x0, 1.f), ix);
  const float wy1 = ev_sub(iy, y0), wy0 = ev_sub(ev_add(y0, 1.f), iy);
  const float w[4] = {ev_mul(wx0, wy0), ev_mul(wx1, wy0), ev_mul(wx0, wy1), ev_mul(wx1, wy1)};
  const int tx[4] = {xi, xi + 1, xi, xi + 1}, ty[4] = {yi, yi, yi + 1, yi + 1};
  for (int c = 0; c < 3; ++c) out[c] = 0.f;
  for (int k = 0; k < 4; ++k) {
    if (tx[k] < 0 || tx[k] >= e.W || ty[k] < 0 || ty[k] >= e.H) continue;
    const int64_t t = (int64_t)ty[k] * e.W + tx[k];
    for (int c = 0; c < 3; ++c) out[c] = ev_add(out[c], ev_mul(e.rgb[t * 3 + c], w[k]));
  }
}

// Surface point o + depth * d of a primary ray (relight_importance.py:105), rounded like the eager ops
RL_HD void rl_surface(const float* ray, float depth, float p[3]) {
  for (int c = 0; c < 3; ++c) p[c] = ev_add(ray[c], ev_mul(depth, ray[3 + c]));
}

// cosine of relight_importance.py:125: the sampled direction against the raw (unnormalised) normal
RL_HD float rl_cosine(const float L[3], const float n[3]) {
  return ev_add(ev_add(ev_mul(L[0], n[0]), ev_mul(L[1], n[1])), ev_mul(L[2], n[2]));
}

// Per hit ray: the GGX point context with the rescaled albedo (masked_albedo_chunk * rescale_value, :159)
RL_HD void rl_point(const float* ray, const float* normal, const float* albedo, const float* rough, int rough_stride,
                    const float* fresnel, const float rescale[3], tir::PointCtx& c) {
  for (int d = 0; d < 3; ++d) {
    c.n[d] = normal[d];
    c.V[d] = -ray[3 + d];
    c.a[d] = ev_mul(albedo[d], rescale[d]);
    c.F0[d] = fresnel[d];
    c.r[d] = rough_stride == 1 ? rough[0] : rough[d];
  }
  tir::ggx_point(c);
}

// One sample's contribution (:158-163): (albedo*rescale/pi + GGX) * (vis * rgb) * cosine / pdf, added to acc[3]
RL_HD void rl_contrib(const tir::PointCtx& c, const float L[3], const float rgb[3], float pdf, float vis,
                      float acc[3]) {
  tir::DirCtx d;
  for (int e = 0; e < 3; ++e) d.L[e] = L[e];
  tir::ggx_dir(c, d);
  for (int ch = 0; ch < 3; ++ch) {
    float frac, nom;
    tir::ggx_terms(c, d, ch, frac, nom);
    const float brdf = c.a[ch] / tir::kPi + frac / nom;
    acc[ch] += brdf * (vis * rgb[ch]) * d.cosr / pdf;
  }
}

#if defined(__CUDA_ARCH__)
#define RL_LDG(p) __ldg(p)
#else
#define RL_LDG(p) (*(p))
#endif

// Visibility of list row q as relight() reads it from the march: vis_kind 0 (nerv) t_last, 1 (nerfactor) 1 - acc
RL_HD float rl_vis(const float* vis_list, int vis_kind, int q) {
  return vis_kind ? 1.f - vis_list[q] : vis_list[q];
}

// The direct per-sample loop of one (map, point): lane `lane` of `lanes` adds rl_contrib of samples lane, lane + lanes,
// ... (bin and list row from bin[] / pos[], vis as relight() reads it from the march) to acc[3].  The kernels run it on
// the 32 lanes of a warp and reduce with warp_sum; the host builds run the 32 lanes in turn and reduce with the same
// xor butterfly.
RL_HD void rl_direct_lane(const TirEnvMap& e, const tir::PointCtx& c, const int32_t* bin, const int32_t* pos,
                          const float* vis_list, int vis_kind, int S, int lane, int lanes, float acc[3]) {
  for (int s = lane; s < S; s += lanes) {
    const int b = bin[s];
    const int q = pos[s];
    float vis = 0.f;
    if (q >= 0) vis = rl_vis(vis_list, vis_kind, q);
    float Ld[3], rgb[3];
    for (int ch = 0; ch < 3; ++ch) { Ld[ch] = RL_LDG(e.dir + (int64_t)b * 3 + ch); rgb[ch] = RL_LDG(e.rgb + (int64_t)b * 3 + ch); }
    rl_contrib(c, Ld, rgb, RL_LDG(e.pdf_return + b), vis, acc);
  }
}

// Composite of one output row (:167-181): without_bg (already toned, or white), background, acc threshold 0.9
RL_HD void rl_composite(const TirEnvMap& e, const float* ray, float acc, const float wo[3], float with_bg[3]) {
  float bg[3];
  rl_background(e, ray + 3, bg);
  const float acc_t = acc <= 0.9f ? 0.f : acc;
  for (int c = 0; c < 3; ++c)
    with_bg[c] = ev_add(ev_mul(acc_t, wo[c]), ev_mul(ev_sub(1.f, acc_t), tir::tone(bg[c], 1)));
}

// argument checks shared by the kernels and the host build: 1 run, 0 nothing to do, < 0 TirStatus
inline int rl_validate(const TirEnvMap* envs, int32_t n_lights, int64_t n, int32_t n_samples) {
  if (n_lights < 0 || n < 0 || n_samples < 0) return TIR_ERR_SHAPE;
  if (n_lights > TIR_RELIGHT_MAX_LIGHTS) return TIR_ERR_SHAPE;
  if (n_lights == 0 || n == 0) return 0;
  if (!envs) return TIR_ERR_NULL;
  for (int l = 0; l < n_lights; ++l) {
    if (envs[l].H <= 0 || envs[l].W <= 0) return TIR_ERR_SHAPE;
    if (!envs[l].rgb || !envs[l].dir || !envs[l].pdf_return || !envs[l].cdf) return TIR_ERR_NULL;
  }
  return 1;
}

// argument checks of a visibility list (list_o, list_d: capacity rows of 3), shared by every tir_*_sample entry and
// its host build: TIR_OK or a TirStatus
inline int rl_check_list(int64_t capacity, const float* list_o, const float* list_d) {
  if (capacity < 0 || capacity > INT32_MAX) return TIR_ERR_SHAPE;
  if (capacity > 0 && (!list_o || !list_d)) return TIR_ERR_NULL;
  return TIR_OK;
}

// argument checks of a shade-type entry's window, shared by every shade-type check: the roughness stride, the
// visibility kind and output rows [row0, row0 + n) inside out_rows.  TIR_OK or a TirStatus
inline int rl_check_window(int32_t rough_stride, int32_t vis_kind, int64_t n, int64_t out_rows, int64_t row0) {
  if (rough_stride != 1 && rough_stride != 3) return TIR_ERR_SHAPE;
  if (vis_kind != 0 && vis_kind != 1) return TIR_ERR_CONFIG;
  if (row0 < 0 || row0 + n > out_rows) return TIR_ERR_SHAPE;
  return TIR_OK;
}

// The whole argument check of each entry, run by tir_relight.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus
inline int rl_sample_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* depth,
                           const float* normal, const float* acc, int64_t n, int32_t n_samples, const double* u,
                           const int32_t* bin, const int32_t* pos, const float* list_o, const float* list_d,
                           int64_t capacity, const int64_t* count) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc <= 0 || n_samples == 0) return rc < 0 ? rc : 0;
  if (!rays || !depth || !normal || !acc || !u || !bin || !pos || !count) return TIR_ERR_NULL;
  const int lrc = rl_check_list(capacity, list_o, list_d);
  return lrc ? lrc : 1;
}

inline int rl_shade_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                          const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                          const float* acc, int64_t n, int32_t n_samples, const float* rescale, const int32_t* bin,
                          const int32_t* pos, int32_t vis_kind, const float* with_bg, const float* without_bg,
                          int64_t out_rows, int64_t row0) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc <= 0) return rc;
  if (n_samples <= 0) return TIR_ERR_SHAPE;
  if (!rays || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !bin || !pos || !with_bg ||
      !without_bg)
    return TIR_ERR_NULL;
  const int wrc = rl_check_window(rough_stride, vis_kind, n, out_rows, row0);
  return wrc ? wrc : 1;
}
