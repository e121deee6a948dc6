// Per (surface point, incident direction) terms of GGX_specular (models/relight_utils.py:17-50) and linear2srgb_torch
// (:489-515), shared by the training shade kernels (tir_shade.cu), the relighting kernel (tir_relight.cu) and the host
// build of the latter (tests/host_relight.cpp).  The callers load the inputs; everything here is pure arithmetic.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define GGX_HD __host__ __device__ __forceinline__
#define GGX_UNROLL _Pragma("unroll")
#else
#define GGX_HD inline
#define GGX_UNROLL
#endif

namespace tir {

constexpr float kPi = 3.14159265358979323846f;

GGX_HD float clamp01e6(float x) { return fminf(fmaxf(x, 1e-6f), 1.f); }
GGX_HD bool in_clamp(float x) { return (x >= 1e-6f) & (x <= 1.f); }

// linear2srgb_torch after the [0,1] clip (relight_utils.py:489-515)
GGX_HD float tone(float x, int srgb) {
  const float t = fminf(fmaxf(x, 0.f), 1.f);
  if (!srgb) return t;
  return t <= 0.0031308f ? t * 12.92f : 1.055f * powf(t + 1e-6f, 1.f / 2.4f) - 0.055f;
}

// Per surface point: n (normal as stored), V (view direction, normalised here), a (albedo), F0 (fresnel), r (roughness)
// are filled by the caller; ggx_point derives the rest.
struct PointCtx {
  float n[3], Np[3], V[3], inv_nn, sgn, NoV, NoV_raw;
  float a[3], F0[3], r[3], alpha2[3], k[3], nom1[3];
};

GGX_HD void ggx_point(PointCtx& c) {
  float nn = 0.f, vn = 0.f;
  GGX_UNROLL
  for (int d = 0; d < 3; ++d) { nn += c.n[d] * c.n[d]; vn += c.V[d] * c.V[d]; }
  c.inv_nn = 1.f / fmaxf(sqrtf(nn), 1e-12f);
  const float inv_vn = 1.f / fmaxf(sqrtf(vn), 1e-12f);
  float nov = 0.f;
  GGX_UNROLL
  for (int d = 0; d < 3; ++d) { c.V[d] *= inv_vn; nov += c.V[d] * c.n[d] * c.inv_nn; }
  c.sgn = (nov > 0.f) ? 1.f : ((nov < 0.f) ? -1.f : 0.f);
  float nov2 = 0.f;
  GGX_UNROLL
  for (int d = 0; d < 3; ++d) { c.Np[d] = c.n[d] * c.inv_nn * c.sgn; nov2 += c.Np[d] * c.V[d]; }
  c.NoV_raw = nov2;
  c.NoV = clamp01e6(nov2);
  GGX_UNROLL
  for (int ch = 0; ch < 3; ++ch) {
    const float al = c.r[ch] * c.r[ch];
    c.alpha2[ch] = al * al;
    c.k[ch] = (al + 2.f * c.r[ch] + 1.f) / 8.f;
    c.nom1[ch] = c.NoV * (1.f - c.k[ch]) + c.k[ch];
  }
}

// Per incident direction, given by value in d.L (as stored, not necessarily unit): cosr = L . n with the raw vectors
// (the reference's cosine), then L and the half vector are normalised for the specular terms.
struct DirCtx {
  float L[3], H[3], cosr, cosv, NoL_raw, NoH_raw, VoH_raw, NoL, NoH, VoH, p2;
};

GGX_HD void ggx_dir(const PointCtx& c, DirCtx& d) {
  float ln = 0.f;
  GGX_UNROLL
  for (int e = 0; e < 3; ++e) ln += d.L[e] * d.L[e];
  d.cosr = d.L[0] * c.n[0] + d.L[1] * c.n[1] + d.L[2] * c.n[2];
  d.cosv = fmaxf(d.cosr, 0.f);
  const float inv_ln = 1.f / fmaxf(sqrtf(ln), 1e-12f);
  float hn = 0.f;
  GGX_UNROLL
  for (int e = 0; e < 3; ++e) { d.L[e] *= inv_ln; d.H[e] = (d.L[e] + c.V[e]) * 0.5f; hn += d.H[e] * d.H[e]; }
  const float inv_hn = 1.f / fmaxf(sqrtf(hn), 1e-12f);
  d.NoL_raw = d.NoH_raw = d.VoH_raw = 0.f;
  GGX_UNROLL
  for (int e = 0; e < 3; ++e) {
    d.H[e] *= inv_hn;
    d.NoL_raw += c.Np[e] * d.L[e]; d.NoH_raw += c.Np[e] * d.H[e]; d.VoH_raw += c.V[e] * d.H[e];
  }
  d.NoL = clamp01e6(d.NoL_raw); d.NoH = clamp01e6(d.NoH_raw); d.VoH = clamp01e6(d.VoH_raw);
  d.p2 = exp2f((-5.55473f * d.VoH - 6.98316f) * d.VoH);
}

// GGX_specular of channel ch is frac / nom with nom = clamp(4 pi nom0^2 nom1 nom2, 1e-6, 4 pi)
GGX_HD void ggx_terms(const PointCtx& c, const DirCtx& d, int ch, float& frac, float& nom) {
  frac = (c.F0[ch] + (1.f - c.F0[ch]) * d.p2) * c.alpha2[ch];
  const float nom0 = d.NoH * d.NoH * (c.alpha2[ch] - 1.f) + 1.f;
  const float nom2 = d.NoL * (1.f - c.k[ch]) + c.k[ch];
  nom = fminf(fmaxf(4.f * kPi * nom0 * nom0 * c.nom1[ch] * nom2, 1e-6f), 4.f * kPi);
}

}  // namespace tir
