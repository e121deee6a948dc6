// Per-ray epilogue of TensorBase.forward (tensorBase_rotated_lights.py:977-1036): background compositing, clamps,
// linear -> sRGB (relight_utils.py:489-515), safe_l2_normalize of the normal map — forward and analytic backward for ONE
// ray.  Input is the 14-channel per-ray sum produced by the fused tail (experiments/primary_tail) plus acc / depth from
// the compositing kernel.  Shared by the CUDA kernels and a host build checked against torch autograd on the CPU.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"

#if defined(__CUDACC__)
#define EPI_HD __host__ __device__ __forceinline__
#else
#define EPI_HD inline
#endif

struct EpiIn {
  float P[14];     // [rgb 3 | normal 3 | albedo 3 | rough | albedo cost | rough cost | normals_diff | orientation]
  float acc, depth;
  float dz;        // rays[..., -1] (z of the ray direction), the reference's background "depth" term
  float fresnel0;  // fixed_fresnel
  int bg;          // white_bg or the train-time coin
};

struct EpiOut {
  float rgb[3], depth, normal[3], albedo[3], rough, fresnel[3], nd, no, ac, rc;
};

EPI_HD float epi_clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }
EPI_HD float epi_gate01(float x) { return (x >= 0.f && x <= 1.f) ? 1.f : 0.f; }   // ATen clamp backward mask

EPI_HD float epi_srgb(float t) {
  return t <= 0.0031308f ? t * 12.92f : 1.055f * powf(t + 1e-6f, 1.f / 2.4f) - 0.055f;
}
EPI_HD float epi_dsrgb(float t) {
  return t <= 0.0031308f ? 12.92f : (1.055f / 2.4f) * powf(t + 1e-6f, 1.f / 2.4f - 1.f);
}

EPI_HD void epi_forward(const EpiIn& in, EpiOut& o) {
  const float om = in.bg ? 1.f - in.acc : 0.f;
  for (int c = 0; c < 3; ++c) {
    o.rgb[c] = epi_srgb(epi_clamp01(in.P[c] + om));
    o.albedo[c] = epi_clamp01(in.P[6 + c] + om);
    o.fresnel[c] = epi_clamp01(in.fresnel0 + om);
  }
  o.depth = in.depth + om * in.dz;
  const float n0 = in.P[3], n1 = in.P[4], n2 = in.P[5] + om;       // background normal (0, 0, 1)
  const float norm = sqrtf(n0 * n0 + n1 * n1 + n2 * n2);
  const float den = fmaxf(norm, 1e-6f);
  o.normal[0] = n0 / den; o.normal[1] = n1 / den; o.normal[2] = n2 / den;
  o.rough = epi_clamp01(in.P[9] + om);
  o.ac = in.P[10]; o.rc = in.P[11]; o.nd = in.P[12]; o.no = in.P[13];
}

// g: gradient w.r.t. every field of EpiOut (ac / rc already divided by n_rays by the caller: they feed torch.mean).
// -> gP[14], g_acc, g_depth
EPI_HD void epi_backward(const EpiIn& in, const EpiOut& g, float gP[14], float* g_acc, float* g_depth) {
  const float om = in.bg ? 1.f - in.acc : 0.f;
  float g_om = 0.f;
  for (int c = 0; c < 3; ++c) {
    const float x = in.P[c] + om;
    // clamp (forward_relight) -> clamp (linear2srgb, identity on [0,1]) -> piecewise curve
    const float t = epi_clamp01(x);
    const float gx = g.rgb[c] * epi_dsrgb(t) * epi_gate01(x);
    gP[c] = gx;
    g_om += gx;
    const float xa = in.P[6 + c] + om;
    gP[6 + c] = g.albedo[c] * epi_gate01(xa);
    g_om += gP[6 + c];
    g_om += g.fresnel[c] * epi_gate01(in.fresnel0 + om);
  }
  *g_depth = g.depth;
  g_om += g.depth * in.dz;
  const float n[3] = {in.P[3], in.P[4], in.P[5] + om};
  const float norm = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  float gn[3];
  if (norm >= 1e-6f) {      // clamp_min passes the gradient to the norm
    const float y[3] = {n[0] / norm, n[1] / norm, n[2] / norm};
    const float dot = y[0] * g.normal[0] + y[1] * g.normal[1] + y[2] * g.normal[2];
    for (int c = 0; c < 3; ++c) gn[c] = (g.normal[c] - y[c] * dot) / norm;
  } else {
    for (int c = 0; c < 3; ++c) gn[c] = g.normal[c] / 1e-6f;
  }
  gP[3] = gn[0]; gP[4] = gn[1]; gP[5] = gn[2];
  g_om += gn[2];
  const float xr = in.P[9] + om;
  gP[9] = g.rough * epi_gate01(xr);
  g_om += gP[9];
  gP[10] = g.ac; gP[11] = g.rc; gP[12] = g.nd; gP[13] = g.no;
  *g_acc = in.bg ? -g_om : 0.f;
}

// The whole argument check of each entry, run by tir_tail.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus.  The maps of g_out and the loss gradients are optional.
inline int epi_fwd_check(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                         const TirRayMaps* out, const uint8_t* acc_mask, const float* losses) {
  if (n <= 0) return 0;
  if (!packed || !acc || !depth || !rays || !out || !acc_mask || !losses) return TIR_ERR_NULL;
  if (!out->rgb || !out->depth || !out->normal || !out->albedo || !out->rough || !out->fresnel || !out->nd || !out->no)
    return TIR_ERR_NULL;
  return 1;
}

inline int epi_bwd_check(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                         const TirRayMaps* g_out, const float* g_packed, const float* g_acc, const float* g_depth) {
  if (n <= 0) return 0;
  if (!packed || !acc || !depth || !rays || !g_out || !g_packed || !g_acc || !g_depth) return TIR_ERR_NULL;
  return 1;
}
