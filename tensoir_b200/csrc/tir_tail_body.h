// Per-sample math of the fused "primary tail": everything between the appearance heads and the per-ray maps of
// TensorBase.forward (tensorBase_rotated_lights.py:930-975) for one appearance sample, forward and backward.
// Shared by the CUDA kernels (tir_tail.cu, tir_primary.cu) and by a host build (tests/host_tail.cpp) that the CPU test
// checks against torch autograd of the expressions in tensoir_b200/primary.py — the math is validated without a GPU.
//
// Channels of the per-ray sums: [rgb 3 | normal 3 | albedo 3 | roughness 1 | albedo cost 1 | roughness cost 1 |
// normals_diff 1 | orientation 1] = 14, each weighted by the sample's compositing weight.
#pragma once
#include <math.h>
#include "../../include/tensoir_b200.h"

#if defined(__CUDACC__)
#define TAIL_HD __host__ __device__ __forceinline__
#else
#define TAIL_HD inline
#endif

#define TAIL_CH 14

struct TailSample {
  float w;          // compositing weight (0 on padding rows)
  float rgb[3];     // radiance head
  float brdf[4];    // BRDF head at x:        albedo rgb, raw roughness
  float brdfj[4];   // BRDF head at x + noise
  float vn[3];      // normal used for shading (predicted, or derived when there is no predicted head)
  float dn[3];      // derived normal (only read when both_normals)
  float vd[3];      // view direction of the sample's ray
};

struct TailGrad {
  float w, rgb[3], brdf[4], brdfj[4], vn[3], dn[3];
};

// relative smoothness term q^2, q = (a - b) / max(max(a, b), 1e-6)   (tensorBase_rotated_lights.py:858-863)
TAIL_HD float tail_rel_cost(float a, float b) {
  const float m = fmaxf(fmaxf(a, b), 1e-6f);
  const float q = (a - b) / m;
  return q * q;
}

// d(q^2)/da, d(q^2)/db with torch's conventions: maximum() splits the gradient evenly on ties, clip(min=) passes the
// gradient where the unclipped value is >= min.
TAIL_HD void tail_rel_cost_grad(float a, float b, float* ga, float* gb) {
  const float raw = fmaxf(a, b);
  const float m = fmaxf(raw, 1e-6f);
  const float d = a - b;
  const float q = d / m;
  const float pass = raw >= 1e-6f ? 1.f : 0.f;
  const float dm_da = pass * (a > b ? 1.f : (a == b ? 0.5f : 0.f));
  const float dm_db = pass * (b > a ? 1.f : (a == b ? 0.5f : 0.f));
  const float dq_dm = -d / (m * m);
  *ga = 2.f * q * (1.f / m + dq_dm * dm_da);
  *gb = 2.f * q * (-1.f / m + dq_dm * dm_db);
}

// values of the 14 channels BEFORE the weight
TAIL_HD void tail_channels(const TailSample& s, bool both_normals, float v[TAIL_CH]) {
  v[0] = s.rgb[0]; v[1] = s.rgb[1]; v[2] = s.rgb[2];
  v[3] = s.vn[0]; v[4] = s.vn[1]; v[5] = s.vn[2];
  v[6] = s.brdf[0]; v[7] = s.brdf[1]; v[8] = s.brdf[2];
  const float rough = s.brdf[3] * 0.9f + 0.09f, rough_j = s.brdfj[3] * 0.9f + 0.09f;
  v[9] = rough;
  v[10] = tail_rel_cost(s.brdf[0], s.brdfj[0]) + tail_rel_cost(s.brdf[1], s.brdfj[1]) +
          tail_rel_cost(s.brdf[2], s.brdfj[2]);
  v[11] = tail_rel_cost(rough, rough_j);
  if (both_normals) {
    const float d0 = s.vn[0] - s.dn[0], d1 = s.vn[1] - s.dn[1], d2 = s.vn[2] - s.dn[2];
    v[12] = d0 * d0 + d1 * d1 + d2 * d2;
    v[13] = fmaxf(s.vd[0] * s.vn[0] + s.vd[1] * s.vn[1] + s.vd[2] * s.vn[2], 0.f);
  } else {
    v[12] = 0.f;
    v[13] = 0.f;
  }
}

// G = gradient of the loss w.r.t. the 14 per-ray sums of this sample's ray
TAIL_HD void tail_backward_sample(const TailSample& s, bool both_normals, const float G[TAIL_CH], TailGrad& g) {
  float v[TAIL_CH];
  tail_channels(s, both_normals, v);
  float gw = 0.f;
  for (int k = 0; k < TAIL_CH; ++k) gw += G[k] * v[k];
  g.w = gw;
  const float w = s.w;
  for (int c = 0; c < 3; ++c) {
    g.rgb[c] = w * G[c];
    g.vn[c] = w * G[3 + c];
    g.dn[c] = 0.f;
    float ga, gb;
    tail_rel_cost_grad(s.brdf[c], s.brdfj[c], &ga, &gb);
    g.brdf[c] = w * G[6 + c] + w * G[10] * ga;
    g.brdfj[c] = w * G[10] * gb;
  }
  {
    const float rough = s.brdf[3] * 0.9f + 0.09f, rough_j = s.brdfj[3] * 0.9f + 0.09f;
    float ga, gb;
    tail_rel_cost_grad(rough, rough_j, &ga, &gb);
    g.brdf[3] = 0.9f * (w * G[9] + w * G[11] * ga);
    g.brdfj[3] = 0.9f * (w * G[11] * gb);
  }
  if (both_normals) {
    const float dot = s.vd[0] * s.vn[0] + s.vd[1] * s.vn[1] + s.vd[2] * s.vn[2];
    const float gate = dot >= 0.f ? 1.f : 0.f;         // clamp(min=0) passes the gradient where input >= min (ATen)
    for (int c = 0; c < 3; ++c) {
      const float d = s.vn[c] - s.dn[c];
      g.vn[c] += w * G[12] * 2.f * d + w * G[13] * gate * s.vd[c];
      g.dn[c] = -w * G[12] * 2.f * d;
    }
  }
}

// The whole argument check of each entry, run by tir_tail.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus.  dn and g_dn are optional.
inline int tail_fwd_check(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                          const float* brdfj, const float* vn, const float* viewdirs, const float* packed) {
  if (n <= 0) return 0;
  if (!w || !ray || !rgb || !brdf || !brdfj || !vn || !viewdirs || !packed) return TIR_ERR_NULL;
  return 1;
}

inline int tail_bwd_check(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                          const float* brdfj, const float* vn, const float* viewdirs, const float* g_packed,
                          const float* g_w, const float* g_rgb, const float* g_brdf, const float* g_brdfj,
                          const float* g_vn) {
  if (n <= 0) return 0;
  if (!w || !ray || !rgb || !brdf || !brdfj || !vn || !viewdirs || !g_packed || !g_w || !g_rgb || !g_brdf || !g_brdfj ||
      !g_vn)
    return TIR_ERR_NULL;
  return 1;
}
