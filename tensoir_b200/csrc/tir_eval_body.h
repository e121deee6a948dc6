// Per-pixel and per-window math of the test-view metrics (renderer.py:211-501, utils.py:93-139).
// Shared by the CUDA kernels (tir_eval.cu) and by a host build (tests/host_eval.cpp) that the CPU tests drive through
// the ctypes wrapper and compare with the oracle's restatement of the reference.
//
// The reference works on float32 tensors / arrays: clamps, products, the gamma power, the normal dot and the angle are
// fp32 here too, each rounded where the reference rounds (no FMA contraction in those).  Sums are fp64.  SSIM squares
// and multiplies in fp32 (img0**2 on a float32 tensor) and convolves in fp64 (scipy promotes to the filter's float64).
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"

#if defined(__CUDACC__)
#define EVAL_HD __host__ __device__ __forceinline__
#else
#define EVAL_HD inline
#endif

#define EVAL_WIN 11          // utils.py:94 filter_size
#define EVAL_HALO 10         // valid-mode convolution drops filter_size - 1 pixels per axis

// per-pixel sums (fp64), in the order of TirEvalView's outputs
enum { EVAL_SSE_RGB = 0, EVAL_SSE_BRDF = 1, EVAL_GSE_SINGLE = 2, EVAL_GSE_THREE = 3, EVAL_ANGLE = 4, EVAL_N_PIX = 5 };

// fp32 operations exactly rounded, never fused: the device compiler would otherwise contract a*b+c into an FMA
EVAL_HD float ev_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
EVAL_HD float ev_add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
EVAL_HD float ev_sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
EVAL_HD float ev_div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// torch.clamp(x, 0, 1): NaN stays NaN
EVAL_HD float ev_clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }

// F.normalize(x, dim=-1): x / max(||x||, 1e-12)
EVAL_HD void ev_normalize(const float x[3], float y[3]) {
  const float ss = ev_add(ev_add(ev_mul(x[0], x[0]), ev_mul(x[1], x[1])), ev_mul(x[2], x[2]));
  float n = sqrtf(ss);
  n = n < 1e-12f ? 1e-12f : n;
  for (int c = 0; c < 3; ++c) y[c] = ev_div(x[c], n);
}

struct EvalPixel {
  float rgb[3], brdf[3], gt[3];     // renderer maps (unclamped) and the ground truth
  float alb[3], gta[3];             // predicted albedo and GT albedo (read when has_albedo)
  int mask;                         // gt_mask of the pixel
  float nrm[3], gtn[3];             // predicted and GT normal (read when has_normal)
};

// One pixel's contribution to the per-view sums, and its two aligned albedo values.
//  - rgb / rgb_with_brdf clamped to [0,1] (renderer.py:265-266), squared error against gt_rgb (:300-303);
//  - aligned albedo: inside the mask clamp(ratio * albedo, 0, 1), else 1 (:274-289); gamma 1/2.2 squared error
//    against gt_albedo^(1/2.2) (:392-394, :462-468);
//  - normal angle: acos(clip(dot(normalize(gt), normalize(pred)), -1, 1)) * 180 / pi over every pixel (:353, :367,
//    :470), the dot in numpy's order (g0*p0 + g1*p1) + g2*p2.
EVAL_HD void eval_pixel(const EvalPixel& p, bool has_albedo, bool has_normal, float ratio_single,
                        const float ratio_three[3], double acc[EVAL_N_PIX], float al1[3], float al3[3]) {
  for (int c = 0; c < 3; ++c) {
    const float d0 = ev_sub(ev_clamp01(p.rgb[c]), p.gt[c]);
    const float d1 = ev_sub(ev_clamp01(p.brdf[c]), p.gt[c]);
    acc[EVAL_SSE_RGB] += (double)ev_mul(d0, d0);
    acc[EVAL_SSE_BRDF] += (double)ev_mul(d1, d1);
  }
  if (has_albedo) {
    const float g = (float)(1.0 / 2.2);       // the float32 array ** (1/2.2) casts the exponent to float32
    for (int c = 0; c < 3; ++c) {
      al1[c] = p.mask ? ev_clamp01(ev_mul(ratio_single, p.alb[c])) : 1.f;
      al3[c] = p.mask ? ev_clamp01(ev_mul(ratio_three[c], p.alb[c])) : 1.f;
      const float gt_g = powf(p.gta[c], g);
      const float e1 = ev_sub(gt_g, powf(al1[c], g));
      const float e3 = ev_sub(gt_g, powf(al3[c], g));
      acc[EVAL_GSE_SINGLE] += (double)ev_mul(e1, e1);
      acc[EVAL_GSE_THREE] += (double)ev_mul(e3, e3);
    }
  }
  if (has_normal) {
    float a[3], b[3];
    ev_normalize(p.gtn, a);
    ev_normalize(p.nrm, b);
    float dot = ev_add(ev_add(ev_mul(a[0], b[0]), ev_mul(a[1], b[1])), ev_mul(a[2], b[2]));
    dot = dot < -1.f ? -1.f : (dot > 1.f ? 1.f : dot);
    acc[EVAL_ANGLE] += (double)ev_div(ev_mul(acosf(dot), 180.f), (float)3.14159265358979323846);
  }
}

// Tap k of the normalised 11-tap Gaussian, sigma 1.5 (utils.py:104-109): exp(-0.5 ((k-5)/1.5)^2) / sum
EVAL_HD double eval_tap(int k) {
  double s = 0.0, t = 0.0;
  for (int i = 0; i < EVAL_WIN; ++i) {
    const double f = (double)(i - EVAL_WIN / 2) / 1.5;
    const double e = exp(-0.5 * (f * f));
    s += e;
    if (i == k) t = e;
  }
  return t / s;
}

// ---- work layout and argument checks (shared by the kernels and the host build) ----------------------------------
#define EVAL_PIX_BLOCKS 512  // blocks of the pixel pass; its partials occupy EVAL_N_PIX * EVAL_PIX_BLOCKS doubles
#define EVAL_TILE 16         // SSIM output tile (EVAL_TILE x EVAL_TILE windows per block)

inline int64_t eval_ssim_tiles(int32_t H, int32_t W) {
  if (H < EVAL_WIN || W < EVAL_WIN) return 0;
  return (int64_t)((W - EVAL_HALO + EVAL_TILE - 1) / EVAL_TILE) * ((H - EVAL_HALO + EVAL_TILE - 1) / EVAL_TILE);
}

inline int64_t eval_work_doubles(int32_t H, int32_t W) {
  return (int64_t)EVAL_N_PIX * EVAL_PIX_BLOCKS + 4 * eval_ssim_tiles(H, W);
}

// The whole argument check of each entry, run by tir_eval.cu and its host builds before their launches / loops:
// 1 run, 0 nothing to do, < 0 TirStatus
inline int eval_work_size_check(int32_t H, int32_t W, const int64_t* n_doubles) {
  if (!n_doubles) return TIR_ERR_NULL;
  return (H < 0 || W < 0) ? TIR_ERR_SHAPE : 1;
}

// the view's own fields; 0 for zero pixels
inline int eval_validate(const TirEvalView* v, bool* has_albedo, bool* has_normal, int* n_ssim) {
  if (!v) return TIR_ERR_NULL;
  if (v->H < 0 || v->W < 0) return TIR_ERR_SHAPE;
  if ((int64_t)v->H * v->W == 0) return 0;
  if (!v->rgb || !v->rgb_brdf || !v->gt_rgb) return TIR_ERR_NULL;
  if ((v->albedo == nullptr) != (v->gt_albedo == nullptr)) return TIR_ERR_NULL;
  if ((v->normal == nullptr) != (v->gt_normal == nullptr)) return TIR_ERR_NULL;
  *has_albedo = v->albedo != nullptr;
  *has_normal = v->normal != nullptr;
  if (*has_albedo && (!v->gt_mask || !v->ratio || !v->aligned_single || !v->aligned_three)) return TIR_ERR_NULL;
  *n_ssim = 0;
  if (v->ssim) {
    if (v->H < EVAL_WIN || v->W < EVAL_WIN) return TIR_ERR_SHAPE;
    *n_ssim = *has_albedo ? 4 : 2;
  }
  return 1;
}

inline int eval_view_check(const TirEvalView* v, const double* work, int64_t work_cap, const double* out,
                           bool* has_albedo, bool* has_normal, int* n_ssim) {
  const int rc = eval_validate(v, has_albedo, has_normal, n_ssim);
  if (rc <= 0) return rc;
  if (!work || !out) return TIR_ERR_NULL;
  return work_cap < eval_work_doubles(v->H, v->W) ? TIR_ERR_CAPACITY : 1;
}

// ---- tir_eval_pairs: [P * EVAL_PAIR_SSE_BLOCKS] squared-error partials, then [P * tiles] SSIM partials -------------
#define EVAL_PAIR_SSE_BLOCKS 64

inline int64_t eval_pairs_work_doubles(int32_t P, int32_t H, int32_t W) {
  return (int64_t)P * (EVAL_PAIR_SSE_BLOCKS + eval_ssim_tiles(H, W));
}

inline int eval_pairs_work_size_check(int32_t P, int32_t H, int32_t W, const int64_t* n_doubles) {
  if (!n_doubles) return TIR_ERR_NULL;
  return (P < 0 || H < 0 || W < 0) ? TIR_ERR_SHAPE : 1;
}

// 0 for no pairs
inline int eval_pairs_validate(const float* a, const float* b, int32_t P, int32_t H, int32_t W, const double* work,
                               int64_t work_cap, const double* out) {
  if (P < 0 || H < 0 || W < 0) return TIR_ERR_SHAPE;
  if (P == 0) return 0;
  if (H < EVAL_WIN || W < EVAL_WIN) return TIR_ERR_SHAPE;
  if (!a || !b || !work || !out) return TIR_ERR_NULL;
  if (work_cap < eval_pairs_work_doubles(P, H, W)) return TIR_ERR_CAPACITY;
  return 1;
}

// SSIM of one window from the blurred moments E[x], E[y], E[x^2], E[y^2], E[xy] (utils.py:118-137, max_val = 1)
EVAL_HD double eval_ssim_point(double mu0, double mu1, double e00, double e11, double e01) {
  const double mu00 = mu0 * mu0, mu11 = mu1 * mu1, mu01 = mu0 * mu1;
  double s00 = e00 - mu00, s11 = e11 - mu11, s01 = e01 - mu01;
  s00 = s00 > 0.0 ? s00 : (s00 == s00 ? 0.0 : s00);          // np.maximum(0., x) keeps NaN
  s11 = s11 > 0.0 ? s11 : (s11 == s11 ? 0.0 : s11);
  const double sg = s01 > 0.0 ? 1.0 : (s01 < 0.0 ? -1.0 : s01);
  s01 = sg * fmin(sqrt(s00 * s11), fabs(s01));
  const double c1 = 0.01 * 0.01, c2 = 0.03 * 0.03;
  const double numer = (2.0 * mu01 + c1) * (2.0 * s01 + c2);
  const double denom = (mu00 + mu11 + c1) * (s00 + s11 + c2);
  return numer / denom;
}
