// Host twin of csrc/tir_eval.cu for the CPU tests of tensoir_b200/evaluation.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (eval_work_size_check, eval_view_check) and per-pixel /
// per-window math of csrc/tir_eval_body.h, with plain loops instead of kernels.  "Device" pointers are host pointers
// here.
#include <vector>
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_eval_body.h"

extern "C" int tir_eval_work_size(int32_t H, int32_t W, int64_t* n_doubles) {
  const int rc = eval_work_size_check(H, W, n_doubles);
  if (rc <= 0) return rc;
  *n_doubles = eval_work_doubles(H, W);
  return TIR_OK;
}

// mean SSIM of one pair over the valid windows of the three channels
static double host_ssim(const TirEvalView& v, const float* a, const float* b, bool clamp_a) {
  const int H = v.H, W = v.W, Ho = H - EVAL_HALO, Wo = W - EVAL_HALO;
  double taps[EVAL_WIN];
  for (int k = 0; k < EVAL_WIN; ++k) taps[k] = eval_tap(k);
  std::vector<double> m(5 * (size_t)Ho * W);
  double sum = 0.0;
  for (int c = 0; c < 3; ++c) {
    for (int r = 0; r < Ho; ++r)
      for (int x = 0; x < W; ++x) {
        double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
        for (int j = 0; j < EVAL_WIN; ++j) {
          const int64_t pix = (int64_t)(r + j) * W + x;
          float xa = a[pix * 3 + c];
          const float xb = b[pix * 3 + c];
          if (clamp_a) xa = ev_clamp01(xa);
          acc[0] += taps[j] * (double)xa;
          acc[1] += taps[j] * (double)xb;
          acc[2] += taps[j] * (double)ev_mul(xa, xa);
          acc[3] += taps[j] * (double)ev_mul(xb, xb);
          acc[4] += taps[j] * (double)ev_mul(xa, xb);
        }
        for (int q = 0; q < 5; ++q) m[((size_t)q * Ho + r) * W + x] = acc[q];
      }
    for (int r = 0; r < Ho; ++r)
      for (int x = 0; x < Wo; ++x) {
        double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
        for (int j = 0; j < EVAL_WIN; ++j)
          for (int q = 0; q < 5; ++q) acc[q] += taps[j] * m[((size_t)q * Ho + r) * W + x + j];
        sum += eval_ssim_point(acc[0], acc[1], acc[2], acc[3], acc[4]);
      }
  }
  return sum / ((double)Ho * (double)Wo * 3.0);
}

extern "C" int tir_eval_view(const TirEvalView* view, double* work, int64_t work_cap, double* out, void*) {
  bool has_albedo = false, has_normal = false;
  int n_ssim = 0;
  const int rc = eval_view_check(view, work, work_cap, out, &has_albedo, &has_normal, &n_ssim);
  if (rc <= 0) return rc;
  const TirEvalView& v = *view;
  float r1 = 0.f, r3[3] = {0.f, 0.f, 0.f};
  if (has_albedo) { r1 = v.ratio[0]; r3[0] = v.ratio[1]; r3[1] = v.ratio[2]; r3[2] = v.ratio[3]; }
  double acc[EVAL_N_PIX] = {0.0, 0.0, 0.0, 0.0, 0.0};
  const int64_t n = (int64_t)v.H * v.W;
  for (int64_t i = 0; i < n; ++i) {
    EvalPixel p;
    for (int c = 0; c < 3; ++c) {
      p.rgb[c] = v.rgb[i * 3 + c]; p.brdf[c] = v.rgb_brdf[i * 3 + c]; p.gt[c] = v.gt_rgb[i * 3 + c];
      p.alb[c] = has_albedo ? v.albedo[i * 3 + c] : 0.f;
      p.gta[c] = has_albedo ? v.gt_albedo[i * 3 + c] : 0.f;
      p.nrm[c] = has_normal ? v.normal[i * 3 + c] : 0.f;
      p.gtn[c] = has_normal ? v.gt_normal[i * 3 + c] : 0.f;
    }
    p.mask = has_albedo ? (v.gt_mask[i] != 0) : 0;
    float al1[3], al3[3];
    eval_pixel(p, has_albedo, has_normal, r1, r3, acc, al1, al3);
    if (has_albedo)
      for (int c = 0; c < 3; ++c) { v.aligned_single[i * 3 + c] = al1[c]; v.aligned_three[i * 3 + c] = al3[c]; }
  }
  for (int q = 0; q < EVAL_N_PIX; ++q) out[q] = acc[q];
  out[5] = n_ssim > 0 ? host_ssim(v, v.rgb, v.gt_rgb, true) : 0.0;
  out[6] = n_ssim > 1 ? host_ssim(v, v.rgb_brdf, v.gt_rgb, true) : 0.0;
  out[7] = n_ssim > 2 ? host_ssim(v, v.aligned_single, v.gt_albedo, false) : 0.0;
  out[8] = n_ssim > 3 ? host_ssim(v, v.aligned_three, v.gt_albedo, false) : 0.0;
  return TIR_OK;
}
