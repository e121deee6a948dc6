// Host twin of csrc/tir_relight.cu and of tir_eval_pairs (csrc/tir_eval.cu) for the CPU tests of
// tensoir_b200/relighting.py: the SAME C-ABI signatures (include/tensoir_b200.h), argument checks and per-sample /
// per-ray / per-window math (csrc/tir_relight_body.h, csrc/tir_eval_body.h), with plain loops instead of kernels.
// "Device" pointers are host pointers here.  The visibility list is filled in slot order.
#include <vector>
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_relight_body.h"

extern "C" int tir_relight_sample(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* depth,
                                  const float* normal, const float* acc, int64_t n, int32_t n_samples,
                                  float acc_mask_threshold, const double* u, int32_t* bin, int32_t* pos,
                                  float* list_o, float* list_d, int64_t capacity, int64_t* count, void*) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc <= 0 || n_samples == 0) return rc < 0 ? rc : TIR_OK;
  if (!rays || !depth || !normal || !acc || !u || !bin || !pos || !count) return TIR_ERR_NULL;
  if (capacity < 0) return TIR_ERR_SHAPE;
  if (capacity > 0 && (!list_o || !list_d)) return TIR_ERR_NULL;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t i = 0; i < n; ++i)
      for (int s = 0; s < n_samples; ++s) {
        const int64_t t = ((int64_t)l * n + i) * n_samples + s;
        bin[t] = 0;
        pos[t] = -1;
        if (!(acc[i] > acc_mask_threshold)) continue;
        const TirEnvMap& e = envs[l];
        const int b = rl_bin(e.cdf, e.H * e.W, u[t]);
        bin[t] = b;
        const float L3[3] = {e.dir[b * 3], e.dir[b * 3 + 1], e.dir[b * 3 + 2]};
        if (!(rl_cosine(L3, normal + i * 3) > 1e-6f)) continue;
        const int64_t row = (*count)++;
        if (row >= capacity) continue;
        float o[3];
        rl_surface(rays + i * 6, depth[i], o);
        for (int c = 0; c < 3; ++c) { list_o[row * 3 + c] = o[c]; list_d[row * 3 + c] = L3[c]; }
        pos[t] = (int32_t)row;
      }
  return TIR_OK;
}

extern "C" int tir_relight_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                                 const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                                 const float* acc, int64_t n, int32_t n_samples, float acc_mask_threshold,
                                 const float* rescale, const int32_t* bin, const int32_t* pos, const float* vis_list,
                                 int32_t vis_kind, float* with_bg, float* without_bg, int64_t out_rows, int64_t row0,
                                 void*) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc <= 0) return rc;
  if (n_samples <= 0) return TIR_ERR_SHAPE;
  if (!rays || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !bin || !pos || !with_bg ||
      !without_bg)
    return TIR_ERR_NULL;
  if (rough_stride != 1 && rough_stride != 3) return TIR_ERR_SHAPE;
  if (vis_kind != 0 && vis_kind != 1) return TIR_ERR_CONFIG;
  if (row0 < 0 || row0 + n > out_rows) return TIR_ERR_SHAPE;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t i = 0; i < n; ++i) {
      const TirEnvMap& e = envs[l];
      const float* ray = rays + i * 6;
      float wo[3] = {1.f, 1.f, 1.f};
      if (acc[i] > acc_mask_threshold) {
        tir::PointCtx c;
        rl_point(ray, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride, fresnel + i * 3,
                 rescale, c);
        // the kernel's order: lane k sums samples k, k+32, ...; then the xor butterfly over the 32 lanes
        float lane[32][3] = {};
        for (int s = 0; s < n_samples; ++s) {
          const int64_t t = ((int64_t)l * n + i) * n_samples + s;
          const int b = bin[t], q = pos[t];
          const float vis = q >= 0 ? (vis_kind ? 1.f - vis_list[q] : vis_list[q]) : 0.f;
          rl_contrib(c, e.dir + (int64_t)b * 3, e.rgb + (int64_t)b * 3, e.pdf_return[b], vis, lane[s % 32]);
        }
        for (int o = 16; o > 0; o >>= 1) {
          float nxt[32][3];
          for (int k = 0; k < 32; ++k)
            for (int ch = 0; ch < 3; ++ch) nxt[k][ch] = lane[k][ch] + lane[k ^ o][ch];
          for (int k = 0; k < 32; ++k)
            for (int ch = 0; ch < 3; ++ch) lane[k][ch] = nxt[k][ch];
        }
        for (int ch = 0; ch < 3; ++ch) wo[ch] = tir::tone(lane[0][ch] / (float)n_samples, 1);
      }
      float wb[3];
      rl_composite(e, ray, acc[i], wo, wb);
      const int64_t r = ((int64_t)l * out_rows + row0 + i) * 3;
      for (int ch = 0; ch < 3; ++ch) { without_bg[r + ch] = wo[ch]; with_bg[r + ch] = wb[ch]; }
    }
  return TIR_OK;
}

extern "C" int tir_eval_pairs_work_size(int32_t P, int32_t H, int32_t W, int64_t* n_doubles) {
  if (!n_doubles) return TIR_ERR_NULL;
  if (P < 0 || H < 0 || W < 0) return TIR_ERR_SHAPE;
  *n_doubles = eval_pairs_work_doubles(P, H, W);
  return TIR_OK;
}

// mean SSIM of one pair over the valid windows of the three channels (tests/host_eval.cpp's loop order)
static double host_ssim(int H, int W, const float* a, const float* b) {
  const int Ho = H - EVAL_HALO, Wo = W - EVAL_HALO;
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
          const float xa = a[pix * 3 + c], xb = b[pix * 3 + c];
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

extern "C" int tir_eval_pairs(const float* a, const float* b, int32_t P, int32_t H, int32_t W, double* work,
                              int64_t work_cap, double* out, void*) {
  const int rc = eval_pairs_validate(a, b, P, H, W, work, work_cap, out);
  if (rc <= 0) return rc;
  const int64_t n = (int64_t)H * W * 3;
  for (int p = 0; p < P; ++p) {
    double sse = 0.0;
    for (int64_t i = 0; i < n; ++i) {
      const float d = ev_sub(a[p * n + i], b[p * n + i]);
      sse += (double)ev_mul(d, d);
    }
    out[2 * p] = sse;
    out[2 * p + 1] = host_ssim(H, W, a + p * n, b + p * n);
  }
  return TIR_OK;
}
