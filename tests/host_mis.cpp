// Host twin of csrc/tir_relight_mis.cu for the tests of tensoir_b200/mis.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (mis_sample_check, mis_shade_check) and per-sample math
// of csrc/tir_mis_body.h, with plain loops instead of kernels.  "Device" pointers are host pointers here.  The
// visibility list is filled in slot order; the warp sums are the kernels' 32 lanes and xor butterfly.  Two more entries
// expose the texel lookup and the BRDF-strategy density to the stage checks.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_mis_body.h"

extern "C" int tir_relight_mis_sample(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* depth,
                                      const float* normal, const float* albedo, const float* rough,
                                      int32_t rough_stride, const float* fresnel, const float* acc, int64_t n,
                                      int32_t S_l, int32_t S_b, float acc_mask_threshold, const double* u_light,
                                      const double* u_brdf, float* dir, int32_t* pos, float* list_o, float* list_d,
                                      int64_t capacity, int64_t* count, void*) {
  const int rc = mis_sample_check(envs, n_lights, rays, depth, normal, albedo, rough, rough_stride, fresnel, acc, n,
                                  S_l, S_b, u_light, u_brdf, dir, pos, list_o, list_d, capacity, count);
  if (rc <= 0) return rc;
  const int64_t n_light = (int64_t)n_lights * n * S_l, total = n_light + n * S_b;
  for (int64_t t = 0; t < total; ++t) {
    const bool light = t < n_light;
    const int64_t i = light ? (t / S_l) % n : (t - n_light) / S_b;
    float w[3] = {0.f, 0.f, 0.f};
    pos[t] = -1;
    if (acc[i] > acc_mask_threshold) {
      if (light) {
        const TirEnvMap& e = envs[t / S_l / n];
        const double* u = u_light + t * 3;
        mis_light_dir(e, rl_bin(e.cdf, e.H * e.W, u[0]), u + 1, w);
      } else {
        tir::PointCtx c;
        const float one[3] = {1.f, 1.f, 1.f};
        rl_point(rays + i * 6, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride, fresnel + i * 3,
                 one, c);
        MisPoint m;
        mis_point(c, m);
        mis_brdf_dir(c, m, u_brdf + (t - n_light) * 3, w);
      }
      if (rl_cosine(w, normal + i * 3) > 1e-6f) {
        const int64_t row = (*count)++;
        if (row < capacity) {
          float o[3];
          rl_surface(rays + i * 6, depth[i], o);
          for (int e = 0; e < 3; ++e) { list_o[row * 3 + e] = o[e]; list_d[row * 3 + e] = w[e]; }
          pos[t] = (int32_t)row;
        }
      }
    }
    for (int e = 0; e < 3; ++e) dir[t * 3 + e] = w[e];
  }
  return TIR_OK;
}

extern "C" int tir_relight_mis_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                                     const float* albedo, const float* rough, int32_t rough_stride,
                                     const float* fresnel, const float* acc, int64_t n, int32_t S_l, int32_t S_b,
                                     float acc_mask_threshold, const float* rescale, const float* dir,
                                     const int32_t* pos, const float* vis_list, int32_t vis_kind, float* with_bg,
                                     float* without_bg, float* linear_out, int64_t out_rows, int64_t row0, void*) {
  const int rc = mis_shade_check(envs, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, S_l, S_b,
                                 rescale, dir, pos, vis_list, vis_kind, with_bg, without_bg, out_rows, row0);
  if (rc <= 0) return rc;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t i = 0; i < n; ++i) {
      const TirEnvMap& e = envs[l];
      const float* ray = rays + i * 6;
      float wo[3] = {1.f, 1.f, 1.f}, lin[3] = {0.f, 0.f, 0.f};
      if (acc[i] > acc_mask_threshold) {
        tir::PointCtx c;
        rl_point(ray, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride, fresnel + i * 3,
                 rescale, c);
        MisPoint m;
        mis_point(c, m);
        const int64_t kl = ((int64_t)l * n + i) * S_l, kb = (int64_t)n_lights * n * S_l + i * S_b;
        float lane[32][3] = {};
        for (int k = 0; k < 32; ++k)
          mis_lane(e, c, m, dir + kl * 3, pos + kl, S_l, dir + kb * 3, pos + kb, S_b, vis_list, vis_kind, k, 32,
                   lane[k]);
        for (int o = 16; o > 0; o >>= 1) {
          float nxt[32][3];
          for (int k = 0; k < 32; ++k)
            for (int ch = 0; ch < 3; ++ch) nxt[k][ch] = lane[k][ch] + lane[k ^ o][ch];
          for (int k = 0; k < 32; ++k)
            for (int ch = 0; ch < 3; ++ch) lane[k][ch] = nxt[k][ch];
        }
        for (int ch = 0; ch < 3; ++ch) {
          lin[ch] = lane[0][ch];
          wo[ch] = tir::tone(lin[ch], 1);
        }
      }
      float wb[3];
      rl_composite(e, ray, acc[i], wo, wb);
      const int64_t r = ((int64_t)l * out_rows + row0 + i) * 3;
      for (int ch = 0; ch < 3; ++ch) {
        without_bg[r + ch] = wo[ch];
        with_bg[r + ch] = wb[ch];
        if (linear_out) linear_out[r + ch] = lin[ch];
      }
    }
  return TIR_OK;
}

// rl_texel and p_light of n directions [n,3] under one map
extern "C" int host_mis_texel(const TirEnvMap* e, const float* d, int64_t n, int32_t* bin, double* p_light) {
  for (int64_t k = 0; k < n; ++k) {
    bin[k] = rl_texel(*e, d + k * 3);
    p_light[k] = mis_pdf_light(*e, bin[k]);
  }
  return TIR_OK;
}

// p_brdf of K directions per ray, dirs [n,K,3], at the GGX context rl_point builds for each ray
extern "C" int host_mis_pdf_brdf(const float* rays, const float* normal, const float* rough, int32_t rough_stride,
                                 int64_t n, const float* dirs, int32_t K, double* p) {
  const float zero[3] = {0.f, 0.f, 0.f}, one[3] = {1.f, 1.f, 1.f};
  for (int64_t i = 0; i < n; ++i) {
    tir::PointCtx c;
    rl_point(rays + i * 6, normal + i * 3, zero, rough + i * rough_stride, rough_stride, zero, one, c);
    MisPoint m;
    mis_point(c, m);
    for (int k = 0; k < K; ++k) p[i * K + k] = mis_pdf_brdf(c, m, dirs + (i * K + k) * 3);
  }
  return TIR_OK;
}
