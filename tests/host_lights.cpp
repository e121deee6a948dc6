// Host twin of csrc/tir_lights.cu for the tests of tensoir_b200/lighting.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (the lt_*_check functions) and per-slot / per-ray math of
// csrc/tir_lights_body.h, with plain loops instead of kernels.  "Device" pointers are host pointers here.  The
// shadow-ray list is filled in slot order.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_lights_body.h"

extern "C" int tir_lights_sample(const TirLight* lights, int32_t n_lights, const float* rays, const float* depth,
                                 const float* normal, const float* acc, int64_t n, float acc_mask_threshold,
                                 const double* u, float* L, float* falloff, int32_t* pos, float* list_o, float* list_d,
                                 int64_t capacity, int64_t* count, void*) {
  LightTable lt;
  const int rc = lt_sample_check(lights, n_lights, rays, depth, normal, acc, n, u, L, falloff, pos, list_o, list_d,
                                 capacity, count, lt);
  if (rc <= 0) return rc;
  for (int j = 0; j < n_lights; ++j)
    for (int64_t i = 0; i < n; ++i)
      for (int s = 0; s < lt.l[j].n_samples; ++s) {
        const int64_t t = n * lt.prefix[j] + i * lt.l[j].n_samples + s;
        for (int c = 0; c < 3; ++c) L[t * 3 + c] = 0.f;
        falloff[t] = 0.f;
        pos[t] = -1;
        if (!(acc[i] > acc_mask_threshold)) continue;
        float o[3];
        rl_surface(rays + i * 6, depth[i], o);
        lt_sample(lt.l[j], o, u + t * 2, L + t * 3, falloff[t]);
        if (!(rl_cosine(L + t * 3, normal + i * 3) > 1e-6f && falloff[t] > 0.f)) continue;
        const int64_t row = (*count)++;
        if (row >= capacity) continue;
        for (int c = 0; c < 3; ++c) { list_o[row * 3 + c] = o[c]; list_d[row * 3 + c] = L[t * 3 + c]; }
        pos[t] = (int32_t)row;
      }
  return TIR_OK;
}

extern "C" int tir_lights_shade(const TirLight* lights, int32_t n_lights, const float* rays, const float* normal,
                                const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                                const float* acc, int64_t n, float acc_mask_threshold, const float* rescale,
                                const float* background, const float* L, const float* falloff, const int32_t* pos,
                                const float* vis_list, int32_t vis_kind, float* with_bg, float* without_bg,
                                float* linear, int64_t out_rows, int64_t row0, void*) {
  LightTable lt;
  const int rc = lt_shade_check(lights, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, rescale,
                                background, L, falloff, pos, vis_list, vis_kind, with_bg, without_bg, out_rows, row0,
                                lt);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i) {
    const bool hit = acc[i] > acc_mask_threshold;
    float lin[3] = {0.f, 0.f, 0.f};
    if (hit) {
      tir::PointCtx c;
      rl_point(rays + i * 6, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride, fresnel + i * 3,
               rescale, c);
      for (int j = 0; j < n_lights; ++j) {
        const int K = lt.l[j].n_samples;
        const int64_t k0 = n * lt.prefix[j] + i * K;
        // the kernel's order: lane k sums slots k, k+32, ...; then the xor butterfly over the 32 lanes
        float lane[32][3] = {};
        for (int s = 0; s < K; ++s) {
          const int q = pos[k0 + s];
          if (q < 0) continue;
          const float vis = rl_vis(vis_list, vis_kind, q);
          lt_contrib(c, L + (k0 + s) * 3, falloff[k0 + s], vis, lane[s % 32]);
        }
        for (int o = 16; o > 0; o >>= 1) {
          float nxt[32][3];
          for (int k = 0; k < 32; ++k)
            for (int ch = 0; ch < 3; ++ch) nxt[k][ch] = lane[k][ch] + lane[k ^ o][ch];
          for (int k = 0; k < 32; ++k)
            for (int ch = 0; ch < 3; ++ch) lane[k][ch] = nxt[k][ch];
        }
        for (int ch = 0; ch < 3; ++ch) lin[ch] = lin[ch] + lt.l[j].power[ch] * (lane[0][ch] / (float)K);
      }
    }
    float wo[3], wb[3];
    lt_finish(hit, acc[i], lin, background, wo, wb);
    const int64_t r = (row0 + i) * 3;
    for (int ch = 0; ch < 3; ++ch) {
      without_bg[r + ch] = wo[ch];
      with_bg[r + ch] = wb[ch];
      if (linear) linear[r + ch] = lin[ch];
    }
  }
  return TIR_OK;
}
