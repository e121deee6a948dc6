// Host twin of csrc/tir_transport.cu for the tests of tensoir_b200/light_fit.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (tt_sample_check, tt_build_check) and per-(hit, texel)
// math of csrc/tir_transport_body.h, with plain loops instead of kernels.  "Device" pointers are host pointers here.
// The visibility list is filled in (ray, texel) order.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_transport_body.h"

extern "C" int tir_transport_sample(const float* dirs, int32_t K, const float* rays, const float* depth,
                                    const float* normal, const float* acc, int64_t n, float acc_mask_threshold,
                                    int32_t* pos, float* list_o, float* list_d, int64_t capacity, int64_t* count,
                                    void*) {
  const int rc = tt_sample_check(dirs, K, rays, depth, normal, acc, n, pos, list_o, list_d, capacity, count);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i)
    for (int k = 0; k < K; ++k) {
      const int64_t t = i * K + k;
      pos[t] = -1;
      if (!(acc[i] > acc_mask_threshold)) continue;
      if (!(rl_cosine(dirs + (int64_t)k * 3, normal + i * 3) > 1e-6f)) continue;
      const int64_t row = (*count)++;
      if (row >= capacity) continue;
      float o[3];
      rl_surface(rays + i * 6, depth[i], o);
      for (int c = 0; c < 3; ++c) { list_o[row * 3 + c] = o[c]; list_d[row * 3 + c] = dirs[k * 3 + c]; }
      pos[t] = (int32_t)row;
    }
  return TIR_OK;
}

extern "C" int tir_transport_build(const float* dirs, const float* domega, int32_t K, const float* rays,
                                   const float* normal, const float* albedo, const float* rough, int32_t rough_stride,
                                   const float* fresnel, const float* acc, int64_t n, float acc_mask_threshold,
                                   const float* rescale, const int32_t* pos, const float* vis_list, int32_t vis_kind,
                                   float* T, void*) {
  const int rc = tt_build_check(dirs, domega, K, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, rescale,
                                pos, vis_list, vis_kind, T);
  if (rc <= 0) return rc;
  const int64_t plane = n * K;
  for (int64_t i = 0; i < n; ++i) {
    const bool hit = acc[i] > acc_mask_threshold;
    tir::PointCtx c;
    if (hit)
      rl_point(rays + i * 6, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride, fresnel + i * 3,
               rescale, c);
    for (int k = 0; k < K; ++k) {
      const int64_t t = i * K + k;
      float v[3] = {0.f, 0.f, 0.f};
      if (hit && pos[t] >= 0) {
        const float vis = rl_vis(vis_list, vis_kind, pos[t]);
        tt_contrib(c, dirs + (int64_t)k * 3, domega[k], vis, v);
      }
      for (int ch = 0; ch < 3; ++ch) T[ch * plane + t] = v[ch];
    }
  }
  return TIR_OK;
}
