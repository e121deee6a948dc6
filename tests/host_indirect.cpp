// Host twin of csrc/tir_indirect.cu for the tests of tensoir_b200/indirect.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (the ind_*_check functions) and per-slot / per-hit math
// of csrc/tir_indirect_body.h, and the direct loop rl_direct_lane of csrc/tir_relight_body.h, with plain loops instead
// of kernels.  Only the scratch size of tir_indirect_hits differs: this build needs none.  "Device" pointers are host
// pointers here.  The secondary list is filled in slot order; the warp sums are the kernels' 32 lanes and xor
// butterfly.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_indirect_body.h"

// the kernels' warp_sum of 32 per-lane partials
static void butterfly(float lane[32][3], float out[3]) {
  for (int o = 16; o > 0; o >>= 1) {
    float nxt[32][3];
    for (int k = 0; k < 32; ++k)
      for (int ch = 0; ch < 3; ++ch) nxt[k][ch] = lane[k][ch] + lane[k ^ o][ch];
    for (int k = 0; k < 32; ++k)
      for (int ch = 0; ch < 3; ++ch) lane[k][ch] = nxt[k][ch];
  }
  for (int ch = 0; ch < 3; ++ch) out[ch] = lane[0][ch];
}

static void direct_sum(const TirEnvMap& e, const tir::PointCtx& c, const int32_t* bin, const int32_t* pos,
                       const float* vis, int vis_kind, int S, float out[3]) {
  float lane[32][3] = {};
  for (int k = 0; k < 32; ++k) rl_direct_lane(e, c, bin, pos, vis, vis_kind, S, k, 32, lane[k]);
  butterfly(lane, out);
}

extern "C" int tir_indirect_sample(const float* rays, const float* depth, const float* normal, const float* albedo,
                                   const float* rough, int32_t rough_stride, const float* fresnel, const float* acc,
                                   int64_t n, int32_t K, float acc_mask_threshold, const float* rescale,
                                   const double* u, float* dir, float* T, int32_t* pos, float* list_o, float* list_d,
                                   int64_t capacity, int64_t* count, void*) {
  const int rc = ind_sample_check(rays, depth, normal, albedo, rough, rough_stride, fresnel, acc, n, K, rescale, u, dir,
                                  T, pos, list_o, list_d, capacity, count);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i)
    for (int k = 0; k < K; ++k) {
      const int64_t t = i * K + k;
      float om[3] = {0.f, 0.f, 0.f}, Tk[3] = {0.f, 0.f, 0.f};
      pos[t] = -1;
      if (acc[i] > acc_mask_threshold) {
        tir::PointCtx c;
        rl_point(rays + i * 6, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride,
                 fresnel + i * 3, rescale, c);
        float z;
        ind_direction(normal + i * 3, u + t * 2, om, z);
        if (ind_throughput(c, om, z, Tk)) {
          const int64_t row = (*count)++;
          if (row < capacity) {
            float o[3];
            rl_surface(rays + i * 6, depth[i], o);
            for (int e = 0; e < 3; ++e) { list_o[row * 3 + e] = o[e]; list_d[row * 3 + e] = om[e]; }
            pos[t] = (int32_t)row;
          }
        }
      }
      for (int e = 0; e < 3; ++e) { dir[t * 3 + e] = om[e]; T[t * 3 + e] = Tk[e]; }
    }
  return TIR_OK;
}

extern "C" int tir_indirect_hits_work_size(int64_t n, int32_t K, int64_t* bytes) {
  const int rc = ind_hits_work_size_check(n, K, bytes);
  if (rc <= 0) return rc;
  *bytes = 0;
  return TIR_OK;
}

extern "C" int tir_indirect_hits(int64_t n, int32_t K, const int32_t* pos, const float* list_o, const float* list_d,
                                 const float* t_last, const float* acc, const float* depth, int32_t vis_kind,
                                 const float* aabb, float* hit_rays, float* xn, float* w, int32_t* hit,
                                 int64_t capacity, int64_t* count, void*, int64_t, void*) {
  const int rc = ind_hits_check(n, K, pos, list_o, list_d, t_last, acc, depth, vis_kind, aabb, hit_rays, xn, w, hit,
                                capacity, count);
  if (rc < 0) return rc;
  *count = 0;
  if (rc == 0) return TIR_OK;
  int64_t row = 0;
  for (int64_t t = 0; t < n * K; ++t) {
    hit[t] = -1;
    const int32_t q = pos[t];
    if (q < 0) continue;
    const float wq = ind_weight(vis_kind, t_last[q], acc[q]);
    if (!ind_is_hit(wq, acc[q])) continue;
    if (row < capacity) {
      float x[3], xq[3];
      ind_point(list_o + (int64_t)q * 3, list_d + (int64_t)q * 3, depth[q], acc[q], aabb, x, xq);
      for (int e = 0; e < 3; ++e) {
        hit_rays[row * 6 + e] = x[e];
        hit_rays[row * 6 + 3 + e] = list_d[(int64_t)q * 3 + e];
        xn[row * 3 + e] = xq[e];
      }
      w[row] = wq;
      hit[t] = (int32_t)row;
    }
    ++row;
  }
  *count = row;
  return TIR_OK;
}

extern "C" int tir_indirect_radiance(const TirEnvMap* envs, int32_t n_lights, const float* hit_rays,
                                     const float* normal, const float* albedo, const float* rough,
                                     int32_t rough_stride, const float* fresnel, int64_t m, int32_t n_samples,
                                     const float* rescale, const int32_t* bin, const int32_t* pos,
                                     const float* vis_list, int32_t vis_kind, float* Lo, int64_t out_rows,
                                     int64_t row0, void*) {
  const int rc = ind_radiance_check(envs, n_lights, hit_rays, normal, albedo, rough, rough_stride, fresnel, m,
                                    n_samples, rescale, bin, pos, vis_list, vis_kind, Lo, out_rows, row0);
  if (rc <= 0) return rc;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t h = 0; h < m; ++h) {
      tir::PointCtx c;
      rl_point(hit_rays + h * 6, normal + h * 3, albedo + h * 3, rough + h * rough_stride, rough_stride,
               fresnel + h * 3, rescale, c);
      const int64_t k0 = ((int64_t)l * m + h) * n_samples;
      float s[3];
      direct_sum(envs[l], c, bin + k0, pos + k0, vis_list, vis_kind, n_samples, s);
      for (int ch = 0; ch < 3; ++ch) Lo[((int64_t)l * out_rows + row0 + h) * 3 + ch] = s[ch] / (float)n_samples;
    }
  return TIR_OK;
}

extern "C" int tir_indirect_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                                  const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                                  const float* acc, int64_t n, int32_t n_samples, float acc_mask_threshold,
                                  const float* rescale, const int32_t* bin, const int32_t* pos, const float* vis_list,
                                  int32_t vis_kind, int32_t K, const float* T, const int32_t* hit, const float* w,
                                  const float* Lo, int64_t m_h, float* with_bg, float* without_bg, float* indirect,
                                  int64_t out_rows, int64_t row0, void*) {
  const int rc = ind_shade_check(envs, n_lights, rays, normal, albedo, rough, rough_stride, fresnel, acc, n, n_samples,
                                 rescale, bin, pos, vis_kind, K, T, hit, w, Lo, m_h, with_bg, without_bg, out_rows,
                                 row0);
  if (rc <= 0) return rc;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t i = 0; i < n; ++i) {
      const TirEnvMap& e = envs[l];
      const float* ray = rays + i * 6;
      float wo[3] = {1.f, 1.f, 1.f}, ind[3] = {0.f, 0.f, 0.f};
      if (acc[i] > acc_mask_threshold) {
        tir::PointCtx c;
        rl_point(ray, normal + i * 3, albedo + i * 3, rough + i * rough_stride, rough_stride, fresnel + i * 3,
                 rescale, c);
        const int64_t k0 = ((int64_t)l * n + i) * n_samples;
        float d[3], s[3];
        direct_sum(e, c, bin + k0, pos + k0, vis_list, vis_kind, n_samples, d);
        float lane[32][3] = {};
        bool any = false;
        for (int k = 0; k < K; ++k) {
          const int64_t t = i * K + k;
          const int h = hit[t];
          if (h < 0) continue;
          any = true;
          ind_add(T + t * 3, w[h], Lo + ((int64_t)l * m_h + h) * 3, lane[k % 32]);
        }
        butterfly(lane, s);
        for (int ch = 0; ch < 3; ++ch) {
          const float dm = d[ch] / (float)n_samples;
          if (any) ind[ch] = ev_div(s[ch], (float)K);
          wo[ch] = tir::tone(any ? ev_add(dm, ind[ch]) : dm, 1);
        }
      }
      float wb[3];
      rl_composite(e, ray, acc[i], wo, wb);
      const int64_t r = ((int64_t)l * out_rows + row0 + i) * 3;
      for (int ch = 0; ch < 3; ++ch) {
        without_bg[r + ch] = wo[ch];
        with_bg[r + ch] = wb[ch];
        if (indirect) indirect[r + ch] = ind[ch];
      }
    }
  return TIR_OK;
}
