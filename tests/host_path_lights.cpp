// Host twin of the analytic-light ground entries of csrc/tir_path.cu for the tests of tensoir_b200/camera_path.py: the
// SAME C-ABI signatures (include/tensoir_b200.h), the library's own argument checks (pt_lights_sample_check,
// pt_lights_composite_check) and per-slot / per-pixel math of csrc/tir_path_body.h, with plain loops instead of
// kernels.  "Device" pointers are host pointers here.  The visibility list is filled in slot order.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_path_body.h"

extern "C" int tir_ground_lights_sample(const TirLight* lights, int32_t n_lights, const float* rays, int64_t n,
                                        float ground_z, const float* box_lo, const float* box_hi, const double* u,
                                        float* g, int32_t* pos, float* list_o, float* list_d, int64_t capacity,
                                        int64_t* count, void*) {
  LightTable lt;
  const int rc = pt_lights_sample_check(lights, n_lights, rays, n, box_lo, box_hi, u, g, pos, list_o, list_d, capacity,
                                        count, lt);
  if (rc <= 0) return rc;
  for (int j = 0; j < n_lights; ++j)
    for (int64_t i = 0; i < n; ++i)
      for (int s = 0; s < lt.l[j].n_samples; ++s) {
        const int64_t t = n * lt.prefix[j] + i * lt.l[j].n_samples + s;
        g[t] = 0.f;
        pos[t] = -1;
        float p[3];
        if (!pt_ground(rays + i * 6, ground_z, p)) continue;
        float L[3], fall, d2 = INFINITY, o[3];
        lt_sample(lt.l[j], p, u + t * 2, L, fall, &d2);
        g[t] = ev_mul(fall, L[2]);
        const int q = pt_light_slot(lt.l[j], p, L, g[t], d2, box_lo, box_hi, o);
        if (q < 0) { pos[t] = q; continue; }
        const int64_t row = (*count)++;
        if (row >= capacity) continue;
        for (int c = 0; c < 3; ++c) { list_o[row * 3 + c] = o[c]; list_d[row * 3 + c] = L[c]; }
        pos[t] = (int32_t)row;
      }
  return TIR_OK;
}

// the kernel's order for one light: lane k sums slots k, k+32, ...; then the xor butterfly over the 32 lanes
static void butterfly(float v[32]) {
  for (int o = 16; o > 0; o >>= 1) {
    float nxt[32];
    for (int k = 0; k < 32; ++k) nxt[k] = v[k] + v[k ^ o];
    for (int k = 0; k < 32; ++k) v[k] = nxt[k];
  }
}

extern "C" int tir_path_lights_composite(const TirLight* lights, int32_t n_lights, const float* rays, const float* acc,
                                         int64_t n, float ground_z, const float* background,
                                         const float* background_linear, const float* g, const int32_t* pos,
                                         const float* vis_list, int32_t vis_kind, const float* without_bg,
                                         float* with_bg, float* shadow, int64_t out_rows, int64_t row0, void*) {
  LightTable lt;
  const int rc = pt_lights_composite_check(lights, n_lights, rays, acc, n, ground_z, background, background_linear, g,
                                           pos, vis_list, vis_kind, without_bg, with_bg, out_rows, row0, lt);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i) {
    float r[3] = {1.f, 1.f, 1.f};
    float p[3];
    if (pt_ground(rays + i * 6, ground_z, p)) {
      float num[3] = {0.f, 0.f, 0.f}, den[3] = {0.f, 0.f, 0.f};
      for (int j = 0; j < n_lights; ++j) {
        const int K = lt.l[j].n_samples;
        const int64_t k0 = n * lt.prefix[j] + i * K;
        float sn[32] = {}, sd[32] = {};
        for (int k = 0; k < 32; ++k) pt_light_lane(g + k0, pos + k0, vis_list, vis_kind, K, k, 32, sn[k], sd[k]);
        butterfly(sn);
        butterfly(sd);
        pt_light_add(lt.l[j], K, sn[0], sd[0], num, den);
      }
      for (int c = 0; c < 3; ++c) r[c] = pt_ratio(num[c], den[c]);
    }
    const int64_t row = (row0 + i) * 3;
    float wb[3];
    pt_lights_composite(background, background_linear, acc[i], without_bg + row, r, wb);
    for (int c = 0; c < 3; ++c) {
      with_bg[row + c] = wb[c];
      if (shadow) shadow[row + c] = r[c];
    }
  }
  return TIR_OK;
}
