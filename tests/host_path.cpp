// Host twin of csrc/tir_path.cu for the tests of tensoir_b200/camera_path.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (pt_sample_check, pt_composite_check) and per-slot /
// per-pixel math of csrc/tir_path_body.h, with plain loops instead of kernels.  "Device" pointers are host pointers
// here.  The visibility list is filled in slot order.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_path_body.h"

extern "C" int tir_ground_sample(const TirEnvMap* envs, int32_t n_lights, const float* rays, int64_t n,
                                 float ground_z, const float* box_lo, const float* box_hi, int32_t n_samples,
                                 const double* u, int32_t* bin, int32_t* pos, float* list_o, float* list_d,
                                 int64_t capacity, int64_t* count, void*) {
  const int rc = pt_sample_check(envs, n_lights, rays, n, box_lo, box_hi, n_samples, u, bin, pos, list_o, list_d,
                                 capacity, count);
  if (rc <= 0) return rc;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t i = 0; i < n; ++i)
      for (int s = 0; s < n_samples; ++s) {
        const int64_t t = ((int64_t)l * n + i) * n_samples + s;
        bin[t] = 0;
        pos[t] = -1;
        float g[3];
        if (!pt_ground(rays + i * 6, ground_z, g)) continue;
        const TirEnvMap& e = envs[l];
        const int b = rl_bin(e.cdf, e.H * e.W, u[t]);
        bin[t] = b;
        const float w[3] = {e.dir[b * 3], e.dir[b * 3 + 1], e.dir[b * 3 + 2]};
        float o[3];
        const int q = pt_ground_slot(g, w, box_lo, box_hi, o);
        if (q < 0) { pos[t] = q; continue; }
        const int64_t row = (*count)++;
        if (row >= capacity) continue;
        for (int c = 0; c < 3; ++c) { list_o[row * 3 + c] = o[c]; list_d[row * 3 + c] = w[c]; }
        pos[t] = (int32_t)row;
      }
  return TIR_OK;
}

extern "C" int tir_path_composite(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* acc,
                                  int64_t n, const float* rot, float ground_z, const int32_t* bin, const int32_t* pos,
                                  const float* vis_list, int32_t vis_kind, int32_t n_samples, const float* without_bg,
                                  float* with_bg, float* shadow, int64_t out_rows, int64_t row0, void*) {
  const int rc = pt_composite_check(envs, n_lights, rays, acc, n, rot, ground_z, bin, pos, vis_list, vis_kind,
                                    n_samples, without_bg, with_bg, out_rows, row0);
  if (rc <= 0) return rc;
  for (int l = 0; l < n_lights; ++l)
    for (int64_t i = 0; i < n; ++i) {
      const TirEnvMap& e = envs[l];
      const float* ray = rays + i * 6;
      float r[3] = {1.f, 1.f, 1.f};
      float g[3];
      if (pt_ground(ray, ground_z, g)) {
        // the kernel's order: lane k sums slots k, k+32, ...; then the xor butterfly over the 32 lanes
        float num[32][3] = {}, den[32][3] = {};
        const int64_t k0 = ((int64_t)l * n + i) * n_samples;
        for (int k = 0; k < 32; ++k)
          pt_shadow_lane(e, bin + k0, pos + k0, vis_list, vis_kind, n_samples, k, 32, num[k], den[k]);
        for (int o = 16; o > 0; o >>= 1) {
          float nn[32][3], nd[32][3];
          for (int k = 0; k < 32; ++k)
            for (int c = 0; c < 3; ++c) {
              nn[k][c] = num[k][c] + num[k ^ o][c];
              nd[k][c] = den[k][c] + den[k ^ o][c];
            }
          for (int k = 0; k < 32; ++k)
            for (int c = 0; c < 3; ++c) { num[k][c] = nn[k][c]; den[k][c] = nd[k][c]; }
        }
        for (int c = 0; c < 3; ++c) r[c] = pt_ratio(num[0][c], den[0][c]);
      }
      const int64_t row = ((int64_t)l * out_rows + row0 + i) * 3;
      float wb[3];
      pt_composite(e, ray, rot, acc[i], without_bg + row, r, wb);
      for (int c = 0; c < 3; ++c) {
        with_bg[row + c] = wb[c];
        if (shadow) shadow[row + c] = r[c];
      }
    }
  return TIR_OK;
}
