// Host twin of csrc/tir_edit.cu for the CPU tests of tensoir_b200/editing.py: the SAME C-ABI signature
// (include/tensoir_b200.h), the library's own argument check (ed_validate) and per-point math of csrc/tir_edit_body.h,
// with a loop instead of a kernel.  "Device" pointers are host pointers here.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_edit_body.h"

extern "C" int tir_material_edit(const TirEditRule* rules, int32_t n_rules, const float* rays, const float* depth,
                                 const float* points, const float* albedo, const float* rough, int32_t rough_stride,
                                 const float* fresnel, const float* acc, int64_t n, float acc_threshold,
                                 const float* scale, float* albedo_out, float* rough_out, float* fresnel_out,
                                 int32_t* sel, void*) {
  const int rc = ed_validate(rules, n_rules, rays, depth, points, albedo, rough, rough_stride, fresnel, acc, n, scale,
                             albedo_out, rough_out, fresnel_out, sel);
  if (rc <= 0) return rc;
  const int rs = rough_stride;
  for (int64_t i = 0; i < n; ++i) {
    float pt[3];
    if (points)
      for (int c = 0; c < 3; ++c) pt[c] = points[i * 3 + c];
    else
      rl_surface(rays + i * 6, depth[i], pt);
    ed_row(rules, n_rules, pt, albedo + i * 3, rough + i * rs, rs, fresnel + i * 3, acc[i] > acc_threshold, scale,
           albedo_out + i * 3, rough_out + i * rs, fresnel_out + i * 3, sel + i);
  }
  return TIR_OK;
}
