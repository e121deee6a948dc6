// Material editing of n surface points (tir_material_edit, include/tensoir_b200.h): one thread per point, the rule
// table passed by value in the kernel parameters, the per-point math in tir_edit_body.h.  It runs between the
// relighting pass's visibility march and its shading, so that several edited materials share one march.
#include "tir_device.cuh"
#include "tir_edit_body.h"

namespace {

constexpr int kThreads = 256;

struct EditParams {
  TirEditRule rules[TIR_EDIT_MAX_RULES];
  int n_rules;
  const float* rays; const float* depth; const float* points;
  const float* albedo; const float* rough; int rough_stride; const float* fresnel; const float* acc;
  int64_t n; float thr;
  const float* scale;
  float* albedo_out; float* rough_out; float* fresnel_out; int32_t* sel;
};

__global__ void __launch_bounds__(kThreads) material_edit_kernel(const EditParams p) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= p.n) return;
  float pt[3];
  if (p.points) {
#pragma unroll
    for (int c = 0; c < 3; ++c) pt[c] = p.points[i * 3 + c];
  } else {
    rl_surface(p.rays + i * 6, p.depth[i], pt);
  }
  const float scale[3] = {__ldg(p.scale), __ldg(p.scale + 1), __ldg(p.scale + 2)};
  const int rs = p.rough_stride;
  ed_row(p.rules, p.n_rules, pt, p.albedo + i * 3, p.rough + i * rs, rs, p.fresnel + i * 3, p.acc[i] > p.thr, scale,
         p.albedo_out + i * 3, p.rough_out + i * rs, p.fresnel_out + i * 3, p.sel + i);
}

}  // namespace

extern "C" int tir_material_edit(const TirEditRule* rules, int32_t n_rules, const float* rays, const float* depth,
                                 const float* points, const float* albedo, const float* rough, int32_t rough_stride,
                                 const float* fresnel, const float* acc, int64_t n, float acc_threshold,
                                 const float* scale, float* albedo_out, float* rough_out, float* fresnel_out,
                                 int32_t* sel, void* stream) {
  const int rc = ed_validate(rules, n_rules, rays, depth, points, albedo, rough, rough_stride, fresnel, acc, n, scale,
                             albedo_out, rough_out, fresnel_out, sel);
  if (rc <= 0) return rc;
  EditParams p{};
  for (int k = 0; k < n_rules; ++k) p.rules[k] = rules[k];
  p.n_rules = n_rules;
  p.rays = rays; p.depth = depth; p.points = points;
  p.albedo = albedo; p.rough = rough; p.rough_stride = rough_stride; p.fresnel = fresnel; p.acc = acc;
  p.n = n; p.thr = acc_threshold; p.scale = scale;
  p.albedo_out = albedo_out; p.rough_out = rough_out; p.fresnel_out = fresnel_out; p.sel = sel;
  material_edit_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}
