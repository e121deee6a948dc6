// Per-(hit, texel) math of the light transport to an environment map's texels (semantics in include/tensoir_b200.h).
// Shared by the CUDA kernels (tir_transport.cu) and by a host build (tests/host_transport.cpp) that the CPU tests drive
// and the GPU tests compare with.  The surface point, the cosine test, the GGX point context and one sample's term are
// the environment-map pass's (tir_relight_body.h).
#pragma once
#include "tir_relight_body.h"

// One texel's transport, per channel: rl_contrib with the solid angle as the radiance and pdf 1
RL_HD void tt_contrib(const tir::PointCtx& c, const float L[3], float domega, float vis, float out[3]) {
  const float rgb[3] = {domega, domega, domega};
  out[0] = out[1] = out[2] = 0.f;
  rl_contrib(c, L, rgb, 1.f, vis, out);
}

// argument checks shared by the kernels and the host build: 1 run, 0 nothing to do, < 0 TirStatus
inline int tt_validate(int32_t K, int64_t n) {
  if (K < 1 || K > TIR_TRANSPORT_MAX_TEXELS || n < 0) return TIR_ERR_SHAPE;
  if (n * (int64_t)K > INT32_MAX) return TIR_ERR_SHAPE;
  return n == 0 ? 0 : 1;
}

// The whole argument check of each entry, run by tir_transport.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus
inline int tt_sample_check(const float* dirs, int32_t K, const float* rays, const float* depth, const float* normal,
                           const float* acc, int64_t n, const int32_t* pos, const float* list_o, const float* list_d,
                           int64_t capacity, const int64_t* count) {
  const int rc = tt_validate(K, n);
  if (rc <= 0) return rc;
  if (!dirs || !rays || !depth || !normal || !acc || !pos || !count) return TIR_ERR_NULL;
  const int lrc = rl_check_list(capacity, list_o, list_d);
  return lrc ? lrc : 1;
}

// T covers all n rows, so the window is [0, n)
inline int tt_build_check(const float* dirs, const float* domega, int32_t K, const float* rays, const float* normal,
                          const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                          const float* acc, int64_t n, const float* rescale, const int32_t* pos,
                          const float* vis_list, int32_t vis_kind, const float* T) {
  const int rc = tt_validate(K, n);
  if (rc <= 0) return rc;
  if (!dirs || !domega || !rays || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !pos ||
      !vis_list || !T)
    return TIR_ERR_NULL;
  const int wrc = rl_check_window(rough_stride, vis_kind, n, n, 0);
  return wrc ? wrc : 1;
}
