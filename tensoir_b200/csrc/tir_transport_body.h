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
