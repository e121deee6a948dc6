// Per-slot and per-hit math of relighting with one bounce of indirect light under environment maps.  Shared by the CUDA
// kernels (tir_indirect.cu) and by a host build (tests/host_indirect.cpp) that the CPU tests drive and the GPU tests
// compare with.  The estimator, for a hit primary ray i (acc > acc_mask_threshold) and map l:
//
//   linear[l,i] = (1/S)  * sum_s direct_s                  (exactly tir_relight_shade's sum, same order, same bits)
//               + (1/K)  * sum_k T[i,k] * w[i,k] * Lo[l, h(i,k)]
//   without_bg  = tone(linear),  with_bg = rl_composite(...)  (as tir_relight_shade)
//
// Direction: slot k of ray i draws u[i,k,0:2], takes (x, y) = lt_disc(u), z = sqrt(max(0, 1 - x^2 - y^2)) and
// omega = x t1 + y t2 + z n^ with n^ = normal / |normal| and (t1, t2) = lt_frame(n^): cosine-weighted hemisphere
// sampling (Malley's method), pdf = z / pi.
// Throughput: T[i,k,c] = (albedo_c * rescale_c / pi + GGX_c(omega)) * cosr / pdf, cosr = omega . normal with the raw
// normal; rl_contrib's term with vis * rgb = 1 and pdf z / pi.  A slot is not marched (T = 0) when cosr <= 1e-6 (the
// direct samples' cosine test) or z <= 1e-6.
// Secondary march: from p = rl_surface(ray, depth), the direct samples' origin, along omega through tir_march_density
// with relight()'s own table (96 samples over [0.05, 1.5]).  An occluder in that range is counted by the direct term
// through vis and by the indirect term through w, so the energy split is consistent by construction.
// Occlusion weight: w = 1 - vis, vis as relight() reads it (t_last for nerv, 1 - acc for nerfactor).  The slot is a
// secondary hit when w > 1e-3 and acc > 0, at x = p + (depth / acc) * omega (depth = the march's sum w z).  A slot with
// w <= 1e-3 contributes 0: the bias this leaves is at most 1e-3 * T * max Lo per slot.
// Secondary radiance: Lo[l,h] = (1/S2) * sum of rl_contrib over S2 importance samples of map l at x with view direction
// -omega, visibility marched from x: direct light only (one bounce), un-toned and unclamped.
#pragma once
#include "tir_lights_body.h"

#define TIR_INDIRECT_HIT_W 1e-3f

// Direction of one slot from its two uniforms: omega and z = pi * pdf
RL_HD void ind_direction(const float normal[3], const double* u, float omega[3], float& z) {
  float nh[3], t1[3], t2[3], x, y;
  ev_normalize(normal, nh);
  lt_frame(nh, t1, t2);
  lt_disc(u[0], u[1], x, y);
  const float zz = ev_sub(ev_sub(1.f, ev_mul(x, x)), ev_mul(y, y));
  z = sqrtf(zz > 0.f ? zz : 0.f);
  for (int e = 0; e < 3; ++e) omega[e] = ev_add(ev_add(ev_mul(x, t1[e]), ev_mul(y, t2[e])), ev_mul(z, nh[e]));
}

// Throughput of one slot into T[3]; false (T = 0) when the slot fails the cosine or z test and is not marched
RL_HD bool ind_throughput(const tir::PointCtx& c, const float omega[3], float z, float T[3]) {
  T[0] = T[1] = T[2] = 0.f;
  if (!(rl_cosine(omega, c.n) > 1e-6f) || !(z > 1e-6f)) return false;
  const float rgb[3] = {1.f, 1.f, 1.f};
  rl_contrib(c, omega, rgb, ev_div(z, tir::kPi), 1.f, T);
  return true;
}

// Occlusion weight of a marched slot and whether it is a secondary hit
RL_HD float ind_weight(int vis_kind, float t_last, float acc) {
  const float vis = vis_kind ? 1.f - acc : t_last;
  return 1.f - vis;
}
RL_HD bool ind_is_hit(float w, float acc) { return w > TIR_INDIRECT_HIT_W && acc > 0.f; }

// The secondary hit point x = p + (depth / acc) * omega and its aabb-normalised coordinate (x - lo) * inv - 1
RL_HD void ind_point(const float p[3], const float omega[3], float depth, float acc, const float* aabb, float x[3],
                     float xn[3]) {
  const float t = ev_div(depth, acc);
  for (int e = 0; e < 3; ++e) {
    x[e] = ev_add(p[e], ev_mul(t, omega[e]));
    xn[e] = ev_sub(ev_mul(ev_sub(x[e], aabb[e]), aabb[3 + e]), 1.f);
  }
}

// One slot's indirect term T * w * Lo, added to acc[3]
RL_HD void ind_add(const float T[3], float w, const float Lo[3], float acc[3]) {
  for (int c = 0; c < 3; ++c) acc[c] = ev_add(acc[c], ev_mul(ev_mul(T[c], w), Lo[c]));
}

// argument checks shared by the kernels and the host build
inline int ind_check_slots(int64_t n, int32_t K) {
  if (n < 0 || K < 1 || K > 1024) return TIR_ERR_SHAPE;
  if (n * (int64_t)K > INT32_MAX) return TIR_ERR_SHAPE;
  return 1;
}
inline int ind_check_samples(int32_t S2) { return (S2 < 1 || S2 > 1024) ? TIR_ERR_SHAPE : 1; }

// The whole argument check of each entry, run by tir_indirect.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus
inline int ind_sample_check(const float* rays, const float* depth, const float* normal, const float* albedo,
                            const float* rough, int32_t rough_stride, const float* fresnel, const float* acc, int64_t n,
                            int32_t K, const float* rescale, const double* u, const float* dir, const float* T,
                            const int32_t* pos, const float* list_o, const float* list_d, int64_t capacity,
                            const int64_t* count) {
  const int rc = ind_check_slots(n, K);
  if (rc <= 0) return rc;
  if (!rays || !depth || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !u || !dir || !T || !pos ||
      !count)
    return TIR_ERR_NULL;
  if (rough_stride != 1 && rough_stride != 3) return TIR_ERR_SHAPE;
  const int lrc = rl_check_list(capacity, list_o, list_d);
  if (lrc) return lrc;
  return n == 0 ? 0 : 1;
}

inline int ind_hits_work_size_check(int64_t n, int32_t K, const int64_t* bytes) {
  if (!bytes) return TIR_ERR_NULL;
  return ind_check_slots(n, K);
}

// 0 (n == 0): the caller only zeroes *count
inline int ind_hits_check(int64_t n, int32_t K, const int32_t* pos, const float* list_o, const float* list_d,
                          const float* t_last, const float* acc, const float* depth, int32_t vis_kind,
                          const float* aabb, const float* hit_rays, const float* xn, const float* w, const int32_t* hit,
                          int64_t capacity, const int64_t* count) {
  const int rc = ind_check_slots(n, K);
  if (rc <= 0) return rc;
  if (!pos || !aabb || !hit || !count) return TIR_ERR_NULL;
  if (vis_kind != 0 && vis_kind != 1) return TIR_ERR_CONFIG;
  if (capacity < 0 || capacity > INT32_MAX) return TIR_ERR_SHAPE;
  if (capacity > 0 && (!hit_rays || !xn || !w)) return TIR_ERR_NULL;
  if (n == 0) return 0;
  // an empty secondary list has no march outputs: every slot then has pos -1 and they are never read
  if (!list_o || !list_d || !t_last || !acc || !depth) return TIR_ERR_NULL;
  return 1;
}

inline int ind_radiance_check(const TirEnvMap* envs, int32_t n_lights, const float* hit_rays, const float* normal,
                              const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                              int64_t m, int32_t n_samples, const float* rescale, const int32_t* bin,
                              const int32_t* pos, const float* vis_list, int32_t vis_kind, const float* Lo,
                              int64_t out_rows, int64_t row0) {
  const int rc = rl_validate(envs, n_lights, m, n_samples);
  if (rc < 0) return rc;
  if (ind_check_samples(n_samples) < 0) return TIR_ERR_SHAPE;
  if (!hit_rays || !normal || !albedo || !rough || !fresnel || !rescale || !bin || !pos || !vis_list || !Lo)
    return TIR_ERR_NULL;
  const int wrc = rl_check_window(rough_stride, vis_kind, m, out_rows, row0);
  if (wrc) return wrc;
  if (m > INT32_MAX) return TIR_ERR_SHAPE;
  return rc;
}

inline int ind_shade_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                           const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                           const float* acc, int64_t n, int32_t n_samples, const float* rescale, const int32_t* bin,
                           const int32_t* pos, int32_t vis_kind, int32_t K, const float* T, const int32_t* hit,
                           const float* w, const float* Lo, int64_t m_h, const float* with_bg,
                           const float* without_bg, int64_t out_rows, int64_t row0) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc < 0) return rc;
  if (n_samples <= 0 || ind_check_slots(n, K) < 0 || m_h < 0 || m_h > INT32_MAX) return TIR_ERR_SHAPE;
  if (!rays || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !bin || !pos || !T || !hit ||
      !with_bg || !without_bg)
    return TIR_ERR_NULL;
  if (m_h > 0 && (!w || !Lo)) return TIR_ERR_NULL;
  const int wrc = rl_check_window(rough_stride, vis_kind, n, out_rows, row0);
  return wrc ? wrc : rc;
}
