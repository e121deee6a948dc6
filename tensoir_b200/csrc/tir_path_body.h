// Per-slot and per-pixel math of camera-path frames: the shadow-catching ground plane and the frame composite under a
// rotated environment map (semantics in include/tensoir_b200.h, "camera-path frames").  Shared by the CUDA kernels
// (tir_path.cu) and by a host build (tests/host_path.cpp) that the CPU tests drive and the GPU tests compare with.  The
// inverse-CDF bin, the background lookup, the visibility read and the tone map are the environment-map pass's
// (tir_relight_body.h).  The ground under analytic lights takes its light samples from tir_lights_body.h.
#pragma once
#include "tir_lights_body.h"
#include "tir_relight_body.h"

// The ground point of a primary ray (o, d): p = o + t d on the plane z = ground_z, when d.z < 0 and t > 0.  A NaN
// ground_z (no ground) gives no point.  p.z is ground_z itself, so every point lies on the plane exactly.
RL_HD bool pt_ground(const float* ray, float ground_z, float p[3]) {
  const float dz = ray[5];
  if (!(dz < 0.f)) return false;
  const float t = ev_div(ev_sub(ground_z, ray[2]), dz);
  if (!(t > 0.f)) return false;
  p[0] = ev_add(ray[0], ev_mul(t, ray[3]));
  p[1] = ev_add(ray[1], ev_mul(t, ray[4]));
  p[2] = ground_z;
  return true;
}

// Slab test of the ray p + t w, t >= 0, against the box [lo, hi]: true, with the entry parameter t_enter >= 0, when the
// ray meets the box.  A box with lo > hi on some axis is empty and is never met.
RL_HD bool pt_slab(const float p[3], const float w[3], const float lo[3], const float hi[3], float& t_enter) {
  float tn = 0.f, tf = INFINITY;
  for (int a = 0; a < 3; ++a) {
    if (!(lo[a] <= hi[a])) return false;
    if (w[a] != 0.f) {
      const float t0 = ev_div(ev_sub(lo[a], p[a]), w[a]), t1 = ev_div(ev_sub(hi[a], p[a]), w[a]);
      tn = fmaxf(tn, fminf(t0, t1));
      tf = fminf(tf, fmaxf(t0, t1));
    } else if (p[a] < lo[a] || p[a] > hi[a]) {
      return false;
    }
  }
  if (!(tn <= tf)) return false;
  t_enter = tn;
  return true;
}

// One ground slot: from the ground point p, the direction w = dir[bin] of the map's (rotated) table.  -> -1 when
// w.z <= 1e-6 (below the horizon of the +z normal: the slot counts nowhere), -2 when the shadow ray p + t w misses the
// box (unoccluded, not marched), 0 when it meets the box; then o is the shadow ray's origin, moved along w to
// TIR_PATH_SHADOW_NEAR before the box entry so that the march's first sample lands on the entry.
RL_HD int pt_ground_slot(const float p[3], const float w[3], const float lo[3], const float hi[3], float o[3]) {
  if (!(w[2] > 1e-6f)) return -1;
  float te;
  if (!pt_slab(p, w, lo, hi, te)) return -2;
  const float s = fmaxf(ev_sub(te, TIR_PATH_SHADOW_NEAR), 0.f);
  for (int c = 0; c < 3; ++c) o[c] = ev_add(p[c], ev_mul(s, w[c]));
  return 0;
}

// Row vector d times the row-major 3x3 rot: (d @ R)_j = sum_i d_i R[i][j]
RL_HD void pt_rotate(const float d[3], const float* rot, float out[3]) {
  for (int j = 0; j < 3; ++j)
    out[j] = ev_add(ev_add(ev_mul(d[0], rot[j]), ev_mul(d[1], rot[3 + j])), ev_mul(d[2], rot[6 + j]));
}

// The ground's per-slot sums of one (map, ground point): lane `lane` of `lanes` adds slots lane, lane + lanes, ... with
// pos != -1 to num[c] += E_c cos V / pdf and den[c] += E_c cos / pdf, cos = w.z, V = 1 for pos -2 and the march's
// visibility for pos >= 0.  The kernels run it on the 32 lanes of a warp and reduce with warp_sum; the host build runs
// the 32 lanes in turn and reduces with the same xor butterfly.
RL_HD void pt_shadow_lane(const TirEnvMap& e, const int32_t* bin, const int32_t* pos, const float* vis_list,
                          int vis_kind, int S, int lane, int lanes, float num[3], float den[3]) {
  for (int s = lane; s < S; s += lanes) {
    const int q = pos[s];
    if (q == -1) continue;
    const int64_t b = bin[s];
    const float v = q >= 0 ? rl_vis(vis_list, vis_kind, q) : 1.f;
    const float w = ev_div(RL_LDG(e.dir + b * 3 + 2), RL_LDG(e.pdf_return + b));
    for (int c = 0; c < 3; ++c) {
      const float ew = ev_mul(RL_LDG(e.rgb + b * 3 + c), w);
      num[c] = ev_add(num[c], ev_mul(ew, v));
      den[c] = ev_add(den[c], ew);
    }
  }
}

// The shadow ratio from the reduced sums: num / den clamped to [0, 1], 1 where den is 0
RL_HD float pt_ratio(float num, float den) {
  if (!(den > 0.f)) return 1.f;
  const float r = ev_div(num, den);
  return r < 0.f ? 0.f : (r > 1.f ? 1.f : r);
}

// One output row of the frame: the background looked up at d @ rot, times the shadow ratio r per channel, composited
// under the object with rl_composite's expression.
RL_HD void pt_composite(const TirEnvMap& e, const float* ray, const float* rot, float acc, const float wo[3],
                        const float r[3], float with_bg[3]) {
  float d[3], bg[3];
  pt_rotate(ray + 3, rot, d);
  rl_background(e, d, bg);
  const float acc_t = acc <= 0.9f ? 0.f : acc;
  for (int c = 0; c < 3; ++c)
    with_bg[c] = ev_add(ev_mul(acc_t, wo[c]), ev_mul(ev_sub(1.f, acc_t), tir::tone(ev_mul(bg[c], r[c]), 1)));
}

// ---- the ground under analytic lights ----

// One ground slot of light l: from the ground point p, the light sample's direction L, its weight g = falloff * L.z
// and, for a point or spot light, the squared distance d2 from p to the sample.  -> -1 when L.z <= 1e-6 or g <= 0
// (counts nowhere), -2 when the shadow ray p + t L misses the box or, for a point or spot light, enters it at or beyond
// the light sample (unoccluded, not marched), 0 when it is marched from o, as pt_ground_slot.
RL_HD int pt_light_slot(const TirLight& l, const float p[3], const float L[3], float g, float d2, const float lo[3],
                        const float hi[3], float o[3]) {
  if (!(L[2] > 1e-6f) || !(g > 0.f)) return -1;
  float te;
  if (!pt_slab(p, L, lo, hi, te)) return -2;
  if (l.type != TIR_LIGHT_DIRECTIONAL && te >= sqrtf(d2)) return -2;
  const float s = fmaxf(ev_sub(te, TIR_PATH_SHADOW_NEAR), 0.f);
  for (int c = 0; c < 3; ++c) o[c] = ev_add(p[c], ev_mul(s, L[c]));
  return 0;
}

// The ground's per-slot sums of one (light, ground point) over its K slots: lane `lane` of `lanes` adds slots lane,
// lane + lanes, ... with pos != -1 to num += g V and den += g, V = 1 for pos -2 and the march's visibility for rows.
// Reduced as pt_shadow_lane's sums are.
RL_HD void pt_light_lane(const float* g, const int32_t* pos, const float* vis_list, int vis_kind, int K, int lane,
                         int lanes, float& num, float& den) {
  for (int s = lane; s < K; s += lanes) {
    const int q = pos[s];
    if (q == -1) continue;
    const float v = q >= 0 ? rl_vis(vis_list, vis_kind, q) : 1.f;
    num = ev_add(num, ev_mul(g[s], v));
    den = ev_add(den, g[s]);
  }
}

// One light's reduced sums added to the ratio's per-channel sums: power_c times the mean over its K slots, the same
// expression for both, so that num == den when every V is 1
RL_HD void pt_light_add(const TirLight& l, int K, float sn, float sd, float num[3], float den[3]) {
  for (int c = 0; c < 3; ++c) {
    num[c] = ev_add(num[c], ev_mul(l.power[c], ev_div(sn, (float)K)));
    den[c] = ev_add(den[c], ev_mul(l.power[c], ev_div(sd, (float)K)));
  }
}

// One output row under a setup of lights: the setup's display background where the ratio is 1, else the linear
// background times r, tone-mapped; composited under the object with lt_finish's expression
RL_HD void pt_lights_composite(const float* background, const float* background_linear, float acc, const float wo[3],
                               const float r[3], float with_bg[3]) {
  const float acc_t = acc <= 0.9f ? 0.f : acc;
  for (int c = 0; c < 3; ++c) {
    const float bg = r[c] == 1.f ? background[c] : tir::tone(ev_mul(background_linear[c], r[c]), 1);
    with_bg[c] = ev_add(ev_mul(acc_t, wo[c]), ev_mul(ev_sub(1.f, acc_t), bg));
  }
}

// The whole argument check of each entry, run by tir_path.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus.  The lights' checks also fill the table.
inline int pt_lights_sample_check(const TirLight* lights, int32_t n_lights, const float* rays, int64_t n,
                                  const float* box_lo, const float* box_hi, const double* u, const float* g,
                                  const int32_t* pos, const float* list_o, const float* list_d, int64_t capacity,
                                  const int64_t* count, LightTable& t) {
  const int rc = lt_validate(lights, n_lights, n, t);
  if (rc <= 0) return rc;
  if (!rays || !box_lo || !box_hi || !u || !g || !pos || !count) return TIR_ERR_NULL;
  const int lrc = rl_check_list(capacity, list_o, list_d);
  return lrc ? lrc : 1;
}

inline int pt_lights_composite_check(const TirLight* lights, int32_t n_lights, const float* rays, const float* acc,
                                     int64_t n, float ground_z, const float* background,
                                     const float* background_linear, const float* g, const int32_t* pos,
                                     const float* vis_list, int32_t vis_kind, const float* without_bg,
                                     const float* with_bg, int64_t out_rows, int64_t row0, LightTable& t) {
  const int rc = lt_validate(lights, n_lights, n, t);
  if (rc <= 0) return rc;
  if (!rays || !acc || !background || !background_linear || !without_bg || !with_bg) return TIR_ERR_NULL;
  if (!isnan(ground_z) && (!g || !pos || !vis_list)) return TIR_ERR_NULL;
  const int wrc = rl_check_window(1, vis_kind, n, out_rows, row0);
  return wrc ? wrc : 1;
}

inline int pt_sample_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, int64_t n,
                           const float* box_lo, const float* box_hi, int32_t n_samples, const double* u,
                           const int32_t* bin, const int32_t* pos, const float* list_o, const float* list_d,
                           int64_t capacity, const int64_t* count) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc <= 0 || n_samples == 0) return rc < 0 ? rc : 0;
  if (!rays || !box_lo || !box_hi || !u || !bin || !pos || !count) return TIR_ERR_NULL;
  const int lrc = rl_check_list(capacity, list_o, list_d);
  return lrc ? lrc : 1;
}

inline int pt_composite_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* acc, int64_t n,
                              const float* rot, float ground_z, const int32_t* bin, const int32_t* pos,
                              const float* vis_list, int32_t vis_kind, int32_t n_samples, const float* without_bg,
                              const float* with_bg, int64_t out_rows, int64_t row0) {
  const int rc = rl_validate(envs, n_lights, n, n_samples);
  if (rc <= 0) return rc;
  if (!rays || !acc || !rot || !without_bg || !with_bg) return TIR_ERR_NULL;
  const bool ground = !isnan(ground_z);
  if (ground && n_samples <= 0) return TIR_ERR_SHAPE;
  if (ground && (!bin || !pos || !vis_list)) return TIR_ERR_NULL;
  const int wrc = rl_check_window(1, vis_kind, n, out_rows, row0);
  return wrc ? wrc : 1;
}
