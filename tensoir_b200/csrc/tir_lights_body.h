// Per-slot and per-ray math of relighting under analytic lights (directional, point and spot lights; semantics in
// include/tensoir_b200.h).  Shared by the CUDA kernels (tir_lights.cu) and by a host build (tests/host_lights.cpp) that
// the CPU tests drive and the GPU tests compare with bit for bit.  The surface point, the cosine test, the GGX point
// context, one sample's contribution and the tone map are the environment-map pass's (tir_relight_body.h).
#pragma once
#include "tir_relight_body.h"

// slots before light j, for one ray: K_0 + ... + K_{j-1}; prefix[n_lights] is the slots of one ray
struct LightTable {
  TirLight l[TIR_LIGHTS_MAX];
  int32_t prefix[TIR_LIGHTS_MAX + 1];
};

// a light that is sampled at its centre and reads no uniform
RL_HD bool lt_centre_only(const TirLight& l) { return l.n_samples == 1 || !(l.extent > 0.f); }

// Concentric map of (u0, u1) in [0,1)^2 to the unit disc (Shirley & Chiu), in fp64, rounded once to fp32.  Written
// without a multiply feeding an add, so the device compiler has nothing to contract and both builds round alike.
RL_HD void lt_disc(double u0, double u1, float& x, float& y) {
  const double a = u0 + u0 - 1.0, b = u1 + u1 - 1.0;
  x = y = 0.f;
  if (a == 0.0 && b == 0.0) return;
  const double quarter_pi = 0.78539816339744830962;
  if (fabs(a) > fabs(b)) {
    const double phi = quarter_pi * (b / a);
    x = (float)(a * cos(phi));
    y = (float)(a * sin(phi));
  } else {                        // phi = pi/2 - pi/4 * a/b: cos and sin swap
    const double phi = quarter_pi * (a / b);
    x = (float)(b * sin(phi));
    y = (float)(b * cos(phi));
  }
}

// Two unit vectors orthogonal to the unit vector w and to each other (Duff et al., "Building an orthonormal basis,
// revisited")
RL_HD void lt_frame(const float w[3], float t1[3], float t2[3]) {
  const float s = copysignf(1.f, w[2]);
  const float a = ev_div(-1.f, ev_add(s, w[2]));
  const float b = ev_mul(ev_mul(w[0], w[1]), a);
  t1[0] = ev_add(1.f, ev_mul(ev_mul(s, ev_mul(w[0], w[0])), a));
  t1[1] = ev_mul(s, b);
  t1[2] = ev_mul(-s, w[0]);
  t2[0] = b;
  t2[1] = ev_add(s, ev_mul(ev_mul(w[1], w[1]), a));
  t2[2] = -w[1];
}

RL_HD float lt_dot(const float a[3], const float b[3]) {
  return ev_add(ev_add(ev_mul(a[0], b[0]), ev_mul(a[1], b[1])), ev_mul(a[2], b[2]));
}

// c + r * (x t1 + y t2), the point of the disc of radius r around c spanned by t1, t2
RL_HD void lt_on_disc(const float c[3], const float w[3], float r, float x, float y, float q[3]) {
  float t1[3], t2[3];
  lt_frame(w, t1, t2);
  for (int e = 0; e < 3; ++e) q[e] = ev_add(c[e], ev_mul(r, ev_add(ev_mul(x, t1[e]), ev_mul(y, t2[e]))));
}

// The sample of light l seen from the surface point p: unit direction L and falloff (see the header).  u is read only
// when the light has an extent and more than one sample.  dist2, when given, gets the squared distance from p to the
// sample of a point or spot light; it is left alone for a directional light.
RL_HD void lt_sample(const TirLight& l, const float p[3], const double* u, float L[3], float& falloff,
                     float* dist2 = nullptr) {
  float x = 0.f, y = 0.f;
  const bool centre = lt_centre_only(l);
  if (!centre) lt_disc(u[0], u[1], x, y);
  if (l.type == TIR_LIGHT_DIRECTIONAL) {
    falloff = 1.f;
    if (centre) {
      for (int e = 0; e < 3; ++e) L[e] = l.dir[e];
      return;
    }
    float q[3];
    lt_on_disc(l.dir, l.dir, l.extent, x, y, q);
    ev_normalize(q, L);
    return;
  }
  float q[3], w[3];
  for (int e = 0; e < 3; ++e) q[e] = l.pos[e];
  if (!centre) {
    float to[3];
    for (int e = 0; e < 3; ++e) to[e] = ev_sub(l.pos[e], p[e]);
    ev_normalize(to, w);
    lt_on_disc(l.pos, w, l.extent, x, y, q);
  }
  for (int e = 0; e < 3; ++e) w[e] = ev_sub(q[e], p[e]);
  const float d2 = lt_dot(w, w);
  if (dist2) *dist2 = d2;
  ev_normalize(w, L);
  float cone = 1.f;
  if (l.type == TIR_LIGHT_SPOT) {
    const float c = -lt_dot(L, l.dir);
    if (c >= l.cos_inner) cone = 1.f;
    else if (c <= l.cos_outer) cone = 0.f;
    else {
      const float t = ev_div(ev_sub(c, l.cos_outer), ev_sub(l.cos_inner, l.cos_outer));
      cone = ev_mul(ev_mul(t, t), ev_sub(3.f, ev_mul(2.f, t)));
    }
  }
  falloff = d2 > 0.f ? ev_div(cone, d2) : 0.f;
}

// One slot's contribution to its light's sum: rl_contrib with the falloff as the radiance and pdf 1
RL_HD void lt_contrib(const tir::PointCtx& c, const float L[3], float falloff, float vis, float acc[3]) {
  const float rgb[3] = {falloff, falloff, falloff};
  rl_contrib(c, L, rgb, 1.f, vis, acc);
}

// One output row from the sum over lights: without_bg, with_bg (acc threshold 0.9 as rl_composite) and linear
RL_HD void lt_finish(bool hit, float acc, const float lin[3], const float* background, float wo[3], float wb[3]) {
  const float acc_t = acc <= 0.9f ? 0.f : acc;
  for (int c = 0; c < 3; ++c) {
    wo[c] = hit ? tir::tone(lin[c], 1) : 1.f;
    wb[c] = ev_add(ev_mul(acc_t, wo[c]), ev_mul(ev_sub(1.f, acc_t), background[c]));
  }
}

// argument checks shared by the kernels and the host build: 1 run, 0 nothing to do, < 0 TirStatus.  Fills the table.
inline int lt_validate(const TirLight* lights, int32_t n_lights, int64_t n, LightTable& t) {
  if (n_lights < 0 || n < 0 || n_lights > TIR_LIGHTS_MAX) return TIR_ERR_SHAPE;
  if (n_lights > 0 && !lights) return TIR_ERR_NULL;
  t.prefix[0] = 0;
  for (int j = 0; j < n_lights; ++j) {
    const TirLight& l = lights[j];
    if (l.type != TIR_LIGHT_DIRECTIONAL && l.type != TIR_LIGHT_POINT && l.type != TIR_LIGHT_SPOT) return TIR_ERR_CONFIG;
    if (l.n_samples < 1 || l.n_samples > TIR_LIGHT_SAMPLES_MAX) return TIR_ERR_SHAPE;
    t.l[j] = l;
    t.prefix[j + 1] = t.prefix[j] + l.n_samples;
  }
  if (n_lights == 0 || n == 0) return 0;
  if (n * (int64_t)t.prefix[n_lights] > INT32_MAX) return TIR_ERR_SHAPE;
  return 1;
}

// The whole argument check of each entry, run by tir_lights.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus.  Fills the table.
inline int lt_sample_check(const TirLight* lights, int32_t n_lights, const float* rays, const float* depth,
                           const float* normal, const float* acc, int64_t n, const double* u, const float* L,
                           const float* falloff, const int32_t* pos, const float* list_o, const float* list_d,
                           int64_t capacity, const int64_t* count, LightTable& t) {
  const int rc = lt_validate(lights, n_lights, n, t);
  if (rc <= 0) return rc;
  if (!rays || !depth || !normal || !acc || !u || !L || !falloff || !pos || !count) return TIR_ERR_NULL;
  const int lrc = rl_check_list(capacity, list_o, list_d);
  return lrc ? lrc : 1;
}

inline int lt_shade_check(const TirLight* lights, int32_t n_lights, const float* rays, const float* normal,
                          const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                          const float* acc, int64_t n, const float* rescale, const float* background, const float* L,
                          const float* falloff, const int32_t* pos, const float* vis_list, int32_t vis_kind,
                          const float* with_bg, const float* without_bg, int64_t out_rows, int64_t row0,
                          LightTable& t) {
  const int rc = lt_validate(lights, n_lights, n, t);
  if (rc <= 0) return rc;
  if (!rays || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !background || !L || !falloff || !pos ||
      !vis_list || !with_bg || !without_bg)
    return TIR_ERR_NULL;
  const int wrc = rl_check_window(rough_stride, vis_kind, n, out_rows, row0);
  return wrc ? wrc : 1;
}
