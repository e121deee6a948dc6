// Per-sample math of relighting under environment maps with multiple importance sampling (MIS).  Shared by the CUDA
// kernels (tir_relight_mis.cu) and by a host build (tests/host_mis.cpp) that the CPU tests drive and the GPU tests
// compare with.  For a hit primary ray i (acc > acc_mask_threshold) and map l the estimate is
//
//   linear[l,i] = sum over the S_l light samples of map l and the S_b BRDF samples of ray i of
//                 f(w) * V(w) * E_l(w) * cos(w) / (S_l * p_light_l(w) + S_b * p_brdf(w))
//
// of Lo = integral of f V E cos over the sphere, with
//   f     the BRDF albedo*rescale/pi + GGX of tir_ggx.h, as tir_relight_shade evaluates it (rl_contrib);
//   cos   w . normal with the raw normal (rl_cosine); a sample with cos <= 1e-6 contributes 0 and is not marched;
//   V     the visibility relight() reads from its march (vis_kind 0, nerv: t_last; 1, nerfactor: 1 - acc);
//   E_l   map l taken as piecewise constant over its lat-long texels: texel (r, c) covers the polar angles
//         [r pi/H, (r+1) pi/H] and the azimuths [pi - (c+1) 2pi/W, pi - c 2pi/W] (hdr_dir's column c sits at the middle,
//         column 0 next to +pi); rl_texel maps a direction to its texel.
// The two strategies, combined with the balance heuristic in its one-formula form (no division by S):
//   light  texel b from the map's fp64 CDF (rl_bin), then a point uniform in the texel's solid angle: z = cos(polar)
//          uniform between the row's bounds, azimuth uniform across the column.  p_light(w) = P_b / dOmega_b with
//          P_b = cdf[b] - cdf[b-1] and dOmega_b = (2pi/W) (cos(r pi/H) - cos((r+1) pi/H)), the exact solid angle.
//   BRDF   one sample of the mixture: with probability 1/2 (u0 < 1/2) a GGX visible-normal half vector (Heitz 2018)
//          with alpha = mean(r)^2 about the view-side normal Np, reflected: w = 2 (V.h) h - V; otherwise a cosine-
//          weighted direction about Np (concentric disc, Malley's method).
//          p_brdf(w) = 1/2 G1(V) D(h) / (4 NoV) + 1/2 max(Np.w, 0) / pi, h = normalize(V + w), which is defined on the
//          whole sphere: a reflected direction below the horizon keeps its density and fails the cosine test.
//          G1(V) D(h) / (4 NoV) is evaluated as D(h) / (2 (NoV + sqrt(alpha^2 + (1 - alpha^2) NoV^2))).
//          The BRDF directions do not depend on the map: one set per ray is shared by every map.
// E and p_light of every sample, from either strategy, come from rl_texel(w) of the direction as rounded, never from
// the bin it was drawn from, so the estimator is exactly the balance heuristic of the sampler as rounded.  p_light > 0
// wherever E > 0, so the light strategy alone covers the integrand: the estimate is unbiased whatever p_brdf does
// (where the raw normal faces away from the view and Np is flipped, for instance).  Sampling and both densities are
// computed in fp64 and rounded once; the BRDF, the cosine and the sum are fp32, as in tir_relight_shade.
#pragma once
#include "tir_lights_body.h"
#include "tir_relight_body.h"

namespace mis {
constexpr double kPi = 3.14159265358979323846;
}

// sin(pi x) and cos(pi x): exact argument reduction on the device, no slow path
RL_HD double mis_sinpi(double x) {
#if defined(__CUDA_ARCH__)
  return sinpi(x);
#else
  return sin(mis::kPi * x);
#endif
}
RL_HD double mis_cospi(double x) {
#if defined(__CUDA_ARCH__)
  return cospi(x);
#else
  return cos(mis::kPi * x);
#endif
}

// Texel of direction d (any length): row = floor(acos(z/|d|) H / pi), column = floor((pi - atan2(y, x)) W / 2pi),
// clamped to the map.  fp32, every operation rounded alone; a direction within a few ulp of a texel edge may land in
// either neighbour, and the estimator stays exact for whichever it returns.
RL_HD int rl_texel(const TirEnvMap& e, const float d[3]) {
  const float pi = tir::kPi;
  const float nn = sqrtf(ev_add(ev_add(ev_mul(d[0], d[0]), ev_mul(d[1], d[1])), ev_mul(d[2], d[2])));
  const float z = fminf(fmaxf(ev_div(d[2], fmaxf(nn, 1e-30f)), -1.f), 1.f);
  const float rf = floorf(ev_div(ev_mul(acosf(z), (float)e.H), pi));
  const float cf = floorf(ev_div(ev_mul(ev_sub(pi, atan2f(d[1], d[0])), (float)e.W), ev_add(pi, pi)));
  const int r = rf < 0.f ? 0 : (rf > (float)(e.H - 1) ? e.H - 1 : (int)rf);
  const int c = cf < 0.f ? 0 : (cf > (float)(e.W - 1) ? e.W - 1 : (int)cf);
  return r * e.W + c;
}

// P_b = cdf[b] - cdf[b-1], the probability of texel b under the light strategy
RL_HD double mis_texel_prob(const TirEnvMap& e, int b) {
  const double hi = RL_LDG(e.cdf + b);
  return b > 0 ? hi - RL_LDG(e.cdf + b - 1) : hi;
}

// Exact solid angle of a texel of row r: (2pi/W)(cos(r pi/H) - cos((r+1) pi/H)), written as a product of sines so that
// the rows next to the poles do not cancel
RL_HD double mis_texel_solid_angle(int H, int W, int r) {
  return (2.0 * mis::kPi / W) * 2.0 * mis_sinpi((r + 0.5) / H) * mis_sinpi(0.5 / H);
}

// p_light(w) of one map: P_b / dOmega_b of b = rl_texel(w); 0 where the map has no intensity
RL_HD double mis_pdf_light(const TirEnvMap& e, int b) {
  return mis_texel_prob(e, b) / mis_texel_solid_angle(e.H, e.W, b / e.W);
}

// Light strategy: a direction uniform in the solid angle of texel b, from (u[0], u[1]) = (z, azimuth) fractions
RL_HD void mis_light_dir(const TirEnvMap& e, int b, const double* u, float w[3]) {
  const int r = b / e.W, c = b - r * e.W;
  const double zt = mis_cospi((double)r / e.H), zb = mis_cospi((double)(r + 1) / e.H);
  const double z = zt + u[0] * (zb - zt);
  const double ph = 1.0 - 2.0 * (c + u[1]) / e.W;          // azimuth / pi
  const double s = sqrt(fmax(0.0, 1.0 - z * z));
  w[0] = (float)(s * mis_cospi(ph));
  w[1] = (float)(s * mis_sinpi(ph));
  w[2] = (float)z;
}

// Per hit, what p_brdf needs besides Np and V: alpha^2 and the VNDF factor 1 / (2 (NoV + sqrt(a2 + (1 - a2) NoV^2)))
struct MisPoint {
  double alpha, a2, vk;
};

RL_HD double mis_dot(const float a[3], const float b[3]) {
  return (double)a[0] * b[0] + (double)a[1] * b[1] + (double)a[2] * b[2];
}

RL_HD void mis_point(const tir::PointCtx& c, MisPoint& m) {
  const double r = ((double)c.r[0] + (double)c.r[1] + (double)c.r[2]) / 3.0;
  m.alpha = r * r;
  m.a2 = m.alpha * m.alpha;
  const double nov = fmax(mis_dot(c.Np, c.V), 0.0);
  m.vk = 0.5 / (nov + sqrt(m.a2 + (1.0 - m.a2) * nov * nov));
}

// GGX D(h) = a2 / (pi (1 - NoH^2 (1 - a2))^2) for NoH > 0, else 0
RL_HD double mis_ggx_d(double a2, double noh) {
  if (!(noh > 0.0)) return 0.0;
  const double t = 1.0 - noh * noh * (1.0 - a2);
  return a2 / (mis::kPi * t * t);
}

// p_brdf(w) of the mixture, for a direction of any length
RL_HD double mis_pdf_brdf(const tir::PointCtx& c, const MisPoint& m, const float w[3]) {
  const double wn = sqrt(mis_dot(w, w));
  if (!(wn > 0.0)) return 0.0;
  double L[3], h[3], hn = 0.0;
  for (int e = 0; e < 3; ++e) { L[e] = w[e] / wn; h[e] = L[e] + c.V[e]; hn += h[e] * h[e]; }
  double nol = 0.0, noh = 0.0;
  for (int e = 0; e < 3; ++e) { nol += c.Np[e] * L[e]; noh += c.Np[e] * h[e]; }
  const double p_cos = fmax(nol, 0.0) / mis::kPi;
  const double p_vndf = hn > 0.0 ? mis_ggx_d(m.a2, noh / sqrt(hn)) * m.vk : 0.0;
  return 0.5 * p_vndf + 0.5 * p_cos;
}

// BRDF strategy: one direction from u[0] (lobe), u[1], u[2], in the frame (t1, t2, Np) of lt_frame
RL_HD void mis_brdf_dir(const tir::PointCtx& c, const MisPoint& m, const double* u, float w[3]) {
  float t1[3], t2[3];
  lt_frame(c.Np, t1, t2);
  double out[3];
  if (u[0] < 0.5) {
    // Heitz 2018, "Sampling the GGX distribution of visible normals", in the local frame z = Np
    const double a = m.alpha;
    const double vl[3] = {mis_dot(c.V, t1), mis_dot(c.V, t2), mis_dot(c.V, c.Np)};
    double vh[3] = {a * vl[0], a * vl[1], vl[2]};
    const double vn = sqrt(vh[0] * vh[0] + vh[1] * vh[1] + vh[2] * vh[2]);
    for (int e = 0; e < 3; ++e) vh[e] = vn > 0.0 ? vh[e] / vn : (e == 2 ? 1.0 : 0.0);
    const double lensq = vh[0] * vh[0] + vh[1] * vh[1];
    double T1[3] = {1.0, 0.0, 0.0};
    if (lensq > 0.0) {
      const double il = 1.0 / sqrt(lensq);
      T1[0] = -vh[1] * il; T1[1] = vh[0] * il; T1[2] = 0.0;
    }
    const double T2[3] = {vh[1] * T1[2] - vh[2] * T1[1], vh[2] * T1[0] - vh[0] * T1[2], vh[0] * T1[1] - vh[1] * T1[0]};
    const double rr = sqrt(u[1]);
    const double p1 = rr * mis_cospi(2.0 * u[2]);
    const double s = 0.5 * (1.0 + vh[2]);
    const double p2 = (1.0 - s) * sqrt(fmax(0.0, 1.0 - p1 * p1)) + s * (rr * mis_sinpi(2.0 * u[2]));
    const double p3 = sqrt(fmax(0.0, 1.0 - p1 * p1 - p2 * p2));
    double nh[3];
    for (int e = 0; e < 3; ++e) nh[e] = p1 * T1[e] + p2 * T2[e] + p3 * vh[e];
    double ne[3] = {a * nh[0], a * nh[1], fmax(0.0, nh[2])};
    const double nn = sqrt(ne[0] * ne[0] + ne[1] * ne[1] + ne[2] * ne[2]);
    for (int e = 0; e < 3; ++e) ne[e] = nn > 0.0 ? ne[e] / nn : (e == 2 ? 1.0 : 0.0);
    double h[3], voh = 0.0;
    for (int e = 0; e < 3; ++e) { h[e] = ne[0] * t1[e] + ne[1] * t2[e] + ne[2] * c.Np[e]; voh += c.V[e] * h[e]; }
    for (int e = 0; e < 3; ++e) out[e] = 2.0 * voh * h[e] - c.V[e];
  } else {
    float x, y;
    lt_disc(u[1], u[2], x, y);
    const double z = sqrt(fmax(0.0, 1.0 - (double)x * x - (double)y * y));
    for (int e = 0; e < 3; ++e) out[e] = (double)x * t1[e] + (double)y * t2[e] + z * c.Np[e];
  }
  for (int e = 0; e < 3; ++e) w[e] = (float)out[e];
}

// The denominator S_l p_light(w) + S_b p_brdf(w) of one sample and the texel it reads E from
RL_HD float mis_denominator(const TirEnvMap& e, const tir::PointCtx& c, const MisPoint& m, int S_l, int S_b,
                            const float w[3], int& b) {
  b = rl_texel(e, w);
  const double p = S_l * mis_pdf_light(e, b) + (S_b > 0 ? S_b * mis_pdf_brdf(c, m, w) : 0.0);
  return (float)p;
}

// The per-sample loop of one (map, ray): lane `lane` of `lanes` adds the terms of samples k = lane, lane + lanes, ...
// of the map's S_l light slots (k < S_l) and then the ray's S_b BRDF slots to acc[3].  A slot with pos < 0 was not
// marched (cos <= 1e-6) and adds nothing; so does one whose denominator is 0 (E = 0 there).  The kernels run it on the
// 32 lanes of a warp and reduce with warp_sum; the host build runs the lanes in turn and reduces with the same xor
// butterfly.
RL_HD void mis_lane(const TirEnvMap& e, const tir::PointCtx& c, const MisPoint& m, const float* dir_l,
                    const int32_t* pos_l, int S_l, const float* dir_b, const int32_t* pos_b, int S_b,
                    const float* vis_list, int vis_kind, int lane, int lanes, float acc[3]) {
  for (int k = lane; k < S_l + S_b; k += lanes) {
    const bool light = k < S_l;
    const int64_t s = light ? k : k - S_l;
    const int q = light ? pos_l[s] : pos_b[s];
    if (q < 0) continue;
    const float* dp = (light ? dir_l : dir_b) + s * 3;
    const float w[3] = {dp[0], dp[1], dp[2]};
    int b;
    const float pdf = mis_denominator(e, c, m, S_l, S_b, w, b);
    if (!(pdf > 0.f)) continue;
    const float vis = rl_vis(vis_list, vis_kind, q);
    float rgb[3];
    for (int ch = 0; ch < 3; ++ch) rgb[ch] = RL_LDG(e.rgb + (int64_t)b * 3 + ch);
    rl_contrib(c, w, rgb, pdf, vis, acc);
  }
}

// argument checks shared by the kernels and the host build: 1 run, 0 nothing to do, < 0 TirStatus
inline int mis_validate(const TirEnvMap* envs, int32_t n_lights, int64_t n, int32_t S_l, int32_t S_b,
                        int32_t rough_stride) {
  if (S_l < 1 || S_b < 0) return TIR_ERR_SHAPE;
  if (rough_stride != 1 && rough_stride != 3) return TIR_ERR_SHAPE;
  return rl_validate(envs, n_lights, n, S_l);
}

// The whole argument check of each entry, run by tir_relight_mis.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus
inline int mis_sample_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* depth,
                            const float* normal, const float* albedo, const float* rough, int32_t rough_stride,
                            const float* fresnel, const float* acc, int64_t n, int32_t S_l, int32_t S_b,
                            const double* u_light, const double* u_brdf, const float* dir, const int32_t* pos,
                            const float* list_o, const float* list_d, int64_t capacity, const int64_t* count) {
  const int rc = mis_validate(envs, n_lights, n, S_l, S_b, rough_stride);
  if (rc < 0) return rc;
  // a bad capacity fails even with nothing to do; missing lists only when there is
  const int lrc = rl_check_list(capacity, list_o, list_d);
  if (lrc == TIR_ERR_SHAPE) return lrc;
  if (rc == 0) return 0;
  if (!rays || !depth || !normal || !albedo || !rough || !fresnel || !acc || !u_light || !dir || !pos || !count)
    return TIR_ERR_NULL;
  if (S_b > 0 && !u_brdf) return TIR_ERR_NULL;
  return lrc ? lrc : 1;
}

inline int mis_shade_check(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                           const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                           const float* acc, int64_t n, int32_t S_l, int32_t S_b, const float* rescale,
                           const float* dir, const int32_t* pos, const float* vis_list, int32_t vis_kind,
                           const float* with_bg, const float* without_bg, int64_t out_rows, int64_t row0) {
  const int rc = mis_validate(envs, n_lights, n, S_l, S_b, rough_stride);
  if (rc < 0) return rc;
  const int wrc = rl_check_window(rough_stride, vis_kind, n, out_rows, row0);
  if (wrc) return wrc;
  if (rc == 0) return 0;
  if (!rays || !normal || !albedo || !rough || !fresnel || !acc || !rescale || !dir || !pos || !vis_list ||
      !with_bg || !without_bg)
    return TIR_ERR_NULL;
  return 1;
}
