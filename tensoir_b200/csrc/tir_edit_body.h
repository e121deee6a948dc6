// Per-point math of material editing (tir_material_edit, include/tensoir_b200.h).  Shared by the CUDA kernel
// (tir_edit.cu) and by a host build (tests/host_edit.cpp) that the CPU tests drive through the ctypes wrapper and
// compare with a numpy restatement of the rules.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"
#include "tir_relight_body.h"

// NaN passes through, as np.clip lets it
RL_HD float ed_clamp(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

RL_HD float ed_apply(int op, float x, float v, float lo, float hi) {
  if (op == TIR_EDIT_SET) return ed_clamp(v, lo, hi);
  if (op == TIR_EDIT_MUL) return ed_clamp(ev_mul(x, v), lo, hi);
  return x;
}

RL_HD bool ed_selects(const TirEditRule& r, const float p[3], const float a0[3]) {
  bool in = true;
  if (r.flags & TIR_EDIT_BOX)
    for (int c = 0; c < 3; ++c) in = in && r.box_lo[c] <= p[c] && p[c] <= r.box_hi[c];
  if (r.flags & TIR_EDIT_KEY)
    for (int c = 0; c < 3; ++c) in = in && fabsf(ev_sub(a0[c], r.key[c])) <= r.key_tol;
  return in;
}

// Row i of tir_material_edit: point p (already formed), its inputs, the rules; writes the outputs of the row.
RL_HD void ed_row(const TirEditRule* rules, int n_rules, const float p[3], const float* albedo, const float* rough,
                  int rough_stride, const float* fresnel, bool edit, const float scale[3], float* albedo_out,
                  float* rough_out, float* fresnel_out, int32_t* sel) {
  float a0[3], a[3], f[3], r[3];
  for (int c = 0; c < 3; ++c) {
    a0[c] = ev_mul(albedo[c], scale[c]);
    a[c] = a0[c];
    f[c] = fresnel[c];
  }
  for (int c = 0; c < 3; ++c) r[c] = c < rough_stride ? rough[c] : 0.f;
  int32_t bits = 0;
  if (edit)
    for (int k = 0; k < n_rules; ++k) {
      const TirEditRule& q = rules[k];
      if (!ed_selects(q, p, a0)) continue;
      bits |= (int32_t)(1u << k);
      for (int c = 0; c < 3; ++c) {
        a[c] = ed_apply(q.albedo_op, a[c], q.albedo[c], 0.f, 1.f);
        f[c] = ed_apply(q.fresnel_op, f[c], q.fresnel[c], 0.f, 1.f);
      }
      for (int c = 0; c < 3; ++c) r[c] = ed_apply(q.rough_op, r[c], q.rough, TIR_EDIT_ROUGH_MIN, TIR_EDIT_ROUGH_MAX);
    }
  for (int c = 0; c < 3; ++c) { albedo_out[c] = a[c]; fresnel_out[c] = f[c]; }
  for (int c = 0; c < 3; ++c)
    if (c < rough_stride) rough_out[c] = r[c];
  *sel = bits;
}

// argument checks shared by the kernel and the host build: 1 run, 0 nothing to do, < 0 TirStatus
inline int ed_validate(const TirEditRule* rules, int32_t n_rules, const float* rays, const float* depth,
                       const float* points, const float* albedo, const float* rough, int32_t rough_stride,
                       const float* fresnel, const float* acc, int64_t n, const float* scale, const float* albedo_out,
                       const float* rough_out, const float* fresnel_out, const int32_t* sel) {
  if (n < 0 || n_rules < 0 || n_rules > TIR_EDIT_MAX_RULES) return TIR_ERR_SHAPE;
  if (rough_stride != 1 && rough_stride != 3) return TIR_ERR_SHAPE;
  if (n_rules > 0 && !rules) return TIR_ERR_NULL;
  for (int k = 0; k < n_rules; ++k) {
    const TirEditRule& r = rules[k];
    if (r.flags & ~(TIR_EDIT_BOX | TIR_EDIT_KEY)) return TIR_ERR_CONFIG;
    const int32_t ops[3] = {r.albedo_op, r.rough_op, r.fresnel_op};
    for (int j = 0; j < 3; ++j)
      if (ops[j] != TIR_EDIT_NONE && ops[j] != TIR_EDIT_SET && ops[j] != TIR_EDIT_MUL) return TIR_ERR_CONFIG;
  }
  if (n == 0) return 0;
  if (!points && (!rays || !depth)) return TIR_ERR_NULL;
  if (!albedo || !rough || !fresnel || !acc || !scale || !albedo_out || !rough_out || !fresnel_out || !sel)
    return TIR_ERR_NULL;
  return 1;
}
