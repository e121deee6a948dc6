// Host twin of csrc/tir_tail.cu for the CPU test of tensoir_b200/tail.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (tail_*_check, epi_*_check) and per-item math of
// csrc/tir_tail_body.h and csrc/tir_epilogue_body.h, with plain loops instead of kernels.  Lets the ctypes marshalling
// and the autograd wrappers run end to end without a GPU.
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_epilogue_body.h"
#include "../tensoir_b200/csrc/tir_tail_body.h"

static TailSample load_sample(int64_t i, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                              const float* brdfj, const float* vn, const float* dn, const float* viewdirs) {
  TailSample s;
  s.w = w[i];
  for (int c = 0; c < 3; ++c) {
    s.rgb[c] = rgb[i * 3 + c]; s.vn[c] = vn[i * 3 + c]; s.dn[c] = dn ? dn[i * 3 + c] : 0.f;
    s.vd[c] = viewdirs[ray[i] * 3 + c];
  }
  for (int c = 0; c < 4; ++c) { s.brdf[c] = brdf[i * 4 + c]; s.brdfj[c] = brdfj[i * 4 + c]; }
  return s;
}

extern "C" int tir_tail_fwd(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                            const float* brdfj, const float* vn, const float* dn, const float* viewdirs, float* packed,
                            void*) {
  const int rc = tail_fwd_check(n, w, ray, rgb, brdf, brdfj, vn, viewdirs, packed);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i) {
    const TailSample s = load_sample(i, w, ray, rgb, brdf, brdfj, vn, dn, viewdirs);
    float v[TAIL_CH];
    tail_channels(s, dn != nullptr, v);
    for (int k = 0; k < TAIL_CH; ++k) packed[ray[i] * TAIL_CH + k] += s.w * v[k];
  }
  return TIR_OK;
}

extern "C" int tir_tail_bwd(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                            const float* brdfj, const float* vn, const float* dn, const float* viewdirs,
                            const float* g_packed, float* g_w, float* g_rgb, float* g_brdf, float* g_brdfj, float* g_vn,
                            float* g_dn, void*) {
  const int rc = tail_bwd_check(n, w, ray, rgb, brdf, brdfj, vn, viewdirs, g_packed, g_w, g_rgb, g_brdf, g_brdfj, g_vn);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i) {
    const TailSample s = load_sample(i, w, ray, rgb, brdf, brdfj, vn, dn, viewdirs);
    TailGrad g;
    tail_backward_sample(s, dn != nullptr, g_packed + ray[i] * TAIL_CH, g);
    g_w[i] = g.w;
    for (int c = 0; c < 3; ++c) {
      g_rgb[i * 3 + c] = g.rgb[c]; g_vn[i * 3 + c] = g.vn[c];
      if (g_dn) g_dn[i * 3 + c] = g.dn[c];
    }
    for (int c = 0; c < 4; ++c) { g_brdf[i * 4 + c] = g.brdf[c]; g_brdfj[i * 4 + c] = g.brdfj[c]; }
  }
  return TIR_OK;
}

static EpiIn load_ray(int64_t r, const float* packed, const float* acc, const float* depth, const float* rays,
                      float fresnel0, int bg) {
  EpiIn in;
  for (int k = 0; k < 14; ++k) in.P[k] = packed[r * 14 + k];
  in.acc = acc[r]; in.depth = depth[r]; in.dz = rays[r * 6 + 5]; in.fresnel0 = fresnel0; in.bg = bg;
  return in;
}

extern "C" int tir_epilogue_fwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                                float fresnel0, int32_t bg, const TirRayMaps* o, uint8_t* acc_mask, float* losses, void*) {
  const int rc = epi_fwd_check(n, packed, acc, depth, rays, o, acc_mask, losses);
  if (rc <= 0) return rc;
  for (int64_t r = 0; r < n; ++r) {
    const EpiIn in = load_ray(r, packed, acc, depth, rays, fresnel0, bg);
    EpiOut e;
    epi_forward(in, e);
    for (int c = 0; c < 3; ++c) {
      o->rgb[r * 3 + c] = e.rgb[c]; o->normal[r * 3 + c] = e.normal[c];
      o->albedo[r * 3 + c] = e.albedo[c]; o->fresnel[r * 3 + c] = e.fresnel[c];
    }
    o->depth[r] = e.depth; o->rough[r] = e.rough; o->nd[r] = e.nd; o->no[r] = e.no;
    acc_mask[r] = in.acc > 0.5f ? 1 : 0;
    losses[0] += e.ac / (float)n; losses[1] += e.rc / (float)n;
  }
  return TIR_OK;
}

extern "C" int tir_epilogue_bwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                                float fresnel0, int32_t bg, const TirRayMaps* g, const float* g_la, const float* g_lr,
                                float* g_packed, float* g_acc, float* g_depth, void*) {
  const int rc = epi_bwd_check(n, packed, acc, depth, rays, g, g_packed, g_acc, g_depth);
  if (rc <= 0) return rc;
  for (int64_t r = 0; r < n; ++r) {
    const EpiIn in = load_ray(r, packed, acc, depth, rays, fresnel0, bg);
    EpiOut e;
    for (int c = 0; c < 3; ++c) {
      e.rgb[c] = g->rgb ? g->rgb[r * 3 + c] : 0.f; e.normal[c] = g->normal ? g->normal[r * 3 + c] : 0.f;
      e.albedo[c] = g->albedo ? g->albedo[r * 3 + c] : 0.f; e.fresnel[c] = g->fresnel ? g->fresnel[r * 3 + c] : 0.f;
    }
    e.depth = g->depth ? g->depth[r] : 0.f; e.rough = g->rough ? g->rough[r] : 0.f;
    e.nd = g->nd ? g->nd[r] : 0.f; e.no = g->no ? g->no[r] : 0.f;
    e.ac = g_la ? g_la[0] / (float)n : 0.f; e.rc = g_lr ? g_lr[0] / (float)n : 0.f;
    float ga, gd;
    epi_backward(in, e, g_packed + r * 14, &ga, &gd);
    g_acc[r] = ga; g_depth[r] = gd;
  }
  return TIR_OK;
}
