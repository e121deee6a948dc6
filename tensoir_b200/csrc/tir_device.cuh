// Device-side building blocks shared by every kernel of the hot path.
// Arithmetic order mirrors what the reference executes through ATen's CUDA kernels, so that the
// threshold tests (in-bbox, alpha-mask > 0, weight > 1e-4) select the same samples:
//   * eager PyTorch never fuses a*b+c, so coordinate arithmetic uses __fmul_rn/__fadd_rn (no FMA
//     contraction);
//   * ATen's grid_sampler_2d CUDA kernel accumulates taps nw,ne,sw,se with FMAs, mirrored with fmaf.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"

namespace tir {

__device__ __constant__ const int kMat0[3] = {0, 0, 1};   // matMode[k][0]  (tensorBase:398)
__device__ __constant__ const int kMat1[3] = {1, 2, 2};   // matMode[k][1]
__device__ __constant__ const int kVec[3] = {2, 1, 0};    // vecMode[k]     (tensorBase:399)

// grid_sampler_unnormalize(align_corners=True): ((coord + 1) / 2) * (size - 1)
__device__ __forceinline__ float unnormalize(float c, int size) {
  return __fmul_rn(__fmul_rn(__fadd_rn(c, 1.f), 0.5f), (float)(size - 1));
}

// floor() without the XU (FRND / F2I run at quarter rate on the conversion pipe and carry a long latency, which made
// the march issue-latency bound): round-to-nearest via the 1.5*2^23 magic constant, then fix up.  Exact for |x| < 2^22
// (grid coordinates are < 2^10); out-of-range inputs fall back to floorf so semantics never change.
struct FloorI {
  float f;
  int i;
};
__device__ __forceinline__ FloorI floor_fi(float x) {
  FloorI r;
  if (fabsf(x) < 4194304.f) {
    const float m = __fadd_rn(x, 12582912.f);
    r.i = __float_as_int(m) - 0x4B400000;
    r.f = __fsub_rn(m, 12582912.f);
    if (r.f > x) { r.f = __fsub_rn(r.f, 1.f); r.i -= 1; }
  } else {
    r.f = floorf(x);
    r.i = (int)r.f;
  }
  return r;
}

// Streaming multiprocessors of the current device (132 on an H100 SXM), queried once per device: persistent kernels
// launch one wave of CTAs and grid-stride kernels cap their grids at a few CTAs per SM.
inline int num_sms() {
  static int cached[16] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  return cached[dev];
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// One whole 32-byte sector of a channel-last row through the read-only path: sm_90 has no 256-bit load, so this is two
// adjacent 128-bit loads issued back to back (the second one hits the sector the first one brought into L1).
// `p` must be 32-byte aligned.
struct Float8 { float4 a, b; };
__device__ __forceinline__ Float8 ldg8(const float* p) {
  Float8 r;
  r.a = __ldg(reinterpret_cast<const float4*>(p));
  r.b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  return r;
}

struct Bilinear {
  int o00, o01, o10, o11;   // element offsets (texel index, not yet multiplied by C)
  float nw, ne, sw, se;     // weights, zeroed for out-of-bounds taps (zero padding)
};

// F.grid_sample(bilinear, zeros, align_corners=True) tap set for one plane (W = grid[m0], H = grid[m1]).
__device__ __forceinline__ Bilinear bilinear_setup(float gx, float gy, int W, int H) {
  float ix = unnormalize(gx, W), iy = unnormalize(gy, H);
  const FloorI fx = floor_fi(ix), fy = floor_fi(iy);
  float x0f = fx.f, y0f = fy.f;
  float wx1 = __fsub_rn(ix, x0f), wx0 = __fsub_rn(__fadd_rn(x0f, 1.f), ix);
  float wy1 = __fsub_rn(iy, y0f), wy0 = __fsub_rn(__fadd_rn(y0f, 1.f), iy);
  int x0 = fx.i, y0 = fy.i, x1 = x0 + 1, y1 = y0 + 1;
  bool bx0 = (x0 >= 0) & (x0 < W), bx1 = (x1 >= 0) & (x1 < W);
  bool by0 = (y0 >= 0) & (y0 < H), by1 = (y1 >= 0) & (y1 < H);
  int cx0 = min(max(x0, 0), W - 1), cx1 = min(max(x1, 0), W - 1);
  int cy0 = min(max(y0, 0), H - 1), cy1 = min(max(y1, 0), H - 1);
  Bilinear b;
  b.o00 = cy0 * W + cx0; b.o01 = cy0 * W + cx1; b.o10 = cy1 * W + cx0; b.o11 = cy1 * W + cx1;
  b.nw = (bx0 & by0) ? __fmul_rn(wx0, wy0) : 0.f;
  b.ne = (bx1 & by0) ? __fmul_rn(wx1, wy0) : 0.f;
  b.sw = (bx0 & by1) ? __fmul_rn(wx0, wy1) : 0.f;
  b.se = (bx1 & by1) ? __fmul_rn(wx1, wy1) : 0.f;
  return b;
}

struct Linear1 {
  int o0, o1;
  float w0, w1;
};

// The W=1 "line" case of the same sampler: x coordinate 0 -> ix = 0, taps nw (weight y1-iy) and sw (iy-y0).
__device__ __forceinline__ Linear1 linear_setup(float gy, int D) {
  float iy = unnormalize(gy, D);
  const FloorI fy = floor_fi(iy);
  float y0f = fy.f;
  int y0 = fy.i, y1 = y0 + 1;
  Linear1 l;
  l.w0 = ((y0 >= 0) & (y0 < D)) ? __fsub_rn(__fadd_rn(y0f, 1.f), iy) : 0.f;
  l.w1 = ((y1 >= 0) & (y1 < D)) ? __fsub_rn(iy, y0f) : 0.f;
  l.o0 = min(max(y0, 0), D - 1);
  l.o1 = min(max(y1, 0), D - 1);
  return l;
}

__device__ __forceinline__ float4 bilerp4(const float4 a, const float4 b, const float4 c, const float4 d,
                                          const Bilinear& w) {
  float4 r;
  r.x = fmaf(d.x, w.se, fmaf(c.x, w.sw, fmaf(b.x, w.ne, __fmul_rn(a.x, w.nw))));
  r.y = fmaf(d.y, w.se, fmaf(c.y, w.sw, fmaf(b.y, w.ne, __fmul_rn(a.y, w.nw))));
  r.z = fmaf(d.z, w.se, fmaf(c.z, w.sw, fmaf(b.z, w.ne, __fmul_rn(a.z, w.nw))));
  r.w = fmaf(d.w, w.se, fmaf(c.w, w.sw, fmaf(b.w, w.ne, __fmul_rn(a.w, w.nw))));
  return r;
}

__device__ __forceinline__ float4 lerp4(const float4 a, const float4 b, const Linear1& w) {
  float4 r;
  r.x = fmaf(b.x, w.w1, __fmul_rn(a.x, w.w0));
  r.y = fmaf(b.y, w.w1, __fmul_rn(a.y, w.w0));
  r.z = fmaf(b.z, w.w1, __fmul_rn(a.z, w.w0));
  r.w = fmaf(b.w, w.w1, __fmul_rn(a.w, w.w0));
  return r;
}

// compute_densityfeature (tensoRF_rotated_lights.py:95-110) at one normalised point, C channels / orientation.
template <int C>
__device__ __forceinline__ float density_feature(const TirField& f, float x, float y, float z) {
  const float xn[3] = {x, y, z};
  float total = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int m0 = kMat0[k], m1 = kMat1[k], v = kVec[k];
    const int W = f.grid[m0], H = f.grid[m1], D = f.grid[v];
    const Bilinear b = bilinear_setup(xn[m0], xn[m1], W, H);
    const Linear1 l = linear_setup(xn[v], D);
    const float* P = f.dplane[k];
    const float* L = f.dline[k];
    const float* p00 = P + (size_t)b.o00 * C;
    const float* p01 = P + (size_t)b.o01 * C;
    const float* p10 = P + (size_t)b.o10 * C;
    const float* p11 = P + (size_t)b.o11 * C;
    const float* l0 = L + (size_t)l.o0 * C;
    const float* l1 = L + (size_t)l.o1 * C;
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < C; c += 8) {          // C is a multiple of 8 for every shipped config (16); same summation order
      const Float8 t00 = ldg8(p00 + c), t01 = ldg8(p01 + c), t10 = ldg8(p10 + c), t11 = ldg8(p11 + c);
      const Float8 u0 = ldg8(l0 + c), u1 = ldg8(l1 + c);
      const float4 pv = bilerp4(t00.a, t01.a, t10.a, t11.a, b);
      const float4 lv = lerp4(u0.a, u1.a, l);
      s = __fadd_rn(s, __fmul_rn(pv.x, lv.x));
      s = __fadd_rn(s, __fmul_rn(pv.y, lv.y));
      s = __fadd_rn(s, __fmul_rn(pv.z, lv.z));
      s = __fadd_rn(s, __fmul_rn(pv.w, lv.w));
      const float4 pw = bilerp4(t00.b, t01.b, t10.b, t11.b, b);
      const float4 lw = lerp4(u0.b, u1.b, l);
      s = __fadd_rn(s, __fmul_rn(pw.x, lw.x));
      s = __fadd_rn(s, __fmul_rn(pw.y, lw.y));
      s = __fadd_rn(s, __fmul_rn(pw.z, lw.z));
      s = __fadd_rn(s, __fmul_rn(pw.w, lw.w));
    }
    total = __fadd_rn(total, s);
  }
  return total;
}

// feature2density (tensorBase:813-817); F.softplus default beta=1, threshold=20.
__device__ __forceinline__ float feature_to_sigma(const TirField& f, float feat) {
  if (f.softplus) {
    float x = __fadd_rn(feat, f.density_shift);
    return (x > 20.f) ? x : log1pf(expf(x));
  }
  return fmaxf(feat, 0.f);
}

// AlphaGridMask.sample_alpha(p) > 0 (tensorBase:112-116) on a binary volume, evaluated exactly:
// a trilinear sum of non-negative terms is > 0 iff some in-bounds corner with value 1 has all three
// weight factors > 0.  Fast path: one byte of the per-cell OR volume when the point is strictly inside a cell.
__device__ __forceinline__ bool alpha_mask_positive(const TirField& f, float px, float py, float pz) {
  const int X = f.agrid[0], Y = f.agrid[1], Z = f.agrid[2];
  float gx = __fsub_rn(__fmul_rn(__fsub_rn(px, f.a_lo[0]), f.a_inv[0]), 1.f);
  float gy = __fsub_rn(__fmul_rn(__fsub_rn(py, f.a_lo[1]), f.a_inv[1]), 1.f);
  float gz = __fsub_rn(__fmul_rn(__fsub_rn(pz, f.a_lo[2]), f.a_inv[2]), 1.f);
  float ix = unnormalize(gx, X), iy = unnormalize(gy, Y), iz = unnormalize(gz, Z);
  const FloorI ffx = floor_fi(ix), ffy = floor_fi(iy), ffz = floor_fi(iz);
  float x0f = ffx.f, y0f = ffy.f, z0f = ffz.f;
  int x0 = ffx.i, y0 = ffy.i, z0 = ffz.i;
  float fx1 = __fsub_rn(ix, x0f), fy1 = __fsub_rn(iy, y0f), fz1 = __fsub_rn(iz, z0f);
  const bool inside = (x0 >= 0) & (x0 < X) & (y0 >= 0) & (y0 < Y) & (z0 >= 0) & (z0 < Z);
  if (inside & (fx1 > 0.f) & (fy1 > 0.f) & (fz1 > 0.f)) {
    return __ldg(f.acell + ((size_t)z0 * Y + y0) * X + x0) != 0;
  }
  // exact path (point on a cell face / outside the volume): factors for the "+0" corners are always > 0
  bool any = false;
#pragma unroll
  for (int dz = 0; dz < 2; ++dz)
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        int xx = x0 + dx, yy = y0 + dy, zz = z0 + dz;
        bool ok = (xx >= 0) & (xx < X) & (yy >= 0) & (yy < Y) & (zz >= 0) & (zz < Z);
        ok = ok & (dx ? (fx1 > 0.f) : true) & (dy ? (fy1 > 0.f) : true) & (dz ? (fz1 > 0.f) : true);
        if (ok) any = any | (__ldg(f.amask + ((size_t)zz * Y + yy) * X + xx) != 0);
      }
  return any;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace tir
