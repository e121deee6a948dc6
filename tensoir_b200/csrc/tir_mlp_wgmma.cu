// Hopper-native appearance MLP (sm_90a): the secondary-ray appearance head of compute_radiance
// (models/relight_utils.py:803-834) = compute_appfeature (tensoRF_rotated_lights.py:197-224) + MLPRender_Fea
// (tensorBase_rotated_lights.py:122-146) on the compacted appearance-sample list, with basis_mat and the two 128-wide
// layers on the tensor cores through warpgroup MMAs:
//
//   * wgmma.mma_async m64nNk16 (bf16 in, fp32 accumulate in registers), one 64-sample tile per warpgroup;
//   * the A operand (MLP input / hidden activations, error-compensated split BF16: hi + lo) is taken from REGISTERS:
//     the gather writes its products, and each layer's epilogue its activations, straight into the A fragments of the
//     next GEMM, so activations never touch shared memory; the B operands (split-BF16 weights, 162 KB) stay resident
//     in shared memory in the canonical no-swizzle K-major layout for the whole persistent CTA;
//   * every product is hi*hi + hi*lo + lo*hi accumulated in fp32 (the dropped lo*lo term is 2^-16 relative);
//   * the K order of a GEMM is free, so each layer's K axis is permuted to match what a thread already holds: in the
//     basis GEMM a thread's four A elements of a k16 step are four adjacent channels (one float4 per tap), in layer 0
//     they are the positional encodings of the basis features that thread's accumulator fragment produced; the weights
//     are staged with the same permutation;
//   * two warpgroups per CTA work on different tiles, so one warpgroup's L2-latency-bound gather overlaps the other's
//     tensor-core work;
//   * three GEMMs per tile: basis_mat (K = 144, N = 32), layer 0 (K = 160, N = 128), layer 1 (K = 128, N = 128).
//   The last layer (128 -> 3/4, < 1 % of the FLOPs) runs in fp32 on the CUDA cores with a quad shuffle reduction.
#include <cuda_bf16.h>
#include "tir_device.cuh"
#include "tir_internal.h"

using namespace tir;

namespace {

constexpr int AC = 48;
constexpr int K0 = 3 * AC;        // 144
constexpr int F = 27;
constexpr int HID = 128;
constexpr int IN = 150;
constexpr int K1 = 160;           // IN padded to k16
constexpr int ROWS = 64;          // samples per tile = wgmma M
constexpr int NWG = 2;            // warpgroups per CTA, each on its own tiles
constexpr int NTHREADS = NWG * 128;

struct SmemW {
  // B operands, canonical K-major no-swizzle layout: byte offset(n, k) = (k >> 3) * (rows * 16) + n * 16 + (k & 7) * 2
  __align__(128) uint8_t w0h[HID * K1 * 2];
  uint8_t w0l[HID * K1 * 2];
  uint8_t w1h[HID * HID * 2];
  uint8_t w1l[HID * HID * 2];
  uint8_t bsh[32 * K0 * 2];       // basis_mat as a B operand: [n = feature (27 -> 32)][k = product channel]
  uint8_t bsl[32 * K0 * 2];
  float w2[4 * HID];
  float b0[HID], b1[HID], b2[4];
  float lmean[K0];
};

struct WgParams {
  TirField f;
  TirMlp mlp;
  // sample-list mode
  const TirAppSample* samples;
  const uint32_t* sample_count;
  int64_t max_samples;
  const float* ray_dirs;
  int n_dirs;
  const int32_t* light_idx;
  float* rgb_out;
  // points mode
  const float* pts_xn;
  const float* pts_x;
  int64_t n_points;
  float* out;
  int act;
  int light_mode;     // 0 none, 1 indexed row, 2 mean row
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t operand_offset(int n, int k, int rows) {
  return (uint32_t)(k >> 3) * (uint32_t)(rows * 16) + (uint32_t)n * 16u + (uint32_t)(k & 7) * 2u;
}
// wgmma shared-memory descriptor, no swizzle: LBO = bytes between K-adjacent core matrices (= operand rows * 16),
// SBO = 128 B between 8-row groups
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((128u >> 4) & 0x3FFFu) << 32;
  return d;
}

__device__ __forceinline__ void wgmma_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(1));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// fp32 pair -> packed split-BF16 words: hi = (bf16(a) | bf16(b) << 16), lo = the residuals
__device__ __forceinline__ void split_pack(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat16 ah = __float2bfloat16_rn(a), bh = __float2bfloat16_rn(b);
  const __nv_bfloat16 al = __float2bfloat16_rn(a - __bfloat162float(ah)), bl = __float2bfloat16_rn(b - __bfloat162float(bh));
  hi = (uint32_t)__bfloat16_as_ushort(ah) | ((uint32_t)__bfloat16_as_ushort(bh) << 16);
  lo = (uint32_t)__bfloat16_as_ushort(al) | ((uint32_t)__bfloat16_as_ushort(bl) << 16);
}

// K permutation inside a k16 step: thread t4 of a quad holds A elements e = 0..3 at positions 2*t4 + (e & 1) + 8*(e >> 1)
// (the wgmma / mma.m16n8k16 A fragment); position p of the step therefore belongs to (t4, e) below.
__host__ __device__ __forceinline__ int pos_t4(int p) { return (p & 7) >> 1; }
__host__ __device__ __forceinline__ int pos_e(int p) { return (p & 1) | ((p >> 3) << 1); }

// Column of the 150-wide MLP input [feat 27 | x 3 | sin PE(feat) 54 | cos 54 | sin PE(x) 6 | cos 6] (tensorBase:12-17,
// :136-142) held in layer-0 slot s = q * 8 + j of quad thread t4, or -1 for a zero slot.  Slot (q, j) is quantity
// q in {v, sin v, sin 2v, cos v, cos 2v} of the thread's j-th basis feature f = 8 * (j >> 1) + 2 * t4 + (j & 1) (the
// accumulator fragment order); the five j = 7 slots of t4 = 1..3 (features 27, 29, 31 do not exist) carry the view
// direction component t4 - 1 instead.
__device__ __forceinline__ int input_column(int t4, int q, int j) {
  const int f = 8 * (j >> 1) + 2 * t4 + (j & 1);
  if (f < F) return q == 0 ? f : (q <= 2 ? 30 + 2 * f + (q - 1) : 84 + 2 * f + (q - 3));
  if (j == 7 && t4 >= 1) {
    const int d = t4 - 1;
    return q == 0 ? F + d : (q <= 2 ? 138 + 2 * d + (q - 1) : 144 + 2 * d + (q - 3));
  }
  return -1;
}

__device__ __forceinline__ void stage(uint8_t* hi, uint8_t* lo, int n, int k, int rows, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v), l = __float2bfloat16_rn(v - __bfloat162float(h));
  *reinterpret_cast<__nv_bfloat16*>(hi + operand_offset(n, k, rows)) = h;
  *reinterpret_cast<__nv_bfloat16*>(lo + operand_offset(n, k, rows)) = l;
}

struct RowIn {
  float xn[3], xv[3], wgt;
  int ray, li;
  bool live;
};

template <bool POINTS>
__device__ __forceinline__ RowIn load_row(const WgParams& p, int64_t i, int64_t total) {
  RowIn r{};
  r.live = i < total;
  if (!r.live) return r;
  if (POINTS) {
    r.xn[0] = p.pts_xn[i * 3]; r.xn[1] = p.pts_xn[i * 3 + 1]; r.xn[2] = p.pts_xn[i * 3 + 2];
    r.xv[0] = p.pts_x[i * 3]; r.xv[1] = p.pts_x[i * 3 + 1]; r.xv[2] = p.pts_x[i * 3 + 2];
    r.li = p.light_idx ? p.light_idx[i] : 0;
  } else {
    const TirAppSample sm = p.samples[i];
    r.xn[0] = sm.xn[0]; r.xn[1] = sm.xn[1]; r.xn[2] = sm.xn[2]; r.wgt = sm.weight; r.ray = sm.ray;
    const int64_t di = p.n_dirs > 0 ? (int64_t)(sm.ray % p.n_dirs) : (int64_t)sm.ray;
    r.xv[0] = __ldg(p.ray_dirs + di * 3); r.xv[1] = __ldg(p.ray_dirs + di * 3 + 1); r.xv[2] = __ldg(p.ray_dirs + di * 3 + 2);
    r.li = p.light_idx ? __ldg(p.light_idx + (p.n_dirs > 0 ? sm.ray / p.n_dirs : sm.ray)) : 0;
  }
  return r;
}

template <bool POINTS>
__global__ void __launch_bounds__(NTHREADS, 1) app_mlp_wgmma_kernel(const WgParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SmemW& s = *reinterpret_cast<SmemW*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wg = warp >> 2, g = lane >> 2, t4 = lane & 3;
  const TirMlp& mlp = p.mlp;
  const int out_dim = mlp.out_dim;

  // ---- stage the split-BF16 weights (K axes permuted as described at the top), once per persistent CTA
  for (int i = tid; i < HID * K1; i += NTHREADS) {
    const int n = i / K1, k = i % K1, pp = k & 15, e = pos_e(pp);
    const int slot = (k >> 4) * 4 + e;
    const int col = input_column(pos_t4(pp), slot >> 3, slot & 7);
    stage(s.w0h, s.w0l, n, k, HID, col >= 0 ? __ldg(mlp.w0 + n * IN + col) : 0.f);
  }
  for (int i = tid; i < HID * HID; i += NTHREADS) stage(s.w1h, s.w1l, i / HID, i % HID, HID, __ldg(mlp.w1 + i));
  for (int i = tid; i < 32 * K0; i += NTHREADS) {
    const int n = i / K0, k = i % K0, pp = k & 15;
    const int ch = (k & ~15) + 4 * pos_t4(pp) + pos_e(pp);          // product channel at logical position k
    stage(s.bsh, s.bsl, n, k, 32, n < F ? __ldg(mlp.basis + n * K0 + ch) : 0.f);
  }
  for (int i = tid; i < 4 * HID; i += NTHREADS) s.w2[i] = (i / HID) < out_dim ? __ldg(mlp.w2 + i) : 0.f;
  for (int i = tid; i < HID; i += NTHREADS) { s.b0[i] = __ldg(mlp.b0 + i); s.b1[i] = __ldg(mlp.b1 + i); }
  if (tid < 4) s.b2[tid] = tid < out_dim ? __ldg(mlp.b2 + tid) : 0.f;
  if (p.light_mode == 2)
    for (int c = tid; c < K0; c += NTHREADS) {
      float a = 0.f;
      for (int l = 0; l < mlp.n_lights; ++l) a += __ldg(mlp.light_line + (size_t)l * K0 + c);
      s.lmean[c] = a / (float)mlp.n_lights;
    }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
  __syncthreads();

  const uint32_t a_bsh = smem_u32(s.bsh), a_bsl = smem_u32(s.bsl);
  const uint32_t a_w0h = smem_u32(s.w0h), a_w0l = smem_u32(s.w0l), a_w1h = smem_u32(s.w1h), a_w1l = smem_u32(s.w1l);
  const int64_t total = POINTS ? p.n_points
                               : (int64_t)min((unsigned long long)*p.sample_count, (unsigned long long)p.max_samples);
  const int64_t n_tiles = (total + ROWS - 1) / ROWS;

  for (int64_t tile = (int64_t)blockIdx.x * NWG + wg; tile < n_tiles; tile += (int64_t)gridDim.x * NWG) {
    // this thread's two rows of the tile: the A / accumulator fragment rows g and g + 8 of its warp's 16-row slice
    const int64_t row0 = tile * ROWS + (warp & 3) * 16 + g;
    RowIn rw[2] = {load_row<POINTS>(p, row0, total), load_row<POINTS>(p, row0 + 8, total)};

    // ---- gather: products (plane * line * light) -> split-BF16 A fragments of the basis GEMM (9 k16 steps)
    uint32_t ah[9][4], al[9][4];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int m0 = kMat0[k], m1 = kMat1[k], v = kVec[k];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const Bilinear b = bilinear_setup(rw[h].xn[m0], rw[h].xn[m1], p.f.grid[m0], p.f.grid[m1]);
        const Linear1 l = linear_setup(rw[h].xn[v], p.f.grid[v]);
        const float* P = p.f.aplane[k];
        const float* L = p.f.aline[k];
        const float* lrow = p.light_mode == 1 ? (mlp.light_line + (size_t)rw[h].li * K0) : nullptr;
#pragma unroll
        for (int ks = 0; ks < AC / 16; ++ks) {
          const int c = ks * 16 + 4 * t4, col = k * AC + c;
          float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
          if (rw[h].live) {
            const float4 pv = bilerp4(ldg4(P + (size_t)b.o00 * AC + c), ldg4(P + (size_t)b.o01 * AC + c),
                                      ldg4(P + (size_t)b.o10 * AC + c), ldg4(P + (size_t)b.o11 * AC + c), b);
            const float4 lv = lerp4(ldg4(L + (size_t)l.o0 * AC + c), ldg4(L + (size_t)l.o1 * AC + c), l);
            x = make_float4(__fmul_rn(pv.x, lv.x), __fmul_rn(pv.y, lv.y), __fmul_rn(pv.z, lv.z), __fmul_rn(pv.w, lv.w));
            if (p.light_mode == 1) {            // (plane * line) * light  (tensoRF_rotated_lights.py:222)
              const float4 lc = ldg4(lrow + col);
              x.x = __fmul_rn(x.x, lc.x); x.y = __fmul_rn(x.y, lc.y); x.z = __fmul_rn(x.z, lc.z); x.w = __fmul_rn(x.w, lc.w);
            } else if (p.light_mode == 2) {
              x.x = __fmul_rn(x.x, s.lmean[col]); x.y = __fmul_rn(x.y, s.lmean[col + 1]);
              x.z = __fmul_rn(x.z, s.lmean[col + 2]); x.w = __fmul_rn(x.w, s.lmean[col + 3]);
            }
          }
          split_pack(x.x, x.y, ah[k * 3 + ks][h], al[k * 3 + ks][h]);
          split_pack(x.z, x.w, ah[k * 3 + ks][2 + h], al[k * 3 + ks][2 + h]);
        }
      }
    }

    // ---- basis_mat on the tensor cores: feat = products @ basis^T (27 of 32 accumulator columns)
    float accb[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) accb[i] = 0.f;
    fence_regs(accb);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < K0 / 16; ++ks) {
      const uint32_t koff = (uint32_t)ks * 2u * (32u * 16u);
      const uint64_t dh = make_desc(a_bsh + koff, 32u * 16u), dl = make_desc(a_bsl + koff, 32u * 16u);
      wgmma_n32(accb, al[ks], dh);         // small terms first
      wgmma_n32(accb, ah[ks], dl);
      wgmma_n32(accb, ah[ks], dh);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(accb);

    // ---- positional encoding -> split-BF16 A fragments of layer 0 (10 k16 steps, slot order of input_column)
    uint32_t a0h[10][4], a0l[10][4];
    {
      float u[2][8], sn[2][8], cs[2][8], keep[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int f = 8 * (j >> 1) + 2 * t4 + (j & 1);
        const bool xslot = j == 7 && t4 >= 1;
        keep[j] = (f < F || xslot) ? 1.f : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          u[h][j] = f < F ? accb[4 * (j >> 1) + 2 * h + (j & 1)] : (xslot ? (t4 == 1 ? rw[h].xv[0] : t4 == 2 ? rw[h].xv[1] : rw[h].xv[2]) : 0.f);
          sincosf(u[h][j], &sn[h][j], &cs[h][j]);
        }
      }
#pragma unroll
      for (int q = 0; q < 5; ++q)
#pragma unroll
        for (int j = 0; j < 8; j += 2)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v2[2];
#pragma unroll
            for (int t = 0; t < 2; ++t) {
              const int jj = j + t;
              const float a = u[h][jj], sa = sn[h][jj], ca = cs[h][jj];
              // frequency 2 via the double-angle identities (agrees with sin(2x) / cos(2x) to rounding level)
              const float val = q == 0 ? a : q == 1 ? sa : q == 2 ? 2.f * sa * ca : q == 3 ? ca : 1.f - 2.f * sa * sa;
              v2[t] = val * keep[jj];
            }
            split_pack(v2[0], v2[1], a0h[2 * q + (j >> 2)][h + 2 * ((j & 3) >> 1)], a0l[2 * q + (j >> 2)][h + 2 * ((j & 3) >> 1)]);
          }
    }

    // ---- layer 0 (K = 160, N = 128)
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    fence_regs(acc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < K1 / 16; ++ks) {
      const uint32_t koff = (uint32_t)ks * 2u * (uint32_t)(HID * 16);
      const uint64_t dh = make_desc(a_w0h + koff, HID * 16), dl = make_desc(a_w0l + koff, HID * 16);
      wgmma_n128(acc, a0l[ks], dh);
      wgmma_n128(acc, a0h[ks], dl);
      wgmma_n128(acc, a0h[ks], dh);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(acc);

    // ---- layer 0 epilogue: bias + ReLU; the accumulator fragment is already the A fragment layout of layer 1
    uint32_t a1h[8][4], a1l[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int n = 8 * (2 * j + (r >> 1)) + 2 * t4;
        const float a = fmaxf(acc[8 * j + 2 * r] + s.b0[n], 0.f), b = fmaxf(acc[8 * j + 2 * r + 1] + s.b0[n + 1], 0.f);
        split_pack(a, b, a1h[j][r], a1l[j][r]);
      }

    // ---- layer 1 (K = 128, N = 128)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    fence_regs(acc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HID / 16; ++ks) {
      const uint32_t koff = (uint32_t)ks * 2u * (uint32_t)(HID * 16);
      const uint64_t dh = make_desc(a_w1h + koff, HID * 16), dl = make_desc(a_w1l + koff, HID * 16);
      wgmma_n128(acc, a1l[ks], dh);
      wgmma_n128(acc, a1h[ks], dl);
      wgmma_n128(acc, a1h[ks], dh);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(acc);

    // ---- layer 1 epilogue + output layer (128 -> out_dim, fp32 on the CUDA cores, quad reduction)
    float o[2][4] = {};
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = 8 * i + 2 * t4 + (e & 1), h = e >> 1;
        const float hv = fmaxf(acc[4 * i + e] + s.b1[n], 0.f);
#pragma unroll
        for (int q = 0; q < 4; ++q) o[h][q] = fmaf(hv, s.w2[q * HID + n], o[h][q]);
      }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        o[h][q] += __shfl_xor_sync(0xffffffffu, o[h][q], 1);
        o[h][q] += __shfl_xor_sync(0xffffffffu, o[h][q], 2);
      }
    const int q = t4;                      // quad thread t4 writes output channel t4 of both rows
    if (q < out_dim) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!rw[h].live) continue;
        const float z = o[h][q] + s.b2[q];
        const float y = p.act == 0 ? 1.f / (1.f + expf(-z)) : tanhf(z);
        const int64_t i = row0 + 8 * h;
        if (POINTS) p.out[i * out_dim + q] = y;
        else atomicAdd(p.rgb_out + (int64_t)rw[h].ray * 3 + q, __fmul_rn(rw[h].wgt, y));
      }
    }
  }
}

int check_shapes(const TirField* f, const TirMlp* m) {
  if (f->aC != AC) return TIR_ERR_SHAPE;
  if (m->feat_dim != F || m->hidden != HID || m->pe_feat != 2 || m->pe_x != 2) return TIR_ERR_SHAPE;
  if (m->out_dim < 1 || m->out_dim > 4) return TIR_ERR_SHAPE;
  if (!m->w0 || !m->b0 || !m->w1 || !m->b1 || !m->w2 || !m->b2 || !m->basis) return TIR_ERR_NULL;
  return TIR_OK;
}

template <bool POINTS>
int launch_wg(const WgParams& p, int64_t max_items, cudaStream_t stream) {
  static bool configured[2] = {false, false};
  const int smem = (int)sizeof(SmemW);
  if (!configured[POINTS]) {
    cudaError_t e = cudaFuncSetAttribute(app_mlp_wgmma_kernel<POINTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured[POINTS] = true;
  }
  const int64_t groups = ((max_items + ROWS - 1) / ROWS + NWG - 1) / NWG;
  const int sms = num_sms();
  const int blocks = (int)(groups < sms ? (groups > 0 ? groups : 1) : sms);
  app_mlp_wgmma_kernel<POINTS><<<blocks, NTHREADS, smem, stream>>>(p);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" int tir_app_mlp_wgmma(const TirField* field, const TirMlp* mlp, const TirAppSample* samples,
                                 const uint32_t* sample_count, int64_t max_samples, const float* ray_dirs,
                                 int32_t n_dirs, const int32_t* light_idx, float* rgb_out, void* stream) {
  if (!field || !mlp || !samples || !sample_count || !ray_dirs || !rgb_out) return TIR_ERR_NULL;
  int rc = check_shapes(field, mlp);
  if (rc) return rc;
  if (mlp->out_dim != 3) return TIR_ERR_SHAPE;
  WgParams p{};
  p.f = *field; p.mlp = *mlp; p.samples = samples; p.sample_count = sample_count; p.max_samples = max_samples;
  p.ray_dirs = ray_dirs; p.n_dirs = n_dirs; p.light_idx = light_idx; p.rgb_out = rgb_out; p.act = 0;
  p.light_mode = mlp->light_line ? 1 : 0;
  return launch_wg<false>(p, max_samples, (cudaStream_t)stream);
}

extern "C" int tir_app_mlp_points_wgmma(const TirField* field, const TirMlp* mlp, const float* xn, const float* x_in,
                                        const int32_t* light_idx, int64_t n, int32_t act, float* out, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!field || !mlp || !xn || !x_in || !out) return TIR_ERR_NULL;
  int rc = check_shapes(field, mlp);
  if (rc) return rc;
  if (act != 0 && act != 1) return TIR_ERR_CONFIG;
  WgParams p{};
  p.f = *field; p.mlp = *mlp; p.pts_xn = xn; p.pts_x = x_in; p.n_points = n; p.light_idx = light_idx; p.out = out;
  p.act = act; p.light_mode = mlp->light_line ? 1 : 0;
  return launch_wg<true>(p, n, (cudaStream_t)stream);
}
