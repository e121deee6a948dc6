// Appearance gather (3 x 48-channel plane*line products) -> * light_line -> basis_mat (144 -> 27) ->
// positional encoding -> 150 -> 128 -> 128 -> {3,4} MLP, on explicit points: the primary appearance heads, up to four
// per launch, with optional activation dumps for the backward.  Replaces compute_appfeature / compute_intrinfeature
// (tensoRF_rotated_lights.py:167-224) + MLPRender_Fea / MLPBRDF_PEandFeature (tensorBase:122-146, :182-208).
// The secondary sample list goes through the wgmma kernel of tir_mlp_wgmma.cu.
//
// The four contractions are genuine dense GEMMs over a tile of 32 samples and run on the tensor cores with
// error-compensated BF16: every fp32 operand x is split into hi = bf16(x), lo = bf16(x - hi) and the product is
// accumulated in fp32 as A_hi*B_hi + A_hi*B_lo + A_lo*B_hi (the dropped lo*lo term is 2^-16 relative), which keeps
// the 1e-4 parity bar that plain BF16/TF32 (~1e-3) would miss.  Persistent CTAs (one per SM) keep all weights
// resident in shared memory as split BF16 (176 KB).  A CTA is two independent groups of 4 warps; each group streams
// its own 32-sample tiles through its own in-place activation buffer and synchronises on its own named barrier, so
// one group's gather and dumps overlap the other group's MMAs.  Fragments are fetched with ldmatrix from rows padded
// to an odd multiple of 16 bytes (conflict free).
#include <cuda_bf16.h>
#include "tir_device.cuh"
#include "tir_internal.h"

using namespace tir;

namespace {

constexpr int AC = 48;            // appearance channels / orientation
constexpr int K0 = 3 * AC;        // 144 = basis K (9 k16 steps)
constexpr int F = 27;             // app_dim
constexpr int FN = 32;            // basis N padded
constexpr int HID = 128;
constexpr int IN = 150;           // 27 + 3 + 54 + 54 + 6 + 6
constexpr int K1 = 160;           // IN padded to k16
constexpr int ON = 8;             // output N padded (<= 4 real)
constexpr int M = 32;             // samples per tile
constexpr int NG = 2;             // warp groups per CTA, one tile in flight each
constexpr int GT = 128;           // threads per group (4 warps)
constexpr int NT = NG * GT;
constexpr int SA = 168;           // activation row stride (bf16 elements); 336 B = odd multiple of 16 B
constexpr int SW0 = 168;          // W0 rows [128][K1 -> 168]
constexpr int SW1 = 136;          // W1 rows [128][128 -> 136]
constexpr int SBS = 152;          // basis rows [32][144 -> 152]
constexpr int SW2 = 136;          // W2 rows [8][128 -> 136]

struct __align__(16) Tile {                  // one warp group's tile
  __nv_bfloat16 ah[M * SA], al[M * SA];      // activations, in place across layers
  float xn[M][3];
  float xv[M][3];
  int light[M];
};

struct Smem {
  __nv_bfloat16 w0h[HID * SW0], w0l[HID * SW0];
  __nv_bfloat16 w1h[HID * SW1], w1l[HID * SW1];
  __nv_bfloat16 bsh[FN * SBS], bsl[FN * SBS];
  __nv_bfloat16 w2h[ON * SW2], w2l[ON * SW2];
  Tile t[NG];
  float b0[HID], b1[HID], b2[ON];
  float lmean[K0];                           // mean light row (light_mode 2, compute_intrinfeature)
};

struct MlpParams {
  TirField f;
  // up to 4 heads, CTA b works on job b % n_jobs (tir_internal.h)
  HeadJobDev jobs[kMaxHeadJobs];
  int n_jobs;
  int64_t n_points;
  const int64_t* n_dev;   // optional device-side row count (<= n_points)
  // legacy dump of the light-scaled products [n,144] (modular heads.py backward); job 0 only
  float* save_xl;
};

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& h, __nv_bfloat16& l) {
  h = __float2bfloat16_rn(x);
  l = __float2bfloat16_rn(x - __bfloat162float(h));
}

__device__ __forceinline__ void store_pair(__nv_bfloat16* hi, __nv_bfloat16* lo, int idx, float a, float b) {
  __nv_bfloat16 ah, al, bh, bl;
  split_bf16(a, ah, al);
  split_bf16(b, bh, bl);
  __nv_bfloat162 vh, vl;
  vh.x = ah; vh.y = bh; vl.x = al; vl.y = bl;
  *reinterpret_cast<__nv_bfloat162*>(hi + idx) = vh;
  *reinterpret_cast<__nv_bfloat162*>(lo + idx) = vl;
}

__device__ __forceinline__ void store_one(__nv_bfloat16* hi, __nv_bfloat16* lo, int idx, float a) {
  __nv_bfloat16 h, l;
  split_bf16(a, h, l);
  hi[idx] = h;
  lo[idx] = l;
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __nv_bfloat16* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

__device__ __forceinline__ void ldsm_x2(uint32_t (&r)[2], const __nv_bfloat16* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(r[0]), "=r"(r[1]) : "r"(a));
}

__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// The named barrier of warp group `grp` (barrier 0 is __syncthreads).
__device__ __forceinline__ void group_sync(int grp) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(grp + 1), "r"(GT) : "memory");
}

// One warp: acc[MT][NTL] (m16 x n8 tiles) += A[m0.., :K] * W[n0.., :K]^T with the 3-term split.
// A row-major [M][SA] (hi/lo), W row-major [N][SWx] (hi/lo) == PyTorch [out,in].  Every acc entry sees the same
// k order whatever MT / NTL are, so the warp mapping does not change the sums.
template <int MT, int NTL>
__device__ __forceinline__ void warp_gemm(float (&acc)[MT][NTL][4], const __nv_bfloat16* ah, const __nv_bfloat16* al,
                                          int m0, const __nv_bfloat16* wh, const __nv_bfloat16* wl, int sw, int n0,
                                          int K, int lane) {
  static_assert(NTL == 1 || NTL % 2 == 0, "n8 tiles are loaded in pairs");
  // ldmatrix source rows: A x4 = {(r0-7,k0-7),(r8-15,k0-7),(r0-7,k8-15),(r8-15,k8-15)}
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int a_col = (lane >> 4) * 8;
  // B x4 (two n8 tiles) = {(n0-7,k0-7),(n0-7,k8-15),(n8-15,k0-7),(n8-15,k8-15)};  x2 (one tile) = first two
  const int b_row = (lane & 7) + (lane >> 4) * 8;
  const int b_col = ((lane >> 3) & 1) * 8;
  for (int k = 0; k < K; k += 16) {
    uint32_t bh[NTL][2], bl[NTL][2];
    if constexpr (NTL % 2 == 0) {
#pragma unroll
      for (int p = 0; p < NTL / 2; ++p) {
        uint32_t t[4];
        ldsm_x4(t, wh + (n0 + p * 16 + b_row) * sw + k + b_col);
        bh[2 * p][0] = t[0]; bh[2 * p][1] = t[1]; bh[2 * p + 1][0] = t[2]; bh[2 * p + 1][1] = t[3];
        ldsm_x4(t, wl + (n0 + p * 16 + b_row) * sw + k + b_col);
        bl[2 * p][0] = t[0]; bl[2 * p][1] = t[1]; bl[2 * p + 1][0] = t[2]; bl[2 * p + 1][1] = t[3];
      }
    } else {
      uint32_t t[2];
      ldsm_x2(t, wh + (n0 + (lane & 7)) * sw + k + b_col);
      bh[0][0] = t[0]; bh[0][1] = t[1];
      ldsm_x2(t, wl + (n0 + (lane & 7)) * sw + k + b_col);
      bl[0][0] = t[0]; bl[0][1] = t[1];
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      uint32_t fh[4], fl[4];
      ldsm_x4(fh, ah + (m0 + mt * 16 + a_row) * SA + k + a_col);
      ldsm_x4(fl, al + (m0 + mt * 16 + a_row) * SA + k + a_col);
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) {
        mma_bf16(acc[mt][nt], fl, bh[nt][0], bh[nt][1]);   // small terms first
        mma_bf16(acc[mt][nt], fh, bl[nt][0], bl[nt][1]);
        mma_bf16(acc[mt][nt], fh, bh[nt][0], bh[nt][1]);
      }
    }
  }
}

// Write columns [0, ncol) of the activation tile (hi + lo) to a row-major fp32 global array (ncol even): a warp writes
// one row at a time as float2 (coalesced 256-byte segments, no integer division).  gtid: thread index in the group.
__device__ __forceinline__ void dump_tile(const __nv_bfloat16* ah, const __nv_bfloat16* al, float* dst, int ncol,
                                          int64_t base, int64_t total, int gtid) {
  const int lane = gtid & 31, warp = gtid >> 5;
  for (int row = warp; row < M; row += GT / 32) {
    if (base + row >= total) break;
    float* d = dst + (base + row) * ncol;
    for (int c = 2 * lane; c < ncol; c += 64) {
      const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(ah + row * SA + c);
      const __nv_bfloat162 l = *reinterpret_cast<const __nv_bfloat162*>(al + row * SA + c);
      *reinterpret_cast<float2*>(d + c) = make_float2(__bfloat162float(h.x) + __bfloat162float(l.x),
                                                     __bfloat162float(h.y) + __bfloat162float(l.y));
    }
  }
}

__global__ void __launch_bounds__(NT, 1) app_mlp_kernel(const MlpParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int n_jobs = p.n_jobs;
  const int job = (int)(blockIdx.x % n_jobs);
  const HeadJobDev& J = p.jobs[job];
  const TirMlp& mlp = J.mlp;
  const int out_dim = mlp.out_dim;
  const int light_mode = J.light_mode;
  const int act = J.act;

  // ---- stage split-BF16 weights once per CTA (PyTorch [out,in] layout is already the mma "col" operand)
  for (int i = tid; i < HID * SW0; i += NT) {
    const int h = i / SW0, k = i % SW0;
    split_bf16(k < IN ? __ldg(mlp.w0 + h * IN + k) : 0.f, s.w0h[i], s.w0l[i]);
  }
  for (int i = tid; i < HID * SW1; i += NT) {
    const int h = i / SW1, k = i % SW1;
    split_bf16(k < HID ? __ldg(mlp.w1 + h * HID + k) : 0.f, s.w1h[i], s.w1l[i]);
  }
  for (int i = tid; i < FN * SBS; i += NT) {
    const int n = i / SBS, k = i % SBS;
    split_bf16((n < F && k < K0) ? __ldg(mlp.basis + n * K0 + k) : 0.f, s.bsh[i], s.bsl[i]);
  }
  for (int i = tid; i < ON * SW2; i += NT) {
    const int n = i / SW2, k = i % SW2;
    split_bf16((n < out_dim && k < HID) ? __ldg(mlp.w2 + n * HID + k) : 0.f, s.w2h[i], s.w2l[i]);
  }
  for (int i = tid; i < HID; i += NT) { s.b0[i] = __ldg(mlp.b0 + i); s.b1[i] = __ldg(mlp.b1 + i); }
  if (tid < ON) s.b2[tid] = (tid < out_dim) ? __ldg(mlp.b2 + tid) : 0.f;
  if (light_mode == 2) {   // torch.mean(light_line(arange(L)), 0)  (tensoRF_rotated_lights.py:160-161)
    for (int c = tid; c < K0; c += NT) {
      float a = 0.f;
      for (int l = 0; l < mlp.n_lights; ++l) a += __ldg(mlp.light_line + (size_t)l * K0 + c);
      s.lmean[c] = a / (float)mlp.n_lights;
    }
  }
  __syncthreads();

  // ---- tiles: group grp of CTA c of this job takes tiles 2c + grp, +2 x (CTAs of the job), ...
  const int grp = tid / GT, gtid = tid % GT, gw = gtid >> 5;
  Tile& T = s.t[grp];
  const int64_t total = list_rows(p.n_points, p.n_dev);
  const int64_t n_tiles = (total + M - 1) / M;
  const int64_t tile0 = (int64_t)(blockIdx.x / n_jobs) * NG + grp;
  const int64_t tstep = (int64_t)(gridDim.x / n_jobs) * NG;

  for (int64_t tile = tile0; tile < n_tiles; tile += tstep) {
    const int64_t base = tile * M;
    // ---- point metadata
    if (gtid < M) {
      const int64_t i = base + gtid;
      float xn0 = 0.f, xn1 = 0.f, xn2 = 0.f, v0 = 0.f, v1 = 0.f, v2 = 0.f;
      int li = 0;
      if (i < total) {
        xn0 = J.xn[i * 3 + 0]; xn1 = J.xn[i * 3 + 1]; xn2 = J.xn[i * 3 + 2];
        const int64_t r = J.x_index ? (int64_t)J.x_index[i] : i;
        const float* xi = J.x_in + r * J.x_in_stride;
        v0 = xi[0]; v1 = xi[1]; v2 = xi[2];
        li = J.light_idx ? J.light_idx[r] : 0;
      }
      T.xn[gtid][0] = xn0; T.xn[gtid][1] = xn1; T.xn[gtid][2] = xn2;
      T.xv[gtid][0] = v0; T.xv[gtid][1] = v1; T.xv[gtid][2] = v2;
      T.light[gtid] = li;
    }
    group_sync(grp);

    // ---- phase 1: gather.  4 threads per sample, 12 channels of each orientation per thread -> A[m][0..143]
    {
      const int m = gtid >> 2, qd = gtid & 3;
      const float xn[3] = {T.xn[m][0], T.xn[m][1], T.xn[m][2]};
      const float* lrow = light_mode == 1 ? (mlp.light_line + (size_t)T.light[m] * K0)
                                          : (light_mode == 2 ? s.lmean : nullptr);
      float* x0_dst = (J.save_x0 && base + m < total) ? J.save_x0 + (base + m) * K0 : nullptr;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int m0 = kMat0[k], m1 = kMat1[k], v = kVec[k];
        const Bilinear b = bilinear_setup(xn[m0], xn[m1], p.f.grid[m0], p.f.grid[m1]);
        const Linear1 l = linear_setup(xn[v], p.f.grid[v]);
        const float* P = p.f.aplane[k];
        const float* L = p.f.aline[k];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const int c = qd * 12 + j * 4;
          const float4 pv = bilerp4(ldg4(P + (size_t)b.o00 * AC + c), ldg4(P + (size_t)b.o01 * AC + c),
                                    ldg4(P + (size_t)b.o10 * AC + c), ldg4(P + (size_t)b.o11 * AC + c), b);
          const float4 lv = lerp4(ldg4(L + (size_t)l.o0 * AC + c), ldg4(L + (size_t)l.o1 * AC + c), l);
          float4 x = make_float4(__fmul_rn(pv.x, lv.x), __fmul_rn(pv.y, lv.y), __fmul_rn(pv.z, lv.z),
                                 __fmul_rn(pv.w, lv.w));
          if (x0_dst) *reinterpret_cast<float4*>(x0_dst + k * AC + c) = x;   // raw products for the backward
          if (lrow) {   // (plane * line) * light  (tensoRF_rotated_lights.py:222)
            const float4 lc = *reinterpret_cast<const float4*>(lrow + k * AC + c);
            x.x = __fmul_rn(x.x, lc.x); x.y = __fmul_rn(x.y, lc.y); x.z = __fmul_rn(x.z, lc.z); x.w = __fmul_rn(x.w, lc.w);
          }
          const int col = k * AC + c;
          store_pair(T.ah, T.al, m * SA + col, x.x, x.y);
          store_pair(T.ah, T.al, m * SA + col + 2, x.z, x.w);
        }
      }
    }
    group_sync(grp);
    if (p.save_xl && job == 0) dump_tile(T.ah, T.al, p.save_xl, K0, base, total, gtid);

    // ---- phase 2: basis_mat (144 -> 27, N padded to 32): warp w -> m-tile w/2, n-tiles 2*(w%2), +1
    {
      float acc[1][2][4] = {};
      const int m0 = (gw >> 1) * 16, n0 = (gw & 1) * 16;
      warp_gemm<1, 2>(acc, T.ah, T.al, m0, s.bsh, s.bsl, SBS, n0, K0, lane);
      group_sync(grp);   // every warp has finished reading the gathered products; A is rewritten in place
      // MLP input [feat 27 | x 3 | sin PE(feat) 54 | cos 54 | sin PE(x) 6 | cos 6 | 0 pad 10]  (tensorBase:12-17,:136-142)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int row = m0 + g + half * 8;
          const int n = n0 + nt * 8 + 2 * t4;
          const float va = acc[0][nt][half * 2], vb = acc[0][nt][half * 2 + 1];
          if (n + 1 < F) {
            store_pair(T.ah, T.al, row * SA + n, va, vb);
          } else if (n < F) {
            store_one(T.ah, T.al, row * SA + n, va);
          }
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int nn = n + e;
            if (nn < F) {
              const float v = e ? vb : va;
              float s1, c1, s2, c2;
              sincosf(v, &s1, &c1);
              sincosf(__fmul_rn(v, 2.f), &s2, &c2);
              store_pair(T.ah, T.al, row * SA + 30 + 2 * nn, s1, s2);
              store_pair(T.ah, T.al, row * SA + 84 + 2 * nn, c1, c2);
            }
          }
        }
      if (gtid < M) {
        const int row = gtid;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          const float v = T.xv[row][d];
          store_one(T.ah, T.al, row * SA + 27 + d, v);
          float s1, c1, s2, c2;
          sincosf(v, &s1, &c1);
          sincosf(__fmul_rn(v, 2.f), &s2, &c2);
          store_pair(T.ah, T.al, row * SA + 138 + 2 * d, s1, s2);
          store_pair(T.ah, T.al, row * SA + 144 + 2 * d, c1, c2);
        }
#pragma unroll
        for (int c = IN; c < K1; c += 2) store_pair(T.ah, T.al, row * SA + c, 0.f, 0.f);
      }
    }
    group_sync(grp);
    if (J.save_in) dump_tile(T.ah, T.al, J.save_in, IN, base, total, gtid);

    // ---- phases 3/4: hidden layers.  warp w of the group -> all 32 rows x units [32w, 32w+32)
    auto hidden_layer = [&](const __nv_bfloat16* wh, const __nv_bfloat16* wl, int sw, const float* bias, int K) {
      float acc[2][4][4] = {};
      warp_gemm<2, 4>(acc, T.ah, T.al, 0, wh, wl, sw, gw * 32, K, lane);
      group_sync(grp);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int n = gw * 32 + nt * 8 + 2 * t4;
          const float ba = bias[n], bb = bias[n + 1];
          store_pair(T.ah, T.al, (mt * 16 + g) * SA + n, fmaxf(acc[mt][nt][0] + ba, 0.f), fmaxf(acc[mt][nt][1] + bb, 0.f));
          store_pair(T.ah, T.al, (mt * 16 + g + 8) * SA + n, fmaxf(acc[mt][nt][2] + ba, 0.f),
                     fmaxf(acc[mt][nt][3] + bb, 0.f));
        }
      group_sync(grp);
    };
    hidden_layer(s.w0h, s.w0l, SW0, s.b0, K1);
    if (J.save_h1) dump_tile(T.ah, T.al, J.save_h1, HID, base, total, gtid);
    hidden_layer(s.w1h, s.w1l, SW1, s.b1, HID);
    if (J.save_h2) dump_tile(T.ah, T.al, J.save_h2, HID, base, total, gtid);

    // ---- phase 5: output layer (N padded to 8) on warps 0..1 of the group, activation
    if (gw < M / 16) {
      float acc[1][1][4] = {};
      warp_gemm<1, 1>(acc, T.ah, T.al, gw * 16, s.w2h, s.w2l, SW2, 0, HID, lane);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = gw * 16 + g + (e >> 1) * 8;
        const int o = 2 * t4 + (e & 1);
        if (o < out_dim) {
          const float a = acc[0][0][e] + s.b2[o];
          const float y = act == 0 ? 1.f / (1.f + expf(-a)) : tanhf(a);
          const int64_t i = base + row;
          if (i < total) J.out[i * J.out_stride + o] = y;
        }
      }
    }
    group_sync(grp);
  }
}

int check_shapes(const TirField* f, const TirMlp* m) {
  if (f->aC != AC) return TIR_ERR_SHAPE;
  if (m->feat_dim != F || m->hidden != HID || m->pe_feat != 2 || m->pe_x != 2) return TIR_ERR_SHAPE;
  if (m->out_dim < 1 || m->out_dim > 4) return TIR_ERR_SHAPE;
  if (!m->w0 || !m->b0 || !m->w1 || !m->b1 || !m->w2 || !m->b2 || !m->basis) return TIR_ERR_NULL;
  return TIR_OK;
}

int launch(const MlpParams& p, int64_t n, cudaStream_t stream) {
  static bool configured = false;
  const int smem = (int)sizeof(Smem);
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(app_mlp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int64_t ctas = (n + NG * M - 1) / (NG * M);     // a CTA has NG tiles in flight
  const int nj = p.n_jobs;
  int per_job = num_sms() / nj;                            // CTAs per job: one wave, one CTA per SM
  if (ctas < per_job) per_job = (int)(ctas > 0 ? ctas : 1);
  app_mlp_kernel<<<per_job * nj, NT, smem, stream>>>(p);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" int tir_app_mlp_points_save(const TirField* field, const TirMlp* mlp, const float* xn, const float* x_in,
                                       const int32_t* light_idx, int64_t n, int32_t act, float* out, float* save_xl,
                                       float* save_in, float* save_h1, float* save_h2, void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !mlp || !xn || !x_in || !out) return TIR_ERR_NULL;
  int rc = check_shapes(field, mlp);
  if (rc) return rc;
  if (act != 0 && act != 1) return TIR_ERR_CONFIG;
  MlpParams p{};
  p.f = *field; p.n_jobs = 1; p.n_points = n; p.n_dev = nullptr; p.save_xl = save_xl;
  HeadJobDev& J = p.jobs[0];
  J.mlp = *mlp; J.xn = xn; J.x_in = x_in; J.x_index = nullptr; J.x_in_stride = 3; J.light_idx = light_idx;
  J.light_mode = mlp->light_line ? 1 : 0; J.act = act; J.out = out; J.out_stride = mlp->out_dim;
  J.save_in = save_in; J.save_h1 = save_h1; J.save_h2 = save_h2;
  return launch(p, n, (cudaStream_t)stream);
}

namespace tir {
int launch_heads_forward(const TirField& f, const HeadJobDev* jobs, int n_jobs, int64_t n, const int64_t* n_dev,
                         cudaStream_t stream) {
  if (n <= 0 || n_jobs <= 0) return TIR_OK;
  if (n_jobs > kMaxHeadJobs) return TIR_ERR_CONFIG;
  MlpParams p{};
  p.f = f; p.n_jobs = n_jobs; p.n_points = n; p.n_dev = n_dev;
  for (int j = 0; j < n_jobs; ++j) {
    int rc = check_shapes(&f, &jobs[j].mlp);
    if (rc) return rc;
    if (!jobs[j].xn || !jobs[j].x_in || !jobs[j].out) return TIR_ERR_NULL;
    if (jobs[j].light_mode != 0 && !jobs[j].mlp.light_line) return TIR_ERR_NULL;
    p.jobs[j] = jobs[j];
  }
  return launch(p, n, stream);
}
}  // namespace tir
