// Backward of the appearance heads (the four 150-128-128-{3,4} MLPs of the primary march, basis_mat, light_line and
// the positional encoding) on the activations dumped by the fused forward (tir_mlp.cu, launch_heads_forward).
// Replaces the autograd graph of MLPRender_Fea / MLPBRDF_PEandFeature (tensorBase_rotated_lights.py:122-146,:182-208)
// and compute_{app,intrin}feature's tail (tensoRF_rotated_lights.py:155-224): in round 1 this was ~300 cuBLAS SIMT
// sgemm / elementwise launches per step; here it is TWO launches for all heads of a step:
//
//   heads_dgrad_kernel   per 32-sample tile, two tiles in flight per CTA: d out -> d z3 -> (W2) -> ReLU' -> (W1^T GEMM)
//                        -> ReLU' -> (W0^T GEMM) -> positional-encoding backward -> d feat -> (basis^T) ->
//                        d (plane*line*light) -> * light -> gx0,
//                        plus the light_line gradient; dumps d z1 / d z2 / d feat for the weight gradients.
//   heads_wgrad_kernel   split-K weight gradients  gW1 = dz2^T h1,  gW0 = dz1^T inp  on the tensor cores (operands are
//                        read "transposed" straight from the row-major tiles with ldmatrix.trans), bias column sums,
//                        gW2 / gb2 / g basis_mat on the CUDA cores; accumulated into the gradient buffers with atomics.
//
// Tensor-core products use the same error-compensated BF16 split as the forward (hi*hi + hi*lo + lo*hi, fp32
// accumulate), so gradients agree with fp32 autograd to ~1e-5 relative.  CTAs are partitioned over the heads
// (and, for the weight gradients, over roles and row slices); every list length may come from a device-side count.
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
constexpr int GIN = 144;          // columns of d input that are needed: [0,27) feat, [30,84) sin, [84,138) cos (pad 144)
constexpr int M = 64;
constexpr int NT = 512;          // 16 warps: the kernels are latency bound, registers are capped at 128
constexpr int SA = 136;           // bf16 row stride of [*,128] tiles (272 B: odd multiple of 16 B)
constexpr int SB = 168;           // bf16 row stride of [*,160] tiles
constexpr int LMAX = 8;           // light rows accumulated in shared memory (more lights fall back to global atomics)
constexpr int GF = 32;            // row stride of the d feat scratch
constexpr int SF = 40;            // bf16 row stride of [*,32] tiles (80 B: odd multiple of 16 B)

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
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __nv_bfloat16* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const __nv_bfloat16* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[MT][2] (m16 x n16) += A[m0.., :K] * W[n0.., :K]^T, A row-major [M][SA], W row-major [N][sw] (hi/lo split)
template <int MT>
__device__ __forceinline__ void warp_gemm_nt(float (&acc)[MT][2][4], const __nv_bfloat16* ah, const __nv_bfloat16* al,
                                             int m0, const __nv_bfloat16* wh, const __nv_bfloat16* wl, int sw, int n0,
                                             int K, int lane, int sa = SA) {
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;
  const int a_col = (lane >> 4) * 8;
  const int b_row = (lane & 7) + (lane >> 4) * 8;
  const int b_col = ((lane >> 3) & 1) * 8;
  for (int k = 0; k < K; k += 16) {
    uint32_t bh[4], bl[4];
    ldsm_x4(bh, wh + (n0 + b_row) * sw + k + b_col);
    ldsm_x4(bl, wl + (n0 + b_row) * sw + k + b_col);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      uint32_t fh[4], fl[4];
      ldsm_x4(fh, ah + (m0 + mt * 16 + a_row) * sa + k + a_col);
      ldsm_x4(fl, al + (m0 + mt * 16 + a_row) * sa + k + a_col);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        mma_bf16(acc[mt][nt], fl, bh[nt * 2], bh[nt * 2 + 1]);
        mma_bf16(acc[mt][nt], fh, bl[nt * 2], bl[nt * 2 + 1]);
        mma_bf16(acc[mt][nt], fh, bh[nt * 2], bh[nt * 2 + 1]);
      }
    }
  }
}

// store(i, load(i)) for i = threadIdx.x, + blockDim.x, ... < n: a CTA-wide copy of read-only global data into shared
// memory.  Each thread issues U loads before it stores any, so U loads are in flight per thread instead of one.
template <int U, class Load, class Store>
__device__ __forceinline__ void staged_fill(int n, Load load, Store store) {
  const int step = (int)blockDim.x;
  for (int i0 = (int)threadIdx.x; i0 < n; i0 += U * step) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = i0 + u * step < n ? load(i0 + u * step) : 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (i0 + u * step < n) store(i0 + u * step, v[u]);
  }
}

__device__ __forceinline__ float act_grad(int act, float y) { return act == 0 ? y * (1.f - y) : 1.f - y * y; }

// ---------------------------------------------------------------------------------------------------------------------
// data gradient
// ---------------------------------------------------------------------------------------------------------------------
constexpr int DM = 32;            // rows of a dgrad tile
constexpr int DG = 2;             // dgrad warp groups per CTA, one tile in flight each
constexpr int DGT = NT / DG;      // threads per dgrad group (8 warps)

struct __align__(16) DgradTile {  // one warp group's tile
  union {
    struct { __nv_bfloat16 h[DM * SA], l[DM * SA]; } a;   // activation-gradient tile (A operand)
    float gin[DM * GIN];                                  // d input of the MLP after the last GEMM
  } u;
  __nv_bfloat16 gfh[DM * SF], gfl[DM * SF];        // d feat tile (A operand of the basis GEMM)
  float gz3[DM * 4];
  int light[DM];
};

struct DgradSmem {
  __nv_bfloat16 w1h[HID * SA], w1l[HID * SA];     // W1^T: [in][out]
  __nv_bfloat16 w0h[GIN * SA], w0l[GIN * SA];     // W0^T: [in < 144][out]
  __nv_bfloat16 bth[K0 * SF], btl[K0 * SF];        // basis^T: [c][f] (f padded to 32)
  DgradTile t[DG];
  float w2[4 * HID];
  float glight[LMAX * K0];
  float lmean[K0];
};

// The named barrier of dgrad warp group `grp` (barrier 0 is __syncthreads).
__device__ __forceinline__ void group_sync(int grp) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(grp + 1), "r"(DGT) : "memory");
}

struct DgradParams {
  TirField f;
  HeadBwdJob jobs[kMaxHeadJobs];
  HeadsBwdShared sh;
  int n_jobs;
  int64_t n;
  const int64_t* n_dev;
};

__global__ void __launch_bounds__(NT, 1) heads_dgrad_kernel(const DgradParams p) {
  // two groups of 8 warps, each on its own 32-row tile; warp w of a group: column block w (16 columns) of every
  // 32 x 128 GEMM output
  extern __shared__ __align__(128) unsigned char smem_raw[];
  DgradSmem& s = *reinterpret_cast<DgradSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int job = (int)(blockIdx.x % p.n_jobs);
  const HeadBwdJob& J = p.jobs[job];
  const TirMlp& mlp = J.mlp;
  const int od = mlp.out_dim, L = mlp.n_lights;
  const int mode = J.light_mode;

  // ---- stage transposed split-BF16 weights (coalesced global reads; the one-off smem bank conflicts are irrelevant)
  constexpr int U = 8;   // staged loads in flight per thread
  staged_fill<U>(HID * HID, [&](int i) { return __ldg(mlp.w1 + i); }, [&](int i, float v) {
    const int o = i / HID, k = i % HID;          // W1[o][k]  ->  w1T[k][o]
    split_bf16(v, s.w1h[k * SA + o], s.w1l[k * SA + o]);
  });
  staged_fill<U>(HID * IN, [&](int i) { return __ldg(mlp.w0 + i); }, [&](int i, float v) {
    const int o = i / IN, k = i % IN;            // W0[o][k]  ->  w0T[k][o], k < 144 only
    if (k < GIN) split_bf16(v, s.w0h[k * SA + o], s.w0l[k * SA + o]);
  });
  staged_fill<U>(K0 * SF, [&](int i) {
                   const int c = i / SF, f = i % SF;
                   return f < F ? __ldg(mlp.basis + f * K0 + c) : 0.f;
                 },
                 [&](int i, float v) { split_bf16(v, s.bth[i], s.btl[i]); });   // basis[f][c] -> bT[c][f]
  for (int i = tid; i < DG * DM * SF; i += NT) {
    s.t[i / (DM * SF)].gfh[i % (DM * SF)] = __float2bfloat16_rn(0.f);
    s.t[i / (DM * SF)].gfl[i % (DM * SF)] = __float2bfloat16_rn(0.f);
  }
  for (int i = tid; i < 4 * HID; i += NT) s.w2[i] = (i / HID) < od ? __ldg(mlp.w2 + i) : 0.f;
  for (int i = tid; i < LMAX * K0; i += NT) s.glight[i] = 0.f;
  if (mode == 2)
    for (int c = tid; c < K0; c += NT) {
      float a = 0.f;
      for (int l = 0; l < L; ++l) a += __ldg(mlp.light_line + (size_t)l * K0 + c);
      s.lmean[c] = a / (float)L;
    }
  __syncthreads();

  const int grp = tid / DGT, gtid = tid % DGT, gw = gtid >> 5;
  DgradTile& T = s.t[grp];
  const int64_t total = list_rows(p.n, p.n_dev);
  const int64_t n_tiles = (total + DM - 1) / DM;
  const float* x0 = p.sh.x0[J.point_set];

  for (int64_t tile = (blockIdx.x / p.n_jobs) * DG + grp; tile < n_tiles; tile += (gridDim.x / p.n_jobs) * DG) {
    const int64_t base = tile * DM;
    // ---- a. d z3 = d out * act'(out)
    {
      const int row = gtid >> 2, o = gtid & 3;
      const int64_t i = base + row;
      float v = 0.f;
      if (row < DM && i < total && o < od)
        v = J.g_out[i * J.out_stride + o] * act_grad(J.act, J.out[i * J.out_stride + o]);
      if (row < DM) T.gz3[row * 4 + o] = v;
      if (gtid < DM) {
        const int64_t ii = base + gtid;
        int li = 0;
        if (ii < total && mode == 1 && J.light_idx) li = J.light_idx[J.x_index ? (int64_t)J.x_index[ii] : ii];
        T.light[gtid] = li;
      }
    }
    group_sync(grp);
    // ---- b. d z2 = (d z3 @ W2) * [h2 > 0]   (K = out_dim <= 4: CUDA cores).  A thread's h2 loads are issued
    //         before its d z2 stores, which the compiler may not move them past.
    constexpr int BN = DM * (HID / 2) / DGT;
    float2 hb[BN];
#pragma unroll
    for (int u = 0; u < BN; ++u) {
      const int idx = gtid + u * DGT, row = idx / (HID / 2), k = (idx % (HID / 2)) * 2;
      hb[u] = base + row < total ? *reinterpret_cast<const float2*>(J.h2 + (base + row) * HID + k)
                                 : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < BN; ++u) {
      const int idx = gtid + u * DGT;
      const int row = idx / (HID / 2), k = (idx % (HID / 2)) * 2;
      const int64_t i = base + row;
      float va = 0.f, vb = 0.f;
      if (i < total) {
        const float2 h = hb[u];
        const float z0 = T.gz3[row * 4], z1 = T.gz3[row * 4 + 1], z2 = T.gz3[row * 4 + 2], z3 = T.gz3[row * 4 + 3];
        va = z0 * s.w2[k] + z1 * s.w2[HID + k] + z2 * s.w2[2 * HID + k] + z3 * s.w2[3 * HID + k];
        vb = z0 * s.w2[k + 1] + z1 * s.w2[HID + k + 1] + z2 * s.w2[2 * HID + k + 1] + z3 * s.w2[3 * HID + k + 1];
        va = h.x > 0.f ? va : 0.f;
        vb = h.y > 0.f ? vb : 0.f;
        *reinterpret_cast<float2*>(J.gz2 + i * HID + k) = make_float2(va, vb);
      }
      store_pair(T.u.a.h, T.u.a.l, row * SA + k, va, vb);
    }
    group_sync(grp);
    // ---- c. d z1 = (d z2 @ W1) * [h1 > 0]
    const int nb = gw;
    {
      float acc[2][2][4] = {};
      warp_gemm_nt<2>(acc, T.u.a.h, T.u.a.l, 0, s.w1h, s.w1l, SA, nb * 16, HID, lane);
      float2 h1v[2][2][2];      // the thread's h1 entries, loaded before its first d z1 store
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int64_t i = base + mt * 16 + g + half * 8;
            h1v[mt][nt][half] = i < total ? *reinterpret_cast<const float2*>(J.h1 + i * HID + nb * 16 + nt * 8 + 2 * t4)
                                          : make_float2(0.f, 0.f);
          }
      group_sync(grp);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = mt * 16 + g + half * 8;
            const int col = nb * 16 + nt * 8 + 2 * t4;
            const int64_t i = base + row;
            float va = 0.f, vb = 0.f;
            if (i < total) {
              const float2 h = h1v[mt][nt][half];
              va = h.x > 0.f ? acc[mt][nt][half * 2] : 0.f;
              vb = h.y > 0.f ? acc[mt][nt][half * 2 + 1] : 0.f;
              *reinterpret_cast<float2*>(J.gz1 + i * HID + col) = make_float2(va, vb);
            }
            store_pair(T.u.a.h, T.u.a.l, row * SA + col, va, vb);
          }
    }
    group_sync(grp);
    // ---- d. d input = d z1 @ W0   (columns [0,144) only: the 3-vector and its encoding carry no gradient)
    {
      float acc[2][2][4] = {};
      float acx[1][2][4] = {};
      warp_gemm_nt<2>(acc, T.u.a.h, T.u.a.l, 0, s.w0h, s.w0l, SA, nb * 16, HID, lane);
      if (gw < DM / 16) warp_gemm_nt<1>(acx, T.u.a.h, T.u.a.l, gw * 16, s.w0h, s.w0l, SA, HID, HID, lane);
      group_sync(grp);          // every warp of the group is done reading the tile that `gin` aliases
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = mt * 16 + g + half * 8, col = nb * 16 + nt * 8 + 2 * t4;
            *reinterpret_cast<float2*>(T.u.gin + row * GIN + col) =
                make_float2(acc[mt][nt][half * 2], acc[mt][nt][half * 2 + 1]);
          }
      if (gw < DM / 16) {
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = gw * 16 + g + half * 8, col = HID + nt * 8 + 2 * t4;
            *reinterpret_cast<float2*>(T.u.gin + row * GIN + col) =
                make_float2(acx[0][nt][half * 2], acx[0][nt][half * 2 + 1]);
          }
      }
    }
    group_sync(grp);
    // ---- e. positional-encoding backward: d feat_f = d in_f + sum_p 2^p (d sin_fp * cos_fp - d cos_fp * sin_fp);
    //         the dumped sin / cos of all a thread's entries are loaded before its d feat stores
    constexpr int EN = (DM * F + DGT - 1) / DGT;
    float4 sc[EN];            // sin 2^0, sin 2^1, cos 2^0, cos 2^1 of feature f
#pragma unroll
    for (int u = 0; u < EN; ++u) {
      const int idx = gtid + u * DGT, row = idx / F, f = idx % F;
      sc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < DM * F && base + row < total) {
        const float* in = J.inp + (base + row) * IN;
        sc[u] = make_float4(in[30 + 2 * f], in[31 + 2 * f], in[84 + 2 * f], in[85 + 2 * f]);
      }
    }
#pragma unroll
    for (int u = 0; u < EN; ++u) {
      const int idx = gtid + u * DGT;
      if (idx >= DM * F) break;
      const int row = idx / F, f = idx % F;
      const int64_t i = base + row;
      float v = 0.f;
      if (i < total) {
        const float* gi = T.u.gin + row * GIN;
        v = gi[f] + (gi[30 + 2 * f] * sc[u].z - gi[84 + 2 * f] * sc[u].x) +
            2.f * (gi[31 + 2 * f] * sc[u].w - gi[85 + 2 * f] * sc[u].y);
        J.gfeat[i * GF + f] = v;
      }
      split_bf16(v, T.gfh[row * SF + f], T.gfl[row * SF + f]);
    }
    group_sync(grp);
    // ---- f. d (products * light) = d feat @ basis (tensor cores: K = 32, N = 144);  gx0 = that * light row;
    //         light_line gradient = sum over samples of d(...) * raw products
    {
      // 9 column blocks of 16 over the tile's 32 rows: warps 0..7 of the group take one, warp 0 the ninth
      for (int cb = gw; cb < 9; cb += DGT / 32) {
        float acc[2][2][4] = {};
        warp_gemm_nt<2>(acc, T.gfh, T.gfl, 0, s.bth, s.btl, SF, cb * 16, 32, lane, SF);
        float gl[2][2][4];            // d(...) * raw products: the light_line gradient contributions
        // the light factors and raw products of the thread's entries, loaded before its first gx0 store
        float2 lf[2][2][2], xr[2][2][2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int row = mt * 16 + g + half * 8, c = cb * 16 + nt * 8 + 2 * t4;
              const int64_t i = base + row;
              lf[mt][nt][half] = make_float2(1.f, 1.f);
              xr[mt][nt][half] = make_float2(0.f, 0.f);
              if (i >= total) continue;
              if (mode == 1)
                lf[mt][nt][half] =
                    __ldg(reinterpret_cast<const float2*>(mlp.light_line + (size_t)T.light[row] * K0 + c));
              else if (mode == 2)
                lf[mt][nt][half] = make_float2(s.lmean[c], s.lmean[c + 1]);
              if (mode != 0) xr[mt][nt][half] = __ldg(reinterpret_cast<const float2*>(x0 + i * K0 + c));
            }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int row = mt * 16 + g + half * 8, c = cb * 16 + nt * 8 + 2 * t4;
              const int64_t i = base + row;
              gl[mt][nt][half * 2] = 0.f; gl[mt][nt][half * 2 + 1] = 0.f;
              if (i >= total) continue;
              const float a0 = acc[mt][nt][half * 2], a1 = acc[mt][nt][half * 2 + 1];
              const float2 lv = lf[mt][nt][half];
              *reinterpret_cast<float2*>(J.gx0 + i * K0 + c) = make_float2(a0 * lv.x, a1 * lv.y);
              if (mode != 0) {
                const float2 xv = xr[mt][nt][half];
                gl[mt][nt][half * 2] = a0 * xv.x; gl[mt][nt][half * 2 + 1] = a1 * xv.y;
              }
            }
        if (mode != 0) {
          // Sum over the warp's 32 rows BEFORE touching shared memory: per light row, add the thread's 4 rows, then
          // butterfly over the 8 row lanes; lanes g == 0 own distinct columns (no same-address atomics in a warp).
          const int nl = mode == 2 ? 1 : (L < LMAX ? L : LMAX);
          for (int l = 0; l < nl; ++l) {
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                float v = 0.f;
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                  for (int half = 0; half < 2; ++half) {
                    const int row = mt * 16 + g + half * 8;
                    if (mode == 2 || T.light[row] == l) v += gl[mt][nt][half * 2 + e];
                  }
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (g == 0 && v != 0.f) atomicAdd(&s.glight[l * K0 + cb * 16 + nt * 8 + 2 * t4 + e], v);
              }
          }
          if (mode == 1 && L > LMAX) {           // rare: more lights than shared rows -> straight to global memory
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
              for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const int row = mt * 16 + g + (e >> 1) * 8, lr = T.light[row];
                  if (lr >= LMAX && gl[mt][nt][e] != 0.f)
                    atomicAdd(p.sh.g_light + (size_t)lr * K0 + cb * 16 + nt * 8 + 2 * t4 + (e & 1), gl[mt][nt][e]);
                }
          }
        }
      }
    }
    group_sync(grp);
  }
  __syncthreads();            // both groups have added their light_line sums
  // ---- flush the light_line gradient
  if (mode == 1) {
    const int rows = L < LMAX ? L : LMAX;
    for (int i = tid; i < rows * K0; i += NT)
      if (s.glight[i] != 0.f) atomicAdd(p.sh.g_light + i, s.glight[i]);
  } else if (mode == 2) {     // forward used the mean row: every light row receives 1/L of the gradient
    for (int c = tid; c < K0; c += NT) {
      const float v = s.glight[c] / (float)L;
      if (v != 0.f)
        for (int l = 0; l < L; ++l) atomicAdd(p.sh.g_light + (size_t)l * K0 + c, v);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// weight gradients
// ---------------------------------------------------------------------------------------------------------------------
struct WgradSmem {
  __nv_bfloat16 ah[M * SA], al[M * SA];     // d z tile   [row][out]   (small role: d feat in cols 0..31, d z3 in 32..47)
  __nv_bfloat16 bh[M * SB], bl[M * SB];     // activation tile [row][in]   (small role: products * light, 144 cols)
  __nv_bfloat16 ch[M * SA], cl[M * SA];     // small role: h2 tile
  float colsum[8 * HID];
  float stage_gz[M * HID];                  // big roles: fp32 rows of the next tile, landing while this one multiplies
  float stage_act[M * IN];
};

// Cost of one row of each weight-gradient role, relative to gW1 (= 1): gW0 loads 150 columns against 128 and runs
// 10 n8-tiles per warp against 8; the small role (gW2, gb2, g basis_mat) loads ~310 floats per row, partly gathered
// through the light index, with no prefetch.  Chosen by timing the kernel in the bench step on H100 (4 heads,
// 33 CTAs each): small-role costs 1.0 / 1.5 / 2.0 / 2.5 / 3.0 / 3.5 gave 249 / 215 / 178 / 170 / 185 / 184 µs, and a
// gW0 cost of 1.0 or 1.4 instead of 1.2 was slower.
constexpr float kRowCostW0 = 1.2f;
constexpr float kRowCostSmall = 2.5f;

// Row slices (CTAs) per head for gW1, gW0 and the small role, from the CTAs a head may use: the split with the
// smallest largest per-CTA cost, so that the roles of one head finish together.
struct WgradSplit { int p1, p0, ps; };
WgradSplit wgrad_split(int ctas) {
  WgradSplit best{1, 1, 1};
  float best_cost = 3.4e38f;
  for (int p1 = 1; p1 <= ctas - 2; ++p1)
    for (int p0 = 1; p1 + p0 <= ctas - 1; ++p0) {
      const int ps = ctas - p1 - p0;
      const float c = fmaxf(fmaxf(1.f / p1, kRowCostW0 / p0), kRowCostSmall / ps);
      if (c < best_cost) { best_cost = c; best = WgradSplit{p1, p0, ps}; }
    }
  return best;
}

// acc[NT8][4] += A^T B over one 64-row tile: rows m0..m0+15 of the gradient (A columns), columns n0.. (B columns).
// A stored [k][m] (stride sa), B stored [k][n] (stride sb): both read transposed with ldmatrix.trans.
template <int NT8>
__device__ __forceinline__ void wgrad_tile(float (&acc)[NT8][4], const __nv_bfloat16* ah, const __nv_bfloat16* al,
                                           int sa, int m0, const __nv_bfloat16* bh, const __nv_bfloat16* bl, int sb,
                                           int n0, int lane) {
  const int i8 = lane >> 3, r = lane & 7;
#pragma unroll
  for (int k = 0; k < M; k += 16) {
    uint32_t fa[4], fl[4];
    // A = (d z)^T: matrices (k0-7,m0-7) (k0-7,m8-15) (k8-15,m0-7) (k8-15,m8-15)
    ldsm_x4_t(fa, ah + (k + (i8 >> 1) * 8 + r) * sa + m0 + (i8 & 1) * 8);
    ldsm_x4_t(fl, al + (k + (i8 >> 1) * 8 + r) * sa + m0 + (i8 & 1) * 8);
#pragma unroll
    for (int n2 = 0; n2 < NT8 / 2; ++n2) {
      uint32_t gb[4], gl[4];
      // B: matrices (k0-7,n0-7) (k8-15,n0-7) (k0-7,n8-15) (k8-15,n8-15)
      ldsm_x4_t(gb, bh + (k + (i8 & 1) * 8 + r) * sb + n0 + n2 * 16 + (i8 >> 1) * 8);
      ldsm_x4_t(gl, bl + (k + (i8 & 1) * 8 + r) * sb + n0 + n2 * 16 + (i8 >> 1) * 8);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mma_bf16(acc[n2 * 2 + h], fl, gb[h * 2], gb[h * 2 + 1]);
        mma_bf16(acc[n2 * 2 + h], fa, gl[h * 2], gl[h * 2 + 1]);
        mma_bf16(acc[n2 * 2 + h], fa, gb[h * 2], gb[h * 2 + 1]);
      }
    }
  }
}

// Copy rows [base, min(base + M, r1)) of a row-major fp32 [*, ncol] array into dst ([M][ncol]) with 16-byte cp.async,
// zero-filling the rest of the tile.  The tile's rows are contiguous, so it is copied as one flat range: with base a
// multiple of 64 and a 16-byte aligned src, every chunk is aligned for ncol = 128 and 150.  Not waited for here.
__device__ __forceinline__ void prefetch_tile(float* dst, const float* src, int ncol, int64_t base, int64_t r1) {
  const int64_t rows = r1 - base < M ? r1 - base : M;
  const int valid = (int)rows * ncol * 4;                // bytes
  const float* s = src + base * ncol;
  for (int c = threadIdx.x; c < M * ncol / 4; c += NT) {
    const int left = valid - c * 16;
    const int n = left < 0 ? 0 : (left > 16 ? 16 : left);
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst + c * 4);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(n ? s + c * 4 : s), "r"(n) : "memory");
  }
  asm volatile("cp.async.commit_group;\n" ::: "memory");
}

// g_w[128][ld] += (d z)^T @ act  over rows [r0, r1);  g_b[128] += column sums of d z.
// 16 warps: warp w owns gradient rows 16 (w % 8).. and the column half w / 8 (NT8H n8-tiles).
// The fp32 rows of tile t + 1 are fetched into stage_* while tile t is multiplied.
template <int NT8H>
__device__ void wgrad_big(WgradSmem& s, const float* __restrict__ gz, const float* __restrict__ actv, int ncol, int ld,
                          int64_t r0, int64_t r1, float* g_w, float* g_b) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int mt = warp & 7, nh = warp >> 3;
  float acc[NT8H][4] = {};
  float cs0 = 0.f, cs1 = 0.f;                 // columns 2 (tid % 64), +1 of d z (512 % 64 == 0: fixed per thread)
  prefetch_tile(s.stage_gz, gz, HID, r0, r1);
  prefetch_tile(s.stage_act, actv, ncol, r0, r1);
  for (int i = tid; i < M * SB; i += NT) { s.bh[i] = __float2bfloat16_rn(0.f); s.bl[i] = __float2bfloat16_rn(0.f); }
  const int half_cols = ncol / 2;             // 64 or 75 float2 per row
  for (int64_t base = r0; base < r1; base += M) {
    // the staged tile has landed, and every warp is done with the previous tile's MMAs
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncthreads();
    for (int idx = tid; idx < M * (HID / 2); idx += NT) {
      const int row = idx / (HID / 2), k = (idx % (HID / 2)) * 2;
      const float2 v = *reinterpret_cast<const float2*>(s.stage_gz + row * HID + k);
      cs0 += v.x; cs1 += v.y;
      store_pair(s.ah, s.al, row * SA + k, v.x, v.y);
    }
    for (int idx = tid; idx < M * half_cols; idx += NT) {
      const int row = idx / half_cols, k = (idx % half_cols) * 2;
      const float2 v = *reinterpret_cast<const float2*>(s.stage_act + row * ncol + k);
      store_pair(s.bh, s.bl, row * SB + k, v.x, v.y);
    }
    __syncthreads();
    if (base + M < r1) {
      prefetch_tile(s.stage_gz, gz, HID, base + M, r1);
      prefetch_tile(s.stage_act, actv, ncol, base + M, r1);
    }
    wgrad_tile<NT8H>(acc, s.ah, s.al, SA, mt * 16, s.bh, s.bl, SB, nh * NT8H * 8, lane);
  }
#pragma unroll
  for (int nt = 0; nt < NT8H; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int m = mt * 16 + g + (e >> 1) * 8, n = nh * NT8H * 8 + nt * 8 + 2 * t4 + (e & 1);
      if (n < ncol && acc[nt][e] != 0.f) atomicAdd(g_w + (size_t)m * ld + n, acc[nt][e]);
    }
  const int kk = (tid % (HID / 2)) * 2, grp = tid / (HID / 2);
  s.colsum[grp * HID + kk] = cs0;
  s.colsum[grp * HID + kk + 1] = cs1;
  __syncthreads();
  if (tid < HID) {
    float v = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) v += s.colsum[q * HID + tid];
    if (v != 0.f) atomicAdd(g_b + tid, v);
  }
}

struct WgradParams {
  HeadBwdJob jobs[kMaxHeadJobs];
  HeadsBwdShared sh;
  int n_jobs;
  WgradSplit split;
  int64_t n;
  const int64_t* n_dev;
};

// gW2 [od,128] = dz3^T h2, gb2, g basis_mat [27,144] += d feat^T (products * light), all on the tensor cores
__device__ void wgrad_small(WgradSmem& s, const HeadBwdJob& J, const HeadsBwdShared& sh, int64_t r0, int64_t r1) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int od = J.mlp.out_dim, mode = J.light_mode, L = J.mlp.n_lights;
  const float* x0 = sh.x0[J.point_set];
  float accb[2][2][4] = {};       // basis: m-tile warp % 2, column blocks warp / 2 (and 8 for warps 0, 1)
  float acc2[2][4] = {};          // gW2: warps 0..7, column block = warp
  float bsum = 0.f;               // gb2: thread tid < 4 * 64 sums d z3[:, tid % 4] over rows tid / 4 (+64 k)
  for (int i = tid; i < M * SA; i += NT) { s.ah[i] = __float2bfloat16_rn(0.f); s.al[i] = __float2bfloat16_rn(0.f); }
  if (mode == 2)
    for (int c = tid; c < K0; c += NT) {
      float a = 0.f;
      for (int l = 0; l < L; ++l) a += __ldg(J.mlp.light_line + (size_t)l * K0 + c);
      s.colsum[c] = a / (float)L;
    }
  __syncthreads();
  for (int64_t base = r0; base < r1; base += M) {
    // d feat tile -> A cols 0..31
    for (int idx = tid; idx < M * 16; idx += NT) {
      const int row = idx / 16, k = (idx % 16) * 2;
      float2 v = make_float2(0.f, 0.f);
      if (base + row < r1 && k < F + 1) {
        v = *reinterpret_cast<const float2*>(J.gfeat + (base + row) * GF + k);
        if (k + 1 >= F) v.y = 0.f;
      }
      store_pair(s.ah, s.al, row * SA + k, v.x, v.y);
    }
    // d z3 tile -> A cols 32..47 (cols >= out_dim zero) + bias sums
    if (tid < M * 4) {
      const int row = tid >> 2, o = tid & 3;
      const int64_t i = base + row;
      float v = 0.f;
      if (i < r1 && o < od) v = J.g_out[i * J.out_stride + o] * act_grad(J.act, J.out[i * J.out_stride + o]);
      bsum += v;
      __nv_bfloat16 h, l;
      split_bf16(v, h, l);
      s.ah[row * SA + 32 + o] = h;
      s.al[row * SA + 32 + o] = l;
    }
    // products * light -> B (144 cols)
    for (int idx = tid; idx < M * (K0 / 2); idx += NT) {
      const int row = idx / (K0 / 2), c = (idx % (K0 / 2)) * 2;
      const int64_t i = base + row;
      float2 v = make_float2(0.f, 0.f);
      if (i < r1) {
        v = *reinterpret_cast<const float2*>(x0 + i * K0 + c);
        if (mode == 1) {
          const int li = J.light_idx ? J.light_idx[J.x_index ? (int64_t)J.x_index[i] : i] : 0;
          const float2 lv = __ldg(reinterpret_cast<const float2*>(J.mlp.light_line + (size_t)li * K0 + c));
          v.x *= lv.x; v.y *= lv.y;
        } else if (mode == 2) {
          v.x *= s.colsum[c]; v.y *= s.colsum[c + 1];
        }
      }
      store_pair(s.bh, s.bl, row * SB + c, v.x, v.y);
    }
    // h2 tile -> C
    for (int idx = tid; idx < M * (HID / 2); idx += NT) {
      const int row = idx / (HID / 2), k = (idx % (HID / 2)) * 2;
      float2 v = make_float2(0.f, 0.f);
      if (base + row < r1) v = *reinterpret_cast<const float2*>(J.h2 + (base + row) * HID + k);
      store_pair(s.ch, s.cl, row * SA + k, v.x, v.y);
    }
    __syncthreads();
    wgrad_tile<2>(accb[0], s.ah, s.al, SA, (warp & 1) * 16, s.bh, s.bl, SB, (warp >> 1) * 16, lane);
    if (warp < 2) wgrad_tile<2>(accb[1], s.ah, s.al, SA, (warp & 1) * 16, s.bh, s.bl, SB, 8 * 16, lane);
    if (warp < 8) wgrad_tile<2>(acc2, s.ah, s.al, SA, 32, s.ch, s.cl, SA, warp * 16, lane);
    __syncthreads();
  }
  // flush
#pragma unroll
  for (int blk = 0; blk < 2; ++blk) {
    if (blk == 1 && warp >= 2) break;
    const int cb = blk == 0 ? (warp >> 1) : 8;
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int f = (warp & 1) * 16 + g + (e >> 1) * 8, c = cb * 16 + nt * 8 + 2 * t4 + (e & 1);
        if (f < F && accb[blk][nt][e] != 0.f) atomicAdd(sh.g_basis + f * K0 + c, accb[blk][nt][e]);
      }
  }
  if (warp < 8) {
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int o = g + (e >> 1) * 8, k = warp * 16 + nt * 8 + 2 * t4 + (e & 1);
        if (o < od && acc2[nt][e] != 0.f) atomicAdd(J.g_w2 + o * HID + k, acc2[nt][e]);
      }
  }
  __syncthreads();
  if (tid < M * 4) s.colsum[K0 + tid] = bsum;
  __syncthreads();
  if (tid < od) {
    float v = 0.f;
    for (int r = 0; r < M; ++r) v += s.colsum[K0 + r * 4 + tid];
    if (v != 0.f) atomicAdd(J.g_b2 + tid, v);
  }
}

__global__ void __launch_bounds__(NT, 1) heads_wgrad_kernel(const WgradParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  WgradSmem& s = *reinterpret_cast<WgradSmem*>(smem_raw);
  const WgradSplit sp = p.split;
  const int per_job = sp.p1 + sp.p0 + sp.ps;
  const int job = (int)(blockIdx.x / per_job), role_id = (int)(blockIdx.x % per_job);
  const HeadBwdJob& J = p.jobs[job];
  const int64_t total = list_rows(p.n, p.n_dev);
  const int role = role_id < sp.p1 ? 0 : (role_id < sp.p1 + sp.p0 ? 1 : 2);
  const int parts = role == 0 ? sp.p1 : (role == 1 ? sp.p0 : sp.ps);
  const int part = role == 0 ? role_id : (role == 1 ? role_id - sp.p1 : role_id - sp.p1 - sp.p0);
  int64_t chunk = (total + parts - 1) / parts;
  chunk = (chunk + M - 1) / M * M;
  const int64_t r0 = (int64_t)part * chunk;
  const int64_t r1 = r0 + chunk < total ? r0 + chunk : total;
  if (r0 >= r1) return;
  if (role == 0) wgrad_big<8>(s, J.gz2, J.h1, HID, HID, r0, r1, J.g_w1, J.g_b1);          // gW1 = dz2^T h1, gb1
  else if (role == 1) wgrad_big<10>(s, J.gz1, J.inp, IN, IN, r0, r1, J.g_w0, J.g_b0);     // gW0 = dz1^T inp, gb0
  else wgrad_small(s, J, p.sh, r0, r1);
}

}  // namespace

namespace tir {

int launch_heads_backward(const TirField& f, const HeadBwdJob* jobs, int n_jobs, const HeadsBwdShared& sh, int64_t n,
                          const int64_t* n_dev, cudaStream_t stream) {
  if (n <= 0 || n_jobs <= 0) return TIR_OK;
  if (n_jobs > kMaxHeadJobs) return TIR_ERR_CONFIG;
  if (!sh.g_basis) return TIR_ERR_NULL;
  for (int j = 0; j < n_jobs; ++j) {
    const HeadBwdJob& J = jobs[j];
    if (f.aC != AC || J.mlp.feat_dim != F || J.mlp.hidden != HID || J.mlp.pe_feat != 2 || J.mlp.pe_x != 2)
      return TIR_ERR_SHAPE;
    if (J.mlp.out_dim < 1 || J.mlp.out_dim > 4 || J.out_stride < J.mlp.out_dim) return TIR_ERR_SHAPE;
    if (!J.out || !J.g_out || !J.inp || !J.h1 || !J.h2 || !J.gz1 || !J.gz2 || !J.gfeat || !J.gx0 || !J.g_w0 ||
        !J.g_b0 || !J.g_w1 || !J.g_b1 || !J.g_w2 || !J.g_b2)
      return TIR_ERR_NULL;
    if (J.light_mode != 0 && (!J.mlp.light_line || !sh.g_light || !sh.x0[J.point_set])) return TIR_ERR_NULL;
    if (J.point_set < 0 || J.point_set > 1) return TIR_ERR_CONFIG;
    // the weight gradients copy 64-row tiles of these with 16-byte cp.async
    if ((reinterpret_cast<uintptr_t>(J.gz1) | reinterpret_cast<uintptr_t>(J.gz2) | reinterpret_cast<uintptr_t>(J.h1) |
         reinterpret_cast<uintptr_t>(J.inp)) & 15)
      return TIR_ERR_CONFIG;
  }
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(heads_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(DgradSmem));
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(heads_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WgradSmem));
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  DgradParams dp{};
  dp.f = f; dp.sh = sh; dp.n_jobs = n_jobs; dp.n = n; dp.n_dev = n_dev;
  WgradParams wp{};
  wp.sh = sh; wp.n_jobs = n_jobs; wp.n = n; wp.n_dev = n_dev;
  for (int j = 0; j < n_jobs; ++j) { dp.jobs[j] = jobs[j]; wp.jobs[j] = jobs[j]; }
  const int64_t ctas = (n + DG * DM - 1) / (DG * DM);   // dgrad: DG tiles of DM rows in flight per CTA
  int per_job = num_sms() / n_jobs;           // one wave: one CTA per SM (both kernels fit one CTA per SM)
  if (per_job < 3) return TIR_ERR_CONFIG;     // the weight gradients need a CTA per role
  wp.split = wgrad_split(per_job);
  if (ctas < per_job) per_job = (int)ctas;
  heads_dgrad_kernel<<<per_job * n_jobs, NT, sizeof(DgradSmem), stream>>>(dp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  heads_wgrad_kernel<<<(wp.split.p1 + wp.split.p0 + wp.split.ps) * n_jobs, NT, sizeof(WgradSmem), stream>>>(wp);
  return (int)cudaGetLastError();
}

}  // namespace tir
