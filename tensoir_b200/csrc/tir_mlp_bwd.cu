// Backward of the appearance heads (the four 150-128-128-{3,4} MLPs of the primary march, basis_mat, light_line and
// the positional encoding) on the activations dumped by the fused forward (tir_mlp.cu, launch_heads_forward).
// Replaces the autograd graph of MLPRender_Fea / MLPBRDF_PEandFeature (tensorBase_rotated_lights.py:122-146,:182-208)
// and compute_{app,intrin}feature's tail (tensoRF_rotated_lights.py:155-224): in round 1 this was ~300 cuBLAS SIMT
// sgemm / elementwise launches per step; here it is TWO launches for all heads of a step:
//
//   heads_dgrad_kernel   per 64-sample tile: d out -> d z3 -> (W2) -> ReLU' -> (W1^T GEMM) -> ReLU' -> (W0^T GEMM) ->
//                        positional-encoding backward -> d feat -> (basis^T) -> d (plane*line*light) -> * light -> gx0,
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

__device__ __forceinline__ float act_grad(int act, float y) { return act == 0 ? y * (1.f - y) : 1.f - y * y; }

// ---------------------------------------------------------------------------------------------------------------------
// data gradient
// ---------------------------------------------------------------------------------------------------------------------
struct DgradSmem {
  __nv_bfloat16 w1h[HID * SA], w1l[HID * SA];     // W1^T: [in][out]
  __nv_bfloat16 w0h[GIN * SA], w0l[GIN * SA];     // W0^T: [in < 144][out]
  union {
    struct { __nv_bfloat16 h[M * SA], l[M * SA]; } a;   // activation-gradient tile (A operand)
    float gin[M * GIN];                                 // d input of the MLP after the last GEMM
  } u;
  __nv_bfloat16 bth[K0 * SF], btl[K0 * SF];        // basis^T: [c][f] (f padded to 32)
  __nv_bfloat16 gfh[M * SF], gfl[M * SF];          // d feat tile (A operand of the basis GEMM)
  float w2[4 * HID];
  float gz3[M * 4];
  float glight[LMAX * K0];
  float lmean[K0];
  int light[M];
};

struct DgradParams {
  TirField f;
  HeadBwdJob jobs[kMaxHeadJobs];
  HeadsBwdShared sh;
  int n_jobs;
  int64_t n;
  const int64_t* n_dev;
};

__global__ void __launch_bounds__(NT, 1) heads_dgrad_kernel(const DgradParams p) {
  // warp w: column block w % 8 (16 columns), row half w / 8 (32 rows) of every 64 x 128 GEMM output
  extern __shared__ __align__(128) unsigned char smem_raw[];
  DgradSmem& s = *reinterpret_cast<DgradSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int job = (int)(blockIdx.x % p.n_jobs);
  const HeadBwdJob& J = p.jobs[job];
  const TirMlp& mlp = J.mlp;
  const int od = mlp.out_dim, L = mlp.n_lights;
  const int mode = J.light_mode;

  // ---- stage transposed split-BF16 weights (coalesced global reads; the one-off smem bank conflicts are irrelevant)
  for (int i = tid; i < HID * HID; i += NT) {
    const int o = i / HID, k = i % HID;          // W1[o][k]  ->  w1T[k][o]
    split_bf16(__ldg(mlp.w1 + i), s.w1h[k * SA + o], s.w1l[k * SA + o]);
  }
  for (int i = tid; i < HID * IN; i += NT) {
    const int o = i / IN, k = i % IN;            // W0[o][k]  ->  w0T[k][o], k < 144 only
    if (k < GIN) split_bf16(__ldg(mlp.w0 + i), s.w0h[k * SA + o], s.w0l[k * SA + o]);
  }
  for (int i = tid; i < K0 * SF; i += NT) {
    const int c = i / SF, f = i % SF;            // basis[f][c] -> bT[c][f]
    split_bf16(f < F ? __ldg(mlp.basis + f * K0 + c) : 0.f, s.bth[i], s.btl[i]);
  }
  for (int i = tid; i < M * SF; i += NT) { s.gfh[i] = __float2bfloat16_rn(0.f); s.gfl[i] = __float2bfloat16_rn(0.f); }
  for (int i = tid; i < 4 * HID; i += NT) s.w2[i] = (i / HID) < od ? __ldg(mlp.w2 + i) : 0.f;
  for (int i = tid; i < LMAX * K0; i += NT) s.glight[i] = 0.f;
  if (mode == 2)
    for (int c = tid; c < K0; c += NT) {
      float a = 0.f;
      for (int l = 0; l < L; ++l) a += __ldg(mlp.light_line + (size_t)l * K0 + c);
      s.lmean[c] = a / (float)L;
    }
  __syncthreads();

  const int64_t total = list_rows(p.n, p.n_dev);
  const int64_t n_tiles = (total + M - 1) / M;
  const float* x0 = p.sh.x0[J.point_set];

  for (int64_t tile = blockIdx.x / p.n_jobs; tile < n_tiles; tile += gridDim.x / p.n_jobs) {
    const int64_t base = tile * M;
    // ---- a. d z3 = d out * act'(out)
    {
      const int row = tid >> 2, o = tid & 3;
      const int64_t i = base + row;
      float v = 0.f;
      if (row < M && i < total && o < od)
        v = J.g_out[i * J.out_stride + o] * act_grad(J.act, J.out[i * J.out_stride + o]);
      if (row < M) s.gz3[row * 4 + o] = v;
      if (tid < M) {
        const int64_t ii = base + tid;
        int li = 0;
        if (ii < total && mode == 1 && J.light_idx) li = J.light_idx[J.x_index ? (int64_t)J.x_index[ii] : ii];
        s.light[tid] = li;
      }
    }
    __syncthreads();
    // ---- b. d z2 = (d z3 @ W2) * [h2 > 0]   (K = out_dim <= 4: CUDA cores)
    for (int idx = tid; idx < M * (HID / 2); idx += NT) {
      const int row = idx / (HID / 2), k = (idx % (HID / 2)) * 2;
      const int64_t i = base + row;
      float va = 0.f, vb = 0.f;
      if (i < total) {
        const float2 h = *reinterpret_cast<const float2*>(J.h2 + i * HID + k);
        const float z0 = s.gz3[row * 4], z1 = s.gz3[row * 4 + 1], z2 = s.gz3[row * 4 + 2], z3 = s.gz3[row * 4 + 3];
        va = z0 * s.w2[k] + z1 * s.w2[HID + k] + z2 * s.w2[2 * HID + k] + z3 * s.w2[3 * HID + k];
        vb = z0 * s.w2[k + 1] + z1 * s.w2[HID + k + 1] + z2 * s.w2[2 * HID + k + 1] + z3 * s.w2[3 * HID + k + 1];
        va = h.x > 0.f ? va : 0.f;
        vb = h.y > 0.f ? vb : 0.f;
        *reinterpret_cast<float2*>(J.gz2 + i * HID + k) = make_float2(va, vb);
      }
      store_pair(s.u.a.h, s.u.a.l, row * SA + k, va, vb);
    }
    __syncthreads();
    // ---- c. d z1 = (d z2 @ W1) * [h1 > 0]
    const int nb = warp & 7, mh = warp >> 3;
    {
      float acc[2][2][4] = {};
      warp_gemm_nt<2>(acc, s.u.a.h, s.u.a.l, mh * 32, s.w1h, s.w1l, SA, nb * 16, HID, lane);
      __syncthreads();
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = mh * 32 + mt * 16 + g + half * 8;
            const int col = nb * 16 + nt * 8 + 2 * t4;
            const int64_t i = base + row;
            float va = 0.f, vb = 0.f;
            if (i < total) {
              const float2 h = *reinterpret_cast<const float2*>(J.h1 + i * HID + col);
              va = h.x > 0.f ? acc[mt][nt][half * 2] : 0.f;
              vb = h.y > 0.f ? acc[mt][nt][half * 2 + 1] : 0.f;
              *reinterpret_cast<float2*>(J.gz1 + i * HID + col) = make_float2(va, vb);
            }
            store_pair(s.u.a.h, s.u.a.l, row * SA + col, va, vb);
          }
    }
    __syncthreads();
    // ---- d. d input = d z1 @ W0   (columns [0,144) only: the 3-vector and its encoding carry no gradient)
    {
      float acc[2][2][4] = {};
      float acx[1][2][4] = {};
      warp_gemm_nt<2>(acc, s.u.a.h, s.u.a.l, mh * 32, s.w0h, s.w0l, SA, nb * 16, HID, lane);
      if (warp < 4) warp_gemm_nt<1>(acx, s.u.a.h, s.u.a.l, warp * 16, s.w0h, s.w0l, SA, HID, HID, lane);
      __syncthreads();          // every warp is done reading the tile that `gin` aliases
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = mh * 32 + mt * 16 + g + half * 8, col = nb * 16 + nt * 8 + 2 * t4;
            *reinterpret_cast<float2*>(s.u.gin + row * GIN + col) =
                make_float2(acc[mt][nt][half * 2], acc[mt][nt][half * 2 + 1]);
          }
      if (warp < 4) {
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int row = warp * 16 + g + half * 8, col = HID + nt * 8 + 2 * t4;
            *reinterpret_cast<float2*>(s.u.gin + row * GIN + col) =
                make_float2(acx[0][nt][half * 2], acx[0][nt][half * 2 + 1]);
          }
      }
    }
    __syncthreads();
    // ---- e. positional-encoding backward: d feat_f = d in_f + sum_p 2^p (d sin_fp * cos_fp - d cos_fp * sin_fp)
    for (int idx = tid; idx < M * F; idx += NT) {
      const int row = idx / F, f = idx % F;
      const int64_t i = base + row;
      float v = 0.f;
      if (i < total) {
        const float* in = J.inp + i * IN;
        const float* gi = s.u.gin + row * GIN;
        v = gi[f] + (gi[30 + 2 * f] * in[84 + 2 * f] - gi[84 + 2 * f] * in[30 + 2 * f]) +
            2.f * (gi[31 + 2 * f] * in[85 + 2 * f] - gi[85 + 2 * f] * in[31 + 2 * f]);
        J.gfeat[i * GF + f] = v;
      }
      split_bf16(v, s.gfh[row * SF + f], s.gfl[row * SF + f]);
    }
    __syncthreads();
    // ---- f. d (products * light) = d feat @ basis (tensor cores: K = 32, N = 144);  gx0 = that * light row;
    //         light_line gradient = sum over samples of d(...) * raw products
    {
      // 9 column blocks of 16 x 2 row halves = 18 warp tasks; warps 0..15 take one, warps 0..1 a second one
      for (int task = warp; task < 18; task += NT / 32) {
        const int cb = task % 9, rh = task / 9;
        float acc[2][2][4] = {};
        warp_gemm_nt<2>(acc, s.gfh, s.gfl, rh * 32, s.bth, s.btl, SF, cb * 16, 32, lane, SF);
        float gl[2][2][4];            // d(...) * raw products: the light_line gradient contributions
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int row = rh * 32 + mt * 16 + g + half * 8, c = cb * 16 + nt * 8 + 2 * t4;
              const int64_t i = base + row;
              gl[mt][nt][half * 2] = 0.f; gl[mt][nt][half * 2 + 1] = 0.f;
              if (i >= total) continue;
              const float a0 = acc[mt][nt][half * 2], a1 = acc[mt][nt][half * 2 + 1];
              float l0 = 1.f, l1 = 1.f;
              if (mode == 1) {
                const float2 lv = __ldg(reinterpret_cast<const float2*>(mlp.light_line + (size_t)s.light[row] * K0 + c));
                l0 = lv.x; l1 = lv.y;
              } else if (mode == 2) {
                l0 = s.lmean[c]; l1 = s.lmean[c + 1];
              }
              *reinterpret_cast<float2*>(J.gx0 + i * K0 + c) = make_float2(a0 * l0, a1 * l1);
              if (mode != 0) {
                const float2 xv = __ldg(reinterpret_cast<const float2*>(x0 + i * K0 + c));
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
                    const int row = rh * 32 + mt * 16 + g + half * 8;
                    if (mode == 2 || s.light[row] == l) v += gl[mt][nt][half * 2 + e];
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
                  const int row = rh * 32 + mt * 16 + g + (e >> 1) * 8, lr = s.light[row];
                  if (lr >= LMAX && gl[mt][nt][e] != 0.f)
                    atomicAdd(p.sh.g_light + (size_t)lr * K0 + cb * 16 + nt * 8 + 2 * t4 + (e & 1), gl[mt][nt][e]);
                }
          }
        }
      }
    }
    __syncthreads();
  }
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
};

constexpr int P_W = 14;     // CTAs (row slices) per head for each of the two big weight gradients
constexpr int P_S = 9;      // CTAs per head for the small ones (gW2, gb2, g basis_mat)
constexpr int CTAS_PER_JOB = 2 * P_W + P_S;

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

// g_w[128][ld] += (d z)^T @ act  over rows [r0, r1);  g_b[128] += column sums of d z.
// 16 warps: warp w owns gradient rows 16 (w % 8).. and the column half w / 8 (NT8H n8-tiles).
template <int NT8H>
__device__ void wgrad_big(WgradSmem& s, const float* __restrict__ gz, const float* __restrict__ actv, int ncol, int ld,
                          int64_t r0, int64_t r1, float* g_w, float* g_b) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int mt = warp & 7, nh = warp >> 3;
  float acc[NT8H][4] = {};
  float cs0 = 0.f, cs1 = 0.f;                 // columns 2 (tid % 64), +1 of d z (512 % 64 == 0: fixed per thread)
  for (int i = tid; i < M * SB; i += NT) { s.bh[i] = __float2bfloat16_rn(0.f); s.bl[i] = __float2bfloat16_rn(0.f); }
  __syncthreads();
  const int half_cols = ncol / 2;             // 64 or 75 float2 per row
  for (int64_t base = r0; base < r1; base += M) {
    for (int idx = tid; idx < M * (HID / 2); idx += NT) {
      const int row = idx / (HID / 2), k = (idx % (HID / 2)) * 2;
      float2 v = make_float2(0.f, 0.f);
      if (base + row < r1) v = *reinterpret_cast<const float2*>(gz + (base + row) * HID + k);
      cs0 += v.x; cs1 += v.y;
      store_pair(s.ah, s.al, row * SA + k, v.x, v.y);
    }
    for (int idx = tid; idx < M * half_cols; idx += NT) {
      const int row = idx / half_cols, k = (idx % half_cols) * 2;
      float2 v = make_float2(0.f, 0.f);
      if (base + row < r1) v = *reinterpret_cast<const float2*>(actv + (base + row) * ncol + k);
      store_pair(s.bh, s.bl, row * SB + k, v.x, v.y);
    }
    __syncthreads();
    wgrad_tile<NT8H>(acc, s.ah, s.al, SA, mt * 16, s.bh, s.bl, SB, nh * NT8H * 8, lane);
    __syncthreads();
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
  const int job = (int)(blockIdx.x / CTAS_PER_JOB), role_id = (int)(blockIdx.x % CTAS_PER_JOB);
  const HeadBwdJob& J = p.jobs[job];
  const int64_t total = list_rows(p.n, p.n_dev);
  const int parts = role_id < 2 * P_W ? P_W : P_S;
  const int part = role_id < P_W ? role_id : (role_id < 2 * P_W ? role_id - P_W : role_id - 2 * P_W);
  int64_t chunk = (total + parts - 1) / parts;
  chunk = (chunk + M - 1) / M * M;
  const int64_t r0 = (int64_t)part * chunk;
  const int64_t r1 = r0 + chunk < total ? r0 + chunk : total;
  if (r0 >= r1) return;
  if (role_id < P_W) wgrad_big<8>(s, J.gz2, J.h1, HID, HID, r0, r1, J.g_w1, J.g_b1);          // gW1 = dz2^T h1, gb1
  else if (role_id < 2 * P_W) wgrad_big<10>(s, J.gz1, J.inp, IN, IN, r0, r1, J.g_w0, J.g_b0); // gW0 = dz1^T inp, gb0
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
  const int64_t tiles = (n + M - 1) / M;
  int per_job = num_sms() / n_jobs;
  if (tiles < per_job) per_job = (int)tiles;
  heads_dgrad_kernel<<<per_job * n_jobs, NT, sizeof(DgradSmem), stream>>>(dp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  heads_wgrad_kernel<<<CTAS_PER_JOB * n_jobs, NT, sizeof(WgradSmem), stream>>>(wp);
  return (int)cudaGetLastError();
}

}  // namespace tir
