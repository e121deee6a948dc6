// Test-view metrics (SURVEY.md §8 f4): everything one rendered view contributes to the evaluation loops of
// renderer.py:134-516 (and their _simple / _general_multi_lights twins), computed from the renderer's device maps.
// The reference copies ten maps per 4096-ray chunk to the host and runs utils.rgb_ssim (scipy, fp64, CPU) four times per
// view; here the maps stay on the device and one call is three launches:
//
//   1. pixel pass      clamp rgb / rgb_with_brdf (renderer.py:265-266), their squared error against gt_rgb (:300-303),
//                      the single- and three-channel aligned albedo maps (:274-289, written out for the PNGs), their
//                      gamma-1/2.2 squared error against gt_albedo (:392-394, :462-468) and the normal angular error
//                      over every pixel (:353, :367, :470);
//   2. SSIM pass       utils.rgb_ssim (utils.py:93-139) for up to four image pairs: per channel a valid-mode separable
//                      11-tap Gaussian (sigma 1.5) of x, y, x^2, y^2, xy -- products in fp32, convolution and SSIM in
//                      fp64 -- over a 16x16 output tile with its 10-pixel halo in shared memory;
//   3. finalize        one block sums the per-block fp64 partials in a fixed order.
//
// No float atomics anywhere: the result is bit-identical from call to call.
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"
#include "tir_eval_body.h"

namespace {

constexpr int kThreads = 256;
constexpr int kIn = EVAL_TILE + EVAL_HALO;     // input tile edge: 26

// fixed-order block sum (tree over shared memory); the result is valid in every thread
__device__ double block_sum_det(double v, double* red) {
  const int t = threadIdx.x;
  red[t] = v;
  __syncthreads();
#pragma unroll
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (t < s) red[t] += red[t + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kThreads) eval_pixel_kernel(TirEvalView v, bool has_albedo, bool has_normal,
                                                              double* __restrict__ work) {
  __shared__ double red[kThreads];
  float r1 = 0.f, r3[3] = {0.f, 0.f, 0.f};
  if (has_albedo) {
    r1 = v.ratio[0];
    r3[0] = v.ratio[1]; r3[1] = v.ratio[2]; r3[2] = v.ratio[3];
  }
  double acc[EVAL_N_PIX] = {0.0, 0.0, 0.0, 0.0, 0.0};
  const int64_t n = (int64_t)v.H * v.W;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    EvalPixel p;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      p.rgb[c] = v.rgb[i * 3 + c]; p.brdf[c] = v.rgb_brdf[i * 3 + c]; p.gt[c] = v.gt_rgb[i * 3 + c];
      p.alb[c] = has_albedo ? v.albedo[i * 3 + c] : 0.f;
      p.gta[c] = has_albedo ? v.gt_albedo[i * 3 + c] : 0.f;
      p.nrm[c] = has_normal ? v.normal[i * 3 + c] : 0.f;
      p.gtn[c] = has_normal ? v.gt_normal[i * 3 + c] : 0.f;
    }
    p.mask = has_albedo ? (v.gt_mask[i] != 0) : 0;
    float al1[3], al3[3];
    eval_pixel(p, has_albedo, has_normal, r1, r3, acc, al1, al3);
    if (has_albedo) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { v.aligned_single[i * 3 + c] = al1[c]; v.aligned_three[i * 3 + c] = al3[c]; }
    }
  }
#pragma unroll
  for (int q = 0; q < EVAL_N_PIX; ++q) {
    const double s = block_sum_det(acc[q], red);
    if (threadIdx.x == 0) work[q * EVAL_PIX_BLOCKS + blockIdx.x] = s;
  }
}

// A batch of SSIM pairs for one launch (blockIdx.z indexes it): image a (clamped to [0,1] first when clamp_a), image b,
// both [H*W,3]; their partials go to part[(first + z) * n_tiles + tile].
constexpr int kPairsPerLaunch = 8;
struct SsimPairs {
  const float* a[kPairsPerLaunch];
  const float* b[kPairsPerLaunch];
  int clamp_a[kPairsPerLaunch];
  int first;
};

__global__ void __launch_bounds__(kThreads) eval_ssim_kernel(int32_t H, int32_t W, SsimPairs pairs, int64_t n_tiles,
                                                             double* __restrict__ part) {
  __shared__ float sx[kIn][kIn + 1], sy[kIn][kIn + 1];
  __shared__ double sv[5][EVAL_TILE][kIn];
  __shared__ double taps[EVAL_WIN];
  __shared__ double red[kThreads];
  const int z = blockIdx.z;
  const int pair = pairs.first + z;
  const float* a = pairs.a[z];
  const float* b = pairs.b[z];
  const bool clamp_a = pairs.clamp_a[z] != 0;
  const int x0 = blockIdx.x * EVAL_TILE, y0 = blockIdx.y * EVAL_TILE;
  const int t = threadIdx.x;
  if (t < EVAL_WIN) taps[t] = eval_tap(t);
  const int ty = t / EVAL_TILE, tx = t % EVAL_TILE;
  const bool out_ok = (y0 + ty) < H - EVAL_HALO && (x0 + tx) < W - EVAL_HALO;
  double acc = 0.0;
  for (int c = 0; c < 3; ++c) {
    __syncthreads();
    for (int k = t; k < kIn * kIn; k += kThreads) {
      const int r = k / kIn, col = k % kIn;
      const int gy = y0 + r, gx = x0 + col;
      float xa = 0.f, xb = 0.f;
      if (gy < H && gx < W) {
        const int64_t pix = (int64_t)gy * W + gx;
        xa = a[pix * 3 + c];
        xb = b[pix * 3 + c];
        if (clamp_a) xa = ev_clamp01(xa);
      }
      sx[r][col] = xa;
      sy[r][col] = xb;
    }
    __syncthreads();
    // convolve2d(z, filt[:, None], 'valid'): along the rows first (utils.py:115-117)
    for (int k = t; k < EVAL_TILE * kIn; k += kThreads) {
      const int r = k / kIn, col = k % kIn;
      double m0 = 0.0, m1 = 0.0, m00 = 0.0, m11 = 0.0, m01 = 0.0;
#pragma unroll
      for (int j = 0; j < EVAL_WIN; ++j) {
        const double w = taps[j];
        const float xa = sx[r + j][col], xb = sy[r + j][col];
        m0 += w * (double)xa;
        m1 += w * (double)xb;
        m00 += w * (double)ev_mul(xa, xa);
        m11 += w * (double)ev_mul(xb, xb);
        m01 += w * (double)ev_mul(xa, xb);
      }
      sv[0][r][col] = m0; sv[1][r][col] = m1; sv[2][r][col] = m00; sv[3][r][col] = m11; sv[4][r][col] = m01;
    }
    __syncthreads();
    // then filt[None, :] along the columns
    if (out_ok) {
      double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int j = 0; j < EVAL_WIN; ++j) {
        const double w = taps[j];
#pragma unroll
        for (int q = 0; q < 5; ++q) m[q] += w * sv[q][ty][tx + j];
      }
      acc += eval_ssim_point(m[0], m[1], m[2], m[3], m[4]);
    }
  }
  const double s = block_sum_det(acc, red);
  if (t == 0) part[(int64_t)pair * n_tiles + (int64_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) eval_finalize_kernel(const double* __restrict__ work, int64_t n_tiles,
                                                                 int n_ssim, double n_windows,
                                                                 double* __restrict__ out) {
  __shared__ double red[kThreads];
  for (int q = 0; q < EVAL_N_PIX; ++q) {
    double v = 0.0;
    for (int b = threadIdx.x; b < EVAL_PIX_BLOCKS; b += kThreads) v += work[q * EVAL_PIX_BLOCKS + b];
    const double s = block_sum_det(v, red);
    if (threadIdx.x == 0) out[q] = s;
  }
  const double* part = work + EVAL_N_PIX * EVAL_PIX_BLOCKS;
  for (int p = 0; p < 4; ++p) {
    double v = 0.0;
    if (p < n_ssim)
      for (int64_t k = threadIdx.x; k < n_tiles; k += kThreads) v += part[p * n_tiles + k];
    const double s = block_sum_det(v, red);
    if (threadIdx.x == 0) out[EVAL_N_PIX + p] = p < n_ssim ? s / n_windows : 0.0;
  }
}

// squared-error partials of pair blockIdx.y: (a - b)^2 in fp32, fp64 sums in a fixed order
__global__ void __launch_bounds__(kThreads) eval_pair_sse_kernel(const float* __restrict__ a,
                                                                 const float* __restrict__ b, int64_t n,
                                                                 double* __restrict__ part) {
  __shared__ double red[kThreads];
  const int64_t off = (int64_t)blockIdx.y * n;
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const float d = ev_sub(a[off + i], b[off + i]);
    acc += (double)ev_mul(d, d);
  }
  const double s = block_sum_det(acc, red);
  if (threadIdx.x == 0) part[(int64_t)blockIdx.y * EVAL_PAIR_SSE_BLOCKS + blockIdx.x] = s;
}

// one block per pair: out[p] = {sse, mean ssim}
__global__ void __launch_bounds__(kThreads) eval_pairs_finalize_kernel(const double* __restrict__ work,
                                                                       int64_t n_tiles, double n_windows,
                                                                       double* __restrict__ out) {
  __shared__ double red[kThreads];
  const int p = blockIdx.x;
  double v = 0.0;
  for (int k = threadIdx.x; k < EVAL_PAIR_SSE_BLOCKS; k += kThreads) v += work[(int64_t)p * EVAL_PAIR_SSE_BLOCKS + k];
  const double sse = block_sum_det(v, red);
  const double* part = work + (int64_t)gridDim.x * EVAL_PAIR_SSE_BLOCKS;
  v = 0.0;
  for (int64_t k = threadIdx.x; k < n_tiles; k += kThreads) v += part[p * n_tiles + k];
  const double ss = block_sum_det(v, red);
  if (threadIdx.x == 0) { out[2 * p] = sse; out[2 * p + 1] = ss / n_windows; }
}

}  // namespace

extern "C" int tir_eval_pairs_work_size(int32_t P, int32_t H, int32_t W, int64_t* n_doubles) {
  const int rc = eval_pairs_work_size_check(P, H, W, n_doubles);
  if (rc <= 0) return rc;
  *n_doubles = eval_pairs_work_doubles(P, H, W);
  return TIR_OK;
}

extern "C" int tir_eval_pairs(const float* a, const float* b, int32_t P, int32_t H, int32_t W, double* work,
                              int64_t work_cap, double* out, void* stream) {
  const int rc = eval_pairs_validate(a, b, P, H, W, work, work_cap, out);
  if (rc <= 0) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t n = (int64_t)H * W * 3;
  const int64_t n_tiles = eval_ssim_tiles(H, W);
  eval_pair_sse_kernel<<<dim3(EVAL_PAIR_SSE_BLOCKS, P), kThreads, 0, s>>>(a, b, n, work);
  double* part = work + (int64_t)P * EVAL_PAIR_SSE_BLOCKS;
  for (int first = 0; first < P; first += kPairsPerLaunch) {
    SsimPairs pairs{};
    const int m = P - first < kPairsPerLaunch ? P - first : kPairsPerLaunch;
    for (int z = 0; z < m; ++z) {
      pairs.a[z] = a + (int64_t)(first + z) * n;
      pairs.b[z] = b + (int64_t)(first + z) * n;
      pairs.clamp_a[z] = 0;
    }
    pairs.first = first;
    const dim3 grid((W - EVAL_HALO + EVAL_TILE - 1) / EVAL_TILE, (H - EVAL_HALO + EVAL_TILE - 1) / EVAL_TILE, m);
    eval_ssim_kernel<<<grid, kThreads, 0, s>>>(H, W, pairs, n_tiles, part);
  }
  const double n_windows = (double)(H - EVAL_HALO) * (double)(W - EVAL_HALO) * 3.0;
  eval_pairs_finalize_kernel<<<P, kThreads, 0, s>>>(work, n_tiles, n_windows, out);
  return (int)cudaGetLastError();
}

extern "C" int tir_eval_work_size(int32_t H, int32_t W, int64_t* n_doubles) {
  const int rc = eval_work_size_check(H, W, n_doubles);
  if (rc <= 0) return rc;
  *n_doubles = eval_work_doubles(H, W);
  return TIR_OK;
}

extern "C" int tir_eval_view(const TirEvalView* view, double* work, int64_t work_cap, double* out, void* stream) {
  bool has_albedo = false, has_normal = false;
  int n_ssim = 0;
  const int rc = eval_view_check(view, work, work_cap, out, &has_albedo, &has_normal, &n_ssim);
  if (rc <= 0) return rc;
  const TirEvalView v = *view;
  const int64_t n_tiles = n_ssim ? eval_ssim_tiles(v.H, v.W) : 0;
  cudaStream_t s = (cudaStream_t)stream;
  eval_pixel_kernel<<<EVAL_PIX_BLOCKS, kThreads, 0, s>>>(v, has_albedo, has_normal, work);
  if (n_ssim) {
    const dim3 grid((v.W - EVAL_HALO + EVAL_TILE - 1) / EVAL_TILE, (v.H - EVAL_HALO + EVAL_TILE - 1) / EVAL_TILE, n_ssim);
    // pair 0 rgb/gt_rgb, 1 rgb_brdf/gt_rgb (the renderer maps are clamped before the metrics),
    // 2 aligned_single/gt_albedo, 3 aligned_three/gt_albedo
    SsimPairs pairs{{v.rgb, v.rgb_brdf, v.aligned_single, v.aligned_three},
                    {v.gt_rgb, v.gt_rgb, v.gt_albedo, v.gt_albedo}, {1, 1, 0, 0}, 0};
    eval_ssim_kernel<<<grid, kThreads, 0, s>>>(v.H, v.W, pairs, n_tiles, work + EVAL_N_PIX * EVAL_PIX_BLOCKS);
  }
  const double n_windows = (double)(v.H - EVAL_HALO) * (double)(v.W - EVAL_HALO) * 3.0;
  eval_finalize_kernel<<<1, kThreads, 0, s>>>(work, n_tiles, n_ssim, n_windows, out);
  return (int)cudaGetLastError();
}
