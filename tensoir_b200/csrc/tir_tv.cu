// Total-variation regulariser of the VM planes (SURVEY.md §8 f3): TVLoss (utils.py:143-162) as called by
// TV_loss_density / TV_loss_app (tensoRF_rotated_lights.py:80-92) during the radiance-only phase of training
// (train_tensoIR.py:276-285).  The reference runs ~14 slice / pow / sum launches per plane forward + backward, each a
// full pass over the plane; here the three planes of one call are ONE forward launch (value) and ONE backward launch
// (5-point stencil added straight into the gradient buffer): 1 read pass + 1 read-modify-write pass.
//
//   TV(x) = 2 * w * ( sum_{h<H-1} (x[h+1]-x[h])^2 / (C (H-1) W)  +  sum_{w<W-1} (x[w+1]-x[w])^2 / (C H (W-1)) )     (batch 1)
//
// The caller folds 2*w*1e-2 / count into scale_h / scale_w.  A zero count (H == 1 or W == 1) is the caller's business:
// the reference divides by zero there; the kernel just multiplies the (empty, zero) sum by the given scale.
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"
#include "tir_device.cuh"

namespace {

constexpr int kThreads = 256;

struct TvJob {
  const float* x;
  float* g;
  int Htot, W, C, Hper;     // storage seen as [Htot][W][C]; rows h and h+1 are neighbours iff (h % Hper) + 1 < Hper
  float sh, sw;
};
struct TvJobs { TvJob j[TIR_TV_MAX_PLANES]; };

template <int V> struct Vec;
template <> struct Vec<4> {
  float v[4];
  __device__ __forceinline__ void load(const float* p) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
};
template <> struct Vec<1> {
  float v[1];
  __device__ __forceinline__ void load(const float* p) { v[0] = *p; }
};

__device__ __forceinline__ float block_sum(float v) {
  __shared__ float part[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x < 32) {
    s = threadIdx.x < kThreads / 32 ? part[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  return s;   // valid in thread 0
}

template <int V>
__global__ void __launch_bounds__(kThreads) tv_fwd_kernel(TvJobs jobs, float* __restrict__ out) {
  const TvJob j = jobs.j[blockIdx.y];
  const int cpv = j.C / V;
  const int64_t n_units = (int64_t)j.Htot * j.W * cpv;
  const int64_t row = (int64_t)j.W * j.C;
  float sh = 0.f, sw = 0.f;
  for (int64_t u = (int64_t)blockIdx.x * kThreads + threadIdx.x; u < n_units; u += (int64_t)gridDim.x * kThreads) {
    const int cg = (int)(u % cpv);
    const int64_t t = u / cpv;
    const int w = (int)(t % j.W);
    const int h = (int)(t / j.W);
    const int64_t base = t * j.C + (int64_t)cg * V;
    Vec<V> a, b;
    a.load(j.x + base);
    if ((h % j.Hper) + 1 < j.Hper) {
      b.load(j.x + base + row);
#pragma unroll
      for (int i = 0; i < V; ++i) { const float d = b.v[i] - a.v[i]; sh = fmaf(d, d, sh); }
    }
    if (w + 1 < j.W) {
      b.load(j.x + base + j.C);
#pragma unroll
      for (int i = 0; i < V; ++i) { const float d = b.v[i] - a.v[i]; sw = fmaf(d, d, sw); }
    }
  }
  const float s = block_sum(j.sh * sh + j.sw * sw);
  if (threadIdx.x == 0 && s != 0.f) atomicAdd(out, s);
}

template <int V>
__global__ void __launch_bounds__(kThreads) tv_bwd_kernel(TvJobs jobs, const float* __restrict__ gout) {
  const TvJob j = jobs.j[blockIdx.y];
  const int cpv = j.C / V;
  const int64_t n_units = (int64_t)j.Htot * j.W * cpv;
  const int64_t row = (int64_t)j.W * j.C;
  const float go = 2.f * gout[0];
  const float kh = go * j.sh, kw = go * j.sw;
  for (int64_t u = (int64_t)blockIdx.x * kThreads + threadIdx.x; u < n_units; u += (int64_t)gridDim.x * kThreads) {
    const int cg = (int)(u % cpv);
    const int64_t t = u / cpv;
    const int w = (int)(t % j.W);
    const int h = (int)(t / j.W);
    const int hin = h % j.Hper;
    const int64_t base = t * j.C + (int64_t)cg * V;
    Vec<V> a, b;
    a.load(j.x + base);
    float acc[V];
#pragma unroll
    for (int i = 0; i < V; ++i) acc[i] = 0.f;
    // d/dx[h] of (x[h+1]-x[h])^2 + (x[h]-x[h-1])^2 = 2 ((x[h]-x[h-1]) - (x[h+1]-x[h])); the 2 is in kh / kw
    if (hin + 1 < j.Hper) {
      b.load(j.x + base + row);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] -= kh * (b.v[i] - a.v[i]);
    }
    if (hin > 0) {
      b.load(j.x + base - row);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] += kh * (a.v[i] - b.v[i]);
    }
    if (w + 1 < j.W) {
      b.load(j.x + base + j.C);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] -= kw * (b.v[i] - a.v[i]);
    }
    if (w > 0) {
      b.load(j.x + base - j.C);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] += kw * (a.v[i] - b.v[i]);
    }
    Vec<V> g;
    g.load(j.g + base);
    if (V == 4) {
      *reinterpret_cast<float4*>(j.g + base) = make_float4(g.v[0] + acc[0], g.v[1 % V] + acc[1 % V], g.v[2 % V] + acc[2 % V],
                                                           g.v[3 % V] + acc[3 % V]);
    } else {
      j.g[base] = g.v[0] + acc[0];
    }
  }
}

// -> 0 ok; fills jobs, the common vector width and the largest unit count
int make_jobs(const TirTvPlane* planes, int n, bool need_grad, TvJobs* jobs, int* vec, int64_t* max_units) {
  if (!planes || n < 1 || n > TIR_TV_MAX_PLANES) return TIR_ERR_SHAPE;
  *vec = 4;
  for (int k = 0; k < n; ++k) {
    const TirTvPlane& p = planes[k];
    if (!p.x || (need_grad && !p.grad)) return TIR_ERR_NULL;
    if (p.H < 1 || p.W < 1 || p.C < 1) return TIR_ERR_SHAPE;
    TvJob& j = jobs->j[k];
    j.x = p.x; j.g = p.grad; j.W = p.W; j.sh = p.scale_h; j.sw = p.scale_w;
    if (p.channel_last) { j.Htot = p.H; j.C = p.C; j.Hper = p.H; }
    else { j.Htot = p.C * p.H; j.C = 1; j.Hper = p.H; }     // [C][H][W] storage: C stacked images of one channel
    const uintptr_t al = reinterpret_cast<uintptr_t>(p.x) | (need_grad ? reinterpret_cast<uintptr_t>(p.grad) : 0);
    if ((j.C & 3) || (al & 15)) *vec = 1;
  }
  *max_units = 0;
  for (int k = 0; k < n; ++k) {
    const int64_t u = (int64_t)jobs->j[k].Htot * jobs->j[k].W * (jobs->j[k].C / *vec);
    if (u > *max_units) *max_units = u;
  }
  return 0;
}

int grid_x(int64_t units) {
  int64_t b = (units + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)tir::num_sms() * 8;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

extern "C" int tir_tv_loss(const TirTvPlane* planes, int32_t n_planes, float* out, void* stream) {
  if (!out) return TIR_ERR_NULL;
  TvJobs jobs; int vec; int64_t units;
  const int rc = make_jobs(planes, n_planes, false, &jobs, &vec, &units);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float), st);
  if (e != cudaSuccess) return (int)e;
  const dim3 grid(grid_x(units), n_planes);
  if (vec == 4) tv_fwd_kernel<4><<<grid, kThreads, 0, st>>>(jobs, out);
  else tv_fwd_kernel<1><<<grid, kThreads, 0, st>>>(jobs, out);
  return (int)cudaGetLastError();
}

extern "C" int tir_tv_loss_bwd(const TirTvPlane* planes, int32_t n_planes, const float* gout, void* stream) {
  if (!gout) return TIR_ERR_NULL;
  TvJobs jobs; int vec; int64_t units;
  const int rc = make_jobs(planes, n_planes, true, &jobs, &vec, &units);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(grid_x(units), n_planes);
  if (vec == 4) tv_bwd_kernel<4><<<grid, kThreads, 0, st>>>(jobs, gout);
  else tv_bwd_kernel<1><<<grid, kThreads, 0, st>>>(jobs, gout);
  return (int)cudaGetLastError();
}
