// One pass over all parameters per optimizer step (SURVEY.md §8 f3): Adam (torch.optim.Adam's update, train_tensoIR.py:206,
// :315-317) + the L1 regulariser's gradient (density_L1, tensoRF_rotated_lights.py:74-78: w * sign(x) / numel, folded into
// the gradient instead of ~25 autograd launches) + clearing the gradient for the next step (the backward kernels
// accumulate with atomics into persistent buffers, so no separate 70 MB memset) — 28 B/parameter of HBM traffic instead of
// the >= 5 passes the reference makes over the 17-31 M VM parameters.  A device-side `found_inf` flag (raised by a
// static-list overflow under CUDA-graph replay) turns the whole step into a no-op that only clears the gradients.
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = kThreads * 16;      // elements per CTA

// Per-tensor step counts, as torch.optim.Adam keeps them (state["step"] of each parameter): every table entry's counter
// advances by one unless found_inf is set, and its bias corrections go to bias[k] = {1 - beta1^t, sqrt(1 - beta2^t)}.
__global__ void adam_prologue_kernel(const TirAdamTensor* __restrict__ table, int n_tensors, float2* __restrict__ bias,
                                     float beta1, float beta2, const float* __restrict__ found_inf) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_tensors || (found_inf && found_inf[0] != 0.f)) return;
  float* counter = table[k].step;
  const float step = counter[0] + 1.f;
  counter[0] = step;
  bias[k] = make_float2(1.f - powf(beta1, step), sqrtf(1.f - powf(beta2, step)));
}

__global__ void __launch_bounds__(kThreads) adam_main_kernel(const TirAdamTensor* __restrict__ table, int n_tensors,
                                                             const int64_t* __restrict__ chunk_prefix,
                                                             const float2* __restrict__ bias,
                                                             const float* __restrict__ found_inf, float beta1,
                                                             float beta2, float eps, int clear_grad) {
  // which tensor does this chunk belong to
  const int64_t chunk = blockIdx.x;
  int lo = 0, hi = n_tensors - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (chunk_prefix[mid] <= chunk) lo = mid; else hi = mid - 1;
  }
  const TirAdamTensor t = table[lo];
  const int64_t base = (chunk - chunk_prefix[lo]) * kChunk;
  const bool skip = found_inf && found_inf[0] != 0.f;
  const float2 bc = skip ? make_float2(1.f, 1.f) : bias[lo];
  const float bc1 = bc.x, bc2s = bc.y;
  const float lr = t.lr_dev ? t.lr_dev[0] : t.lr;
  const float step_size = lr / bc1;
  const bool vec = ((reinterpret_cast<uintptr_t>(t.p) | reinterpret_cast<uintptr_t>(t.g) | reinterpret_cast<uintptr_t>(t.m) |
                     reinterpret_cast<uintptr_t>(t.v)) & 15) == 0;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int64_t i = base + (int64_t)(it * kThreads + threadIdx.x) * 4;
    if (i >= t.n) break;
    float p[4], g[4], m[4], v[4];
    const int cnt = (int)((t.n - i) < 4 ? (t.n - i) : 4);
    if (vec && cnt == 4) {
      const float4 gp = *reinterpret_cast<const float4*>(t.g + i);
      g[0] = gp.x; g[1] = gp.y; g[2] = gp.z; g[3] = gp.w;
      if (!skip) {
        const float4 pp = *reinterpret_cast<const float4*>(t.p + i), mp = *reinterpret_cast<const float4*>(t.m + i),
                     vp = *reinterpret_cast<const float4*>(t.v + i);
        p[0] = pp.x; p[1] = pp.y; p[2] = pp.z; p[3] = pp.w; m[0] = mp.x; m[1] = mp.y; m[2] = mp.z; m[3] = mp.w;
        v[0] = vp.x; v[1] = vp.y; v[2] = vp.z; v[3] = vp.w;
      }
    } else {
      for (int e = 0; e < cnt; ++e) {
        g[e] = t.g[i + e];
        if (!skip) { p[e] = t.p[i + e]; m[e] = t.m[i + e]; v[e] = t.v[i + e]; }
      }
    }
    if (!skip) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (e >= cnt) break;
        float ge = g[e];
        if (t.l1 != 0.f) ge += t.l1 * (p[e] > 0.f ? 1.f : (p[e] < 0.f ? -1.f : 0.f));     // d |x| / dx = sign(x)
        m[e] = m[e] + (1.f - beta1) * (ge - m[e]);                  // exp_avg.lerp_(grad, 1 - beta1)
        v[e] = beta2 * v[e] + (1.f - beta2) * ge * ge;
        const float denom = sqrtf(v[e]) / bc2s + eps;
        p[e] -= step_size * (m[e] / denom);
      }
    }
    if (vec && cnt == 4) {
      if (!skip) {
        *reinterpret_cast<float4*>(t.p + i) = make_float4(p[0], p[1], p[2], p[3]);
        *reinterpret_cast<float4*>(t.m + i) = make_float4(m[0], m[1], m[2], m[3]);
        *reinterpret_cast<float4*>(t.v + i) = make_float4(v[0], v[1], v[2], v[3]);
      }
      if (clear_grad) *reinterpret_cast<float4*>(t.g + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      for (int e = 0; e < cnt; ++e) {
        if (!skip) { t.p[i + e] = p[e]; t.m[i + e] = m[e]; t.v[i + e] = v[e]; }
        if (clear_grad) t.g[i + e] = 0.f;
      }
    }
  }
}

}  // namespace

extern "C" int tir_adam_chunk_elems(void) { return kChunk; }

extern "C" int tir_adam_step(const TirAdamTensor* table_dev, int32_t n_tensors, const int64_t* chunk_prefix_dev,
                             int64_t total_chunks, float* bias_dev, float beta1, float beta2, float eps,
                             const float* found_inf_dev, int32_t clear_grad, void* stream_) {
  if (n_tensors <= 0) return TIR_OK;
  if (!table_dev || !chunk_prefix_dev || !bias_dev) return TIR_ERR_NULL;
  cudaStream_t stream = (cudaStream_t)stream_;
  constexpr int kPrologueThreads = 128;
  // tensors with no elements still count a step, like torch.optim.Adam's
  adam_prologue_kernel<<<(n_tensors + kPrologueThreads - 1) / kPrologueThreads, kPrologueThreads, 0, stream>>>(
      table_dev, n_tensors, reinterpret_cast<float2*>(bias_dev), beta1, beta2, found_inf_dev);
  if (total_chunks > 0)
    adam_main_kernel<<<(unsigned)total_chunks, kThreads, 0, stream>>>(table_dev, n_tensors, chunk_prefix_dev,
                                                                     reinterpret_cast<const float2*>(bias_dev),
                                                                     found_inf_dev, beta1, beta2, eps, clear_grad);
  return (int)cudaGetLastError();
}
