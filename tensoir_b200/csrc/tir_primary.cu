// Fused primary march: TensorBase.forward with is_relight=True (models/tensorBase_rotated_lights.py:868-1036) and its
// whole backward as three C-ABI calls (tir_primary_march / tir_primary_heads / tir_primary_backward) that chain the
// kernels of the path on one stream with no host round trip: every list length stays on the device.
//
//   forward   valid count -> scan -> valid fill -> density + sigma -> compositing (+ appearance counts) -> scan ->
//             appearance list (+ jittered points) -> 4 heads in ONE launch -> derived-normal gather -> per-sample tail
//             (+ derived normals, costs, 14 composited channels) -> per-ray epilogue                  = 11 launches
//   backward  epilogue -> tail (+ derived-normal backward, weight scatter) -> heads dgrad -> heads wgrad -> 2 appearance
//             scatters -> derived-normal scatter -> compositing (+ softplus') -> density scatter        = 9 launches
// (round 1: ~25 own + ~500 torch launches for the same work.)
#include "tir_device.cuh"
#include "tir_internal.h"
#include "tir_tail_body.h"

using namespace tir;

namespace {

constexpr int K0 = 144;

// exclusive scan of int32 counts -> int64 offsets[n+1] (one block; n is a ray count); records the total
__global__ void __launch_bounds__(1024) scan_counts_kernel(const int32_t* __restrict__ counts, int64_t n,
                                                           int64_t* __restrict__ offsets, int64_t cap,
                                                           int64_t* __restrict__ status, int slot) {
  __shared__ int64_t warp_sums[32];
  __shared__ int64_t carry_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { carry_s = 0; offsets[0] = 0; }
  __syncthreads();
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + tid;
    int64_t v = i < n ? (int64_t)counts[i] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    if (lane == 31) warp_sums[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int64_t w = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += t;
      }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int64_t carry = carry_s;
    const int64_t incl = carry + v + (warp > 0 ? warp_sums[warp - 1] : 0);
    if (i < n) offsets[i + 1] = incl;
    __syncthreads();
    if (tid == 1023) carry_s = incl;
    __syncthreads();
  }
  if (tid == 0 && status) {
    const int64_t total = carry_s;
    status[slot] = total;
    if (total > cap) status[2] = 1;
  }
}

// compute_densityfeature + feature2density on the valid list (tensoRF_rotated_lights.py:95-110, tensorBase:813-817)
__global__ void primary_density_kernel(TirField f, const float* __restrict__ xn, int64_t cap,
                                       const int64_t* __restrict__ n_dev, float* __restrict__ feat,
                                       float* __restrict__ sigma) {
  const int64_t n = list_rows(cap, n_dev);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float ft = density_feature<16>(f, xn[i * 3], xn[i * 3 + 1], xn[i * 3 + 2]);
    feat[i] = ft;
    sigma[i] = feature_to_sigma(f, ft);
  }
}

// raw2alpha over ray segments, sequential like torch.cumprod (tensorBase:21-28), + acc / depth (:974-975) + the number
// of appearance samples (weight > rayMarch_weight_thres, :925) of the ray
__global__ void primary_composite_fwd_kernel(const float* __restrict__ sigma, const float* __restrict__ dist,
                                             const float* __restrict__ z, const int64_t* __restrict__ offsets,
                                             int64_t n_rays, float scale, int64_t cap, float thres,
                                             float* __restrict__ weight, float* __restrict__ trans,
                                             float* __restrict__ t_last, float* __restrict__ acc,
                                             float* __restrict__ depth, int32_t* __restrict__ a_counts) {
  const int64_t ray = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  float T = 1.f, a = 0.f, d = 0.f;
  int na = 0;
  const int64_t e_ = offsets[ray + 1] < cap ? offsets[ray + 1] : cap;
  for (int64_t i = offsets[ray]; i < e_; ++i) {
    const float alpha = __fsub_rn(1.f, expf(__fmul_rn(-sigma[i], __fmul_rn(dist[i], scale))));
    const float w = __fmul_rn(alpha, T);
    weight[i] = w;
    trans[i] = T;
    a += w;
    d = fmaf(w, z[i], d);
    na += w > thres ? 1 : 0;
    T = __fmul_rn(T, __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f));
  }
  t_last[ray] = T; acc[ray] = a; depth[ray] = d; a_counts[ray] = na;
}

// backward of the above incl. feature2density: d L / d feature (valid list).  One WARP per ray: the only sequential
// dependence of raw2alpha's backward is the suffix sum  S_i = sum_{j>i} (dL/dw_j) w_j,  computed with a warp scan over
// 32-sample chunks walked from the far end of the ray (the one-thread-per-ray loop this replaces was 5 % of the step).
__global__ void primary_composite_bwd_kernel(TirField f, const float* __restrict__ feat, const float* __restrict__ sigma,
                                             const float* __restrict__ dist, const float* __restrict__ z,
                                             const int64_t* __restrict__ offsets, int64_t n_rays, float scale,
                                             int64_t cap, const float* __restrict__ weight,
                                             const float* __restrict__ trans, const float* __restrict__ g_weight,
                                             const float* __restrict__ g_acc, const float* __restrict__ g_acc_ext,
                                             const float* __restrict__ g_depth, float* __restrict__ g_feat) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (ray >= n_rays) return;
  const int64_t b = offsets[ray], e = offsets[ray + 1] < cap ? offsets[ray + 1] : cap;
  // acc_map is returned to the caller as well: its own gradient adds to the one coming back through the epilogue
  const float ga = g_acc[ray] + (g_acc_ext ? g_acc_ext[ray] : 0.f), gd = g_depth[ray];
  float carry = 0.f;                                  // sum over the chunks already done (samples farther along the ray)
  for (int64_t top = e; top > b; top -= 32) {
    const int64_t i = top - 1 - lane;                 // lane 0 = farthest sample of the chunk
    const bool on = i >= b;
    float gw = 0.f, t = 0.f;
    if (on) {
      gw = g_weight[i] + ga + gd * z[i];
      t = gw * weight[i];
    }
    float incl = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    const float suffix = carry + (incl - t);          // everything strictly beyond sample i
    carry += __shfl_sync(0xffffffffu, incl, 31);
    if (on) {
      const float d = dist[i] * scale;
      const float ex = expf(-sigma[i] * d);
      const float alpha = 1.f - ex;
      const float om = (1.f - alpha) + 1e-10f;
      const float g_alpha = gw * trans[i] - suffix / om;
      const float g_sigma = g_alpha * d * ex;
      float ds;                                       // d sigma / d feature
      if (f.softplus) {
        const float x = feat[i] + f.density_shift;
        ds = x > 20.f ? 1.f : 1.f / (1.f + expf(-x));
      } else {
        ds = feat[i] > 0.f ? 1.f : 0.f;
      }
      g_feat[i] = g_sigma * ds;
    }
  }
}

// appearance list in the reference's boolean-mask order: one warp per ray walks its segment of the valid list
__global__ void app_fill_kernel(const float* __restrict__ weight, const float* __restrict__ v_xn,
                                const int64_t* __restrict__ offsets, const int64_t* __restrict__ a_offsets,
                                int64_t n_rays, int64_t cap_valid, int64_t cap_app, float thres,
                                int64_t* __restrict__ a_src, int32_t* __restrict__ a_ray, float* __restrict__ a_w,
                                float* __restrict__ a_xn) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (ray >= n_rays) return;
  const int64_t b = offsets[ray], e = offsets[ray + 1] < cap_valid ? offsets[ray + 1] : cap_valid;
  int64_t pos = a_offsets[ray];
  for (int64_t base = b; base < e; base += 32) {
    const int64_t i = base + lane;
    const float w = i < e ? weight[i] : 0.f;
    const bool sel = i < e && w > thres;
    const unsigned m = __ballot_sync(0xffffffffu, sel);
    const int64_t o = pos + __popc(m & ((1u << lane) - 1u));
    if (sel && o < cap_app) {
      a_src[o] = i; a_ray[o] = (int32_t)ray; a_w[o] = w;
#pragma unroll
      for (int c = 0; c < 3; ++c) a_xn[o * 3 + c] = v_xn[i * 3 + c];
    }
    pos += __popc(m);
  }
}

// jittered points of the BRDF smoothness term: xyz + randn * 0.01 (tensorBase:937)
__global__ void jitter_points_kernel(const float* __restrict__ a_xn, const float* __restrict__ noise, int64_t cap,
                                     const int64_t* __restrict__ n_dev, float* __restrict__ a_xj) {
  const int64_t n = list_rows(cap, n_dev) * 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    a_xj[i] = a_xn[i] + noise[i] * 0.01f;
}

// ---- per-sample tail ---------------------------------------------------------------------------------------------------
struct TailPtrs {
  const float* w; const int32_t* ray; const float* rays;      // rays [n_rays,6]: view direction = rays + 3
  const float* rgb; const float* brdf; const float* brdfj; const float* vn;   // head outputs, row stride 4 (vn may be NULL)
  const float* dn_feat; const float* dn_dfdx;                  // derived-normal inputs (may be NULL)
  int normals_kind; int softplus; float shift;
};

// compute_derived_normals (tensorBase:839-856): n = -normalize(d sigma / d x_hat), d sigma = act'(f + shift) * d f
struct DerivedNormal {
  float n[3];
  float gvec[3];     // act' * dfdx
  float dsig, s, norm;
};
__device__ __forceinline__ DerivedNormal derived_normal(const TailPtrs& p, int64_t i) {
  DerivedNormal d;
  const float ft = p.dn_feat[i];
  if (p.softplus) {
    const float x = ft + p.shift;
    d.s = 1.f / (1.f + expf(-x));
    d.dsig = x > 20.f ? 1.f : d.s;
    if (x > 20.f) d.s = -1.f;            // marks the linear branch (no second derivative)
  } else {
    d.dsig = ft > 0.f ? 1.f : 0.f;
    d.s = -1.f;
  }
  float n2 = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) { d.gvec[c] = d.dsig * p.dn_dfdx[i * 3 + c]; n2 += d.gvec[c] * d.gvec[c]; }
  d.norm = sqrtf(n2);
  const float den = fmaxf(d.norm, 1e-6f);     // F.normalize(eps=1e-6)
#pragma unroll
  for (int c = 0; c < 3; ++c) d.n[c] = -d.gvec[c] / den;
  return d;
}

__device__ __forceinline__ TailSample load_tail(const TailPtrs& p, int64_t i, const DerivedNormal* dn) {
  TailSample s;
  s.w = p.w[i];
  const int64_t r = p.ray[i];
  const float4 b = *reinterpret_cast<const float4*>(p.brdf + i * 4), bj = *reinterpret_cast<const float4*>(p.brdfj + i * 4);
  s.brdf[0] = b.x; s.brdf[1] = b.y; s.brdf[2] = b.z; s.brdf[3] = b.w;
  s.brdfj[0] = bj.x; s.brdfj[1] = bj.y; s.brdfj[2] = bj.z; s.brdfj[3] = bj.w;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    s.rgb[c] = p.rgb[i * 4 + c];
    s.vd[c] = __ldg(p.rays + r * 6 + 3 + c);
    s.dn[c] = dn ? dn->n[c] : 0.f;
    s.vn[c] = p.normals_kind == TIR_NORMALS_DERIVED ? dn->n[c] : p.vn[i * 4 + c];
  }
  return s;
}

__global__ void primary_tail_fwd_kernel(TailPtrs p, int64_t cap, const int64_t* __restrict__ n_dev,
                                        float* __restrict__ packed) {
  const int64_t n = list_rows(cap, n_dev);
  const bool both = p.normals_kind == TIR_NORMALS_DERIVED_PLUS_PREDICTED;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    DerivedNormal dn;
    const bool has_dn = p.normals_kind != TIR_NORMALS_PREDICTED;
    if (has_dn) dn = derived_normal(p, i);
    const TailSample s = load_tail(p, i, has_dn ? &dn : nullptr);
    float v[TAIL_CH];
    tail_channels(s, both, v);
    float* dst = packed + (int64_t)p.ray[i] * TAIL_CH;
#pragma unroll
    for (int k = 0; k < TAIL_CH; ++k) atomicAdd(dst + k, s.w * v[k]);
  }
}

struct TailGradPtrs {
  float* g_rgb; float* g_brdf; float* g_brdfj; float* g_vn;   // head output gradients, row stride 4 (g_vn may be NULL)
  float* g_dn_feat; float* g_dn_dfdx;                          // (may be NULL)
  float* g_weight; const int64_t* a_src;                       // d L / d weight scattered to the valid list
};

__global__ void primary_tail_bwd_kernel(TailPtrs p, TailGradPtrs q, int64_t cap, const int64_t* __restrict__ n_dev,
                                        const float* __restrict__ g_packed) {
  const int64_t n = list_rows(cap, n_dev);
  const bool both = p.normals_kind == TIR_NORMALS_DERIVED_PLUS_PREDICTED;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    DerivedNormal dn;
    const bool has_dn = p.normals_kind != TIR_NORMALS_PREDICTED;
    if (has_dn) dn = derived_normal(p, i);
    const TailSample s = load_tail(p, i, has_dn ? &dn : nullptr);
    float G[TAIL_CH];
    const float* src = g_packed + (int64_t)p.ray[i] * TAIL_CH;
#pragma unroll
    for (int k = 0; k < TAIL_CH; ++k) G[k] = __ldg(src + k);
    TailGrad g;
    tail_backward_sample(s, both, G, g);
    q.g_weight[q.a_src[i]] = g.w;
    *reinterpret_cast<float4*>(q.g_rgb + i * 4) = make_float4(g.rgb[0], g.rgb[1], g.rgb[2], 0.f);
    *reinterpret_cast<float4*>(q.g_brdf + i * 4) = make_float4(g.brdf[0], g.brdf[1], g.brdf[2], g.brdf[3]);
    *reinterpret_cast<float4*>(q.g_brdfj + i * 4) = make_float4(g.brdfj[0], g.brdfj[1], g.brdfj[2], g.brdfj[3]);
    if (p.normals_kind != TIR_NORMALS_DERIVED)
      *reinterpret_cast<float4*>(q.g_vn + i * 4) = make_float4(g.vn[0], g.vn[1], g.vn[2], 0.f);
    if (has_dn) {
      // gradient arriving at the derived normal: the |vn - dn|^2 term, plus everything vn receives when it IS the
      // shading normal (purely_derived)
      float gn[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) gn[c] = g.dn[c] + (p.normals_kind == TIR_NORMALS_DERIVED ? g.vn[c] : 0.f);
      // n = -v / max(|v|, eps)
      float gv[3];
      if (dn.norm > 1e-6f) {
        const float inv = 1.f / dn.norm;
        const float dot = -(dn.n[0] * gn[0] + dn.n[1] * gn[1] + dn.n[2] * gn[2]);     // (v/|v|) . gn
#pragma unroll
        for (int c = 0; c < 3; ++c) gv[c] = -(gn[c] - (-dn.n[c]) * dot) * inv;
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) gv[c] = -gn[c] * 1e6f;
      }
      // v = dsig * dfdx
      float g_dsig = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        q.g_dn_dfdx[i * 3 + c] = gv[c] * dn.dsig;
        g_dsig += gv[c] * p.dn_dfdx[i * 3 + c];
      }
      q.g_dn_feat[i] = dn.s >= 0.f ? g_dsig * dn.s * (1.f - dn.s) : 0.f;      // sigmoid' on the softplus branch
    }
  }
}

inline int blocks_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)num_sms() * 8;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

int find_job(const TirHeadJob* jobs, int n_jobs, int role) {
  for (int j = 0; j < n_jobs; ++j)
    if (jobs[j].role == role) return j;
  return -1;
}

int check_jobs(const TirHeadJob* jobs, int n_jobs, int normals_kind, int* j_rgb, int* j_brdf, int* j_brdfj, int* j_n) {
  if (!jobs || n_jobs < 3 || n_jobs > TIR_MAX_HEADS) return TIR_ERR_CONFIG;
  *j_rgb = find_job(jobs, n_jobs, TIR_HEAD_RGB);
  *j_brdf = find_job(jobs, n_jobs, TIR_HEAD_BRDF);
  *j_brdfj = find_job(jobs, n_jobs, TIR_HEAD_BRDF_JITTER);
  *j_n = find_job(jobs, n_jobs, TIR_HEAD_NORMAL);
  if (*j_rgb < 0 || *j_brdf < 0 || *j_brdfj < 0) return TIR_ERR_CONFIG;
  if (normals_kind != TIR_NORMALS_DERIVED && *j_n < 0) return TIR_ERR_CONFIG;
  if (normals_kind < 0 || normals_kind > 2) return TIR_ERR_CONFIG;
  return TIR_OK;
}

TailPtrs tail_ptrs(const TirField* field, const TirPrimaryWork* w, const float* rays, int normals_kind, int j_rgb,
                   int j_brdf, int j_brdfj, int j_n) {
  TailPtrs t{};
  t.w = w->a_w; t.ray = w->a_ray; t.rays = rays;
  t.rgb = w->out[j_rgb]; t.brdf = w->out[j_brdf]; t.brdfj = w->out[j_brdfj]; t.vn = j_n >= 0 ? w->out[j_n] : nullptr;
  t.dn_feat = w->dn_feat; t.dn_dfdx = w->dn_dfdx;
  t.normals_kind = normals_kind; t.softplus = field->softplus; t.shift = field->density_shift;
  return t;
}

}  // namespace

extern "C" int tir_epilogue_fwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                                float fresnel0, int32_t bg, const TirRayMaps* out, uint8_t* acc_mask, float* losses,
                                void* stream);
extern "C" int tir_epilogue_bwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                                float fresnel0, int32_t bg, const TirRayMaps* g_out, const float* g_loss_albedo,
                                const float* g_loss_rough, float* g_packed, float* g_acc, float* g_depth, void* stream);

extern "C" int tir_primary_march(const TirField* field, const float* rays, int64_t n_rays, const TirMarchCfg* cfg,
                                 const TirPrimaryWork* w, uint64_t* counters, void* stream_) {
  if (n_rays <= 0) return TIR_OK;
  if (!field || !rays || !cfg || !w) return TIR_ERR_NULL;
  if (!w->counts || !w->offsets || !w->t_last || !w->acc || !w->depth || !w->a_counts || !w->a_offsets || !w->v_ray ||
      !w->v_sample || !w->v_xn || !w->v_z || !w->v_dist || !w->v_feat || !w->v_sigma || !w->v_weight || !w->v_trans ||
      !w->status)
    return TIR_ERR_NULL;
  if (field->dC != 16) return TIR_ERR_SHAPE;
  if (w->cap_valid <= 0 || w->cap_app <= 0) return TIR_ERR_CAPACITY;
  if (cfg->sampling == TIR_SAMPLE_TABLE && !cfg->z_table) return TIR_ERR_NULL;
  cudaStream_t stream = (cudaStream_t)stream_;
  cudaError_t e = cudaMemsetAsync(w->status, 0, 4 * sizeof(int64_t), stream);
  if (e != cudaSuccess) return (int)e;
  int rc = launch_valid_samples(*field, *cfg, rays, n_rays, false, w->counts, nullptr, nullptr, nullptr, nullptr, nullptr,
                                nullptr, counters, 0, stream);
  if (rc) return rc;
  scan_counts_kernel<<<1, 1024, 0, stream>>>(w->counts, n_rays, w->offsets, w->cap_valid, w->status, 0);
  rc = launch_valid_samples(*field, *cfg, rays, n_rays, true, nullptr, w->offsets, w->v_ray, w->v_sample, w->v_xn,
                            w->v_z, w->v_dist, nullptr, w->cap_valid, stream);
  if (rc) return rc;
  const int64_t* n_valid = w->offsets + n_rays;
  primary_density_kernel<<<blocks_for(w->cap_valid, 128), 128, 0, stream>>>(*field, w->v_xn, w->cap_valid, n_valid,
                                                                            w->v_feat, w->v_sigma);
  primary_composite_fwd_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, stream>>>(
      w->v_sigma, w->v_dist, w->v_z, w->offsets, n_rays, field->distance_scale, w->cap_valid, field->weight_thres,
      w->v_weight, w->v_trans, w->t_last, w->acc, w->depth, w->a_counts);
  scan_counts_kernel<<<1, 1024, 0, stream>>>(w->a_counts, n_rays, w->a_offsets, w->cap_app, w->status, 1);
  return (int)cudaGetLastError();
}

extern "C" int tir_primary_app_list(const TirField* field, int64_t n_rays, const TirPrimaryWork* w, void* stream_) {
  if (n_rays <= 0) return TIR_OK;
  if (!field || !w) return TIR_ERR_NULL;
  if (!w->v_weight || !w->v_xn || !w->offsets || !w->a_offsets || !w->a_src || !w->a_ray || !w->a_w || !w->a_xn)
    return TIR_ERR_NULL;
  const int threads = 256;
  const unsigned blocks = (unsigned)((n_rays * 32 + threads - 1) / threads);
  app_fill_kernel<<<blocks, threads, 0, (cudaStream_t)stream_>>>(w->v_weight, w->v_xn, w->offsets, w->a_offsets, n_rays,
                                                                 w->cap_valid, w->cap_app, field->weight_thres, w->a_src,
                                                                 w->a_ray, w->a_w, w->a_xn);
  return (int)cudaGetLastError();
}

extern "C" int tir_primary_heads(const TirField* field, const TirHeadJob* jobs, int32_t n_jobs, int32_t normals_kind,
                                 const float* rays, const int32_t* light_idx, int64_t n_rays, const TirPrimaryWork* w,
                                 float fresnel0, int32_t white_bg, const TirRayMaps* out, uint8_t* acc_mask,
                                 float* losses, uint64_t* counters, void* stream_) {
  if (n_rays <= 0) return TIR_OK;
  if (!field || !rays || !w || !out || !acc_mask || !losses) return TIR_ERR_NULL;
  int j_rgb, j_brdf, j_brdfj, j_n;
  int rc = check_jobs(jobs, n_jobs, normals_kind, &j_rgb, &j_brdf, &j_brdfj, &j_n);
  if (rc) return rc;
  if (!w->a_src || !w->a_ray || !w->a_w || !w->a_xn || !w->a_xj || !w->noise || !w->packed) return TIR_ERR_NULL;
  if (normals_kind != TIR_NORMALS_PREDICTED && (!w->dn_feat || !w->dn_dfdx)) return TIR_ERR_NULL;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int64_t cap = w->cap_app;
  const int64_t* n_app = w->a_offsets + n_rays;
  jitter_points_kernel<<<blocks_for(cap * 3, 256), 256, 0, stream>>>(w->a_xn, w->noise, cap, n_app, w->a_xj);
  HeadJobDev dev[kMaxHeadJobs];
  for (int j = 0; j < n_jobs; ++j) {
    if (!w->out[j]) return TIR_ERR_NULL;
    HeadJobDev& d = dev[j];
    d = HeadJobDev{};
    d.mlp = jobs[j].mlp;
    d.xn = jobs[j].point_set == 0 ? w->a_xn : w->a_xj;
    if (jobs[j].x_in == 0) { d.x_in = rays + 3; d.x_in_stride = 6; d.x_index = w->a_ray; }
    else { d.x_in = d.xn; d.x_in_stride = 3; d.x_index = nullptr; }
    d.light_mode = jobs[j].mlp.light_line ? jobs[j].light_mode : 0;
    if (d.light_mode == 1) { d.light_idx = light_idx; d.x_index = w->a_ray; }
    if (d.light_mode == 1 && jobs[j].x_in != 0) return TIR_ERR_CONFIG;   // an indexed light needs the ray index table
    d.act = jobs[j].act;
    d.out = w->out[j]; d.out_stride = 4;
    d.save_in = w->inp[j]; d.save_h1 = w->h1[j]; d.save_h2 = w->h2[j];
  }
  // the raw products are dumped once per point set (by the first head that visits it)
  bool saved[2] = {false, false};
  for (int j = 0; j < n_jobs; ++j) {
    const int ps = jobs[j].point_set;
    if (ps < 0 || ps > 1) return TIR_ERR_CONFIG;
    if (!saved[ps] && w->x0[ps]) { dev[j].save_x0 = w->x0[ps]; saved[ps] = true; }
  }
  rc = launch_heads_forward(*field, dev, n_jobs, cap, n_app, stream);
  if (rc) return rc;
  if (normals_kind != TIR_NORMALS_PREDICTED) {
    rc = launch_density_grad(*field, w->a_xn, cap, n_app, w->dn_feat, w->dn_dfdx, stream);
    if (rc) return rc;
  }
  cudaError_t e = cudaMemsetAsync(w->packed, 0, (size_t)n_rays * TAIL_CH * sizeof(float), stream);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemsetAsync(losses, 0, 2 * sizeof(float), stream);
  if (e != cudaSuccess) return (int)e;
  const TailPtrs t = tail_ptrs(field, w, rays, normals_kind, j_rgb, j_brdf, j_brdfj, j_n);
  primary_tail_fwd_kernel<<<blocks_for(cap, 256), 256, 0, stream>>>(t, cap, n_app, w->packed);
  (void)counters;   // appearance samples are counted by the host wrapper from work->status[1]
  return tir_epilogue_fwd(n_rays, w->packed, w->acc, w->depth, rays, fresnel0, white_bg, out, acc_mask, losses, stream_);
}

extern "C" int tir_primary_backward(const TirField* field, const TirHeadJob* jobs, int32_t n_jobs, int32_t normals_kind,
                                    const float* rays, const int32_t* light_idx, int64_t n_rays,
                                    const TirPrimaryWork* w, const TirPrimaryBwdWork* b, float fresnel0,
                                    int32_t white_bg, const TirRayMaps* g_maps, const float* g_acc_map,
                                    const float* g_loss_albedo, const float* g_loss_rough, const TirPrimaryGrads* gr,
                                    void* stream_) {
  if (n_rays <= 0) return TIR_OK;
  if (!field || !rays || !w || !b || !g_maps || !gr) return TIR_ERR_NULL;
  int j_rgb, j_brdf, j_brdfj, j_n;
  int rc = check_jobs(jobs, n_jobs, normals_kind, &j_rgb, &j_brdf, &j_brdfj, &j_n);
  if (rc) return rc;
  if (!b->g_packed || !b->g_acc || !b->g_depth || !b->g_weight || !b->g_feat) return TIR_ERR_NULL;
  if (normals_kind != TIR_NORMALS_PREDICTED && (!b->g_dn_feat || !b->g_dn_dfdx)) return TIR_ERR_NULL;
  if (!w->x0[0] || !w->x0[1]) return TIR_ERR_NULL;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int64_t cap = w->cap_app;
  const int64_t* n_app = w->a_offsets + n_rays;
  const int64_t* n_valid = w->offsets + n_rays;

  // 1. per-ray epilogue
  rc = tir_epilogue_bwd(n_rays, w->packed, w->acc, w->depth, rays, fresnel0, white_bg, g_maps, g_loss_albedo,
                        g_loss_rough, b->g_packed, b->g_acc, b->g_depth, stream_);
  if (rc) return rc;
  // 2. per-sample tail (+ derived normals), d L / d weight scattered onto the valid list
  cudaError_t e = cudaMemsetAsync(b->g_weight, 0, (size_t)w->cap_valid * sizeof(float), stream);
  if (e != cudaSuccess) return (int)e;
  const TailPtrs t = tail_ptrs(field, w, rays, normals_kind, j_rgb, j_brdf, j_brdfj, j_n);
  TailGradPtrs q{};
  q.g_rgb = b->g_out[j_rgb]; q.g_brdf = b->g_out[j_brdf]; q.g_brdfj = b->g_out[j_brdfj];
  q.g_vn = j_n >= 0 ? b->g_out[j_n] : nullptr;
  q.g_dn_feat = b->g_dn_feat; q.g_dn_dfdx = b->g_dn_dfdx; q.g_weight = b->g_weight; q.a_src = w->a_src;
  if (!q.g_rgb || !q.g_brdf || !q.g_brdfj || (normals_kind != TIR_NORMALS_DERIVED && !q.g_vn)) return TIR_ERR_NULL;
  primary_tail_bwd_kernel<<<blocks_for(cap, 256), 256, 0, stream>>>(t, q, cap, n_app, b->g_packed);
  // 3. heads: data gradient + weight gradients
  HeadBwdJob hb[kMaxHeadJobs];
  for (int j = 0; j < n_jobs; ++j) {
    HeadBwdJob& h = hb[j];
    h = HeadBwdJob{};
    h.mlp = jobs[j].mlp;
    h.light_mode = jobs[j].mlp.light_line ? jobs[j].light_mode : 0;
    h.x_index = h.light_mode == 1 ? w->a_ray : nullptr;
    h.light_idx = h.light_mode == 1 ? light_idx : nullptr;
    h.act = jobs[j].act; h.point_set = jobs[j].point_set;
    h.out = w->out[j]; h.out_stride = 4; h.g_out = b->g_out[j];
    h.inp = w->inp[j]; h.h1 = w->h1[j]; h.h2 = w->h2[j];
    h.gz1 = b->gz1[j]; h.gz2 = b->gz2[j]; h.gfeat = b->gfeat[j]; h.gx0 = b->gx0[j];
    h.g_w0 = gr->w0[j]; h.g_b0 = gr->b0[j]; h.g_w1 = gr->w1[j]; h.g_b1 = gr->b1[j]; h.g_w2 = gr->w2[j]; h.g_b2 = gr->b2[j];
  }
  HeadsBwdShared sh{};
  sh.x0[0] = w->x0[0]; sh.x0[1] = w->x0[1]; sh.g_basis = gr->basis; sh.g_light = gr->light_line;
  rc = launch_heads_backward(*field, hb, n_jobs, sh, cap, n_app, stream);
  if (rc) return rc;
  // 4. appearance scatters: one per point set, the heads of a set summed on load
  GradPtrs ga{}, gd{};
  for (int k = 0; k < 3; ++k) {
    ga.plane[k] = gr->aplane[k]; ga.line[k] = gr->aline[k];
    gd.plane[k] = gr->dplane[k]; gd.line[k] = gr->dline[k];
    if (!ga.plane[k] || !ga.line[k] || !gd.plane[k] || !gd.line[k]) return TIR_ERR_NULL;
  }
  for (int ps = 0; ps < 2; ++ps) {
    const float* g3[3] = {nullptr, nullptr, nullptr};
    int m = 0;
    for (int j = 0; j < n_jobs; ++j)
      if (jobs[j].point_set == ps) {
        if (m >= 3) return TIR_ERR_CONFIG;
        g3[m++] = b->gx0[j];
      }
    if (m == 0) continue;
    rc = launch_app_products_bwd(*field, ps == 0 ? w->a_xn : w->a_xj, cap, n_app, g3[0], g3[1], g3[2], ga, stream);
    if (rc) return rc;
  }
  // 5. derived normals: double backward of the density gather (tensorBase:846-853)
  if (normals_kind != TIR_NORMALS_PREDICTED) {
    rc = launch_density_grad_bwd(*field, w->a_xn, cap, n_app, b->g_dn_feat, b->g_dn_dfdx, gd, stream);
    if (rc) return rc;
  }
  // 6. compositing (+ feature2density), acc_map / depth_map gradients folded in
  primary_composite_bwd_kernel<<<(unsigned)((n_rays * 32 + 255) / 256), 256, 0, stream>>>(
      *field, w->v_feat, w->v_sigma, w->v_dist, w->v_z, w->offsets, n_rays, field->distance_scale, w->cap_valid,
      w->v_weight, w->v_trans, b->g_weight, b->g_acc, g_acc_map, b->g_depth, b->g_feat);
  // 7. density scatter
  rc = launch_density_bwd(*field, w->v_xn, w->cap_valid, n_valid, b->g_feat, gd, stream);
  if (rc) return rc;
  return (int)cudaGetLastError();
}
