// Point-wise VM gathers with backward, the modular (autograd-facing) half of the primary march:
//   * tir_vm_app_products         plane*line products of the appearance tensors   (tensoRF_rotated_lights.py:141-153)
//   * tir_vm_density_grad         density feature + analytic d f / d x_hat with the clamped-index sampler
//                                 (compute_densityfeature_with_xyz_grad tensoRF:113-129 + relight_utils.py:57-107)
//   * backward scatters of the three gathers into channel-last gradient shadows (float4 atomics, sm_90+, summed over
//     runs of rows that hit the same texel first)
//   * ray-sorted valid-sample lists (count / fill) and the sequential compositing scan with its backward
//     (raw2alpha, tensorBase:21-28)
#include "tir_device.cuh"
#include "tir_internal.h"

using namespace tir;

namespace {

__device__ __forceinline__ void red4(float* p, float4 v) {
  atomicAdd(reinterpret_cast<float4*>(p), v);
}

// Bilinear taps of the custom sampler (relight_utils.py:57-107): weights from unclamped corners, indices clamped,
// plus d w / d ix, d w / d iy.
struct BilinearD {
  int o00, o01, o10, o11;
  float nw, ne, sw, se;
  float dx_nw, dx_ne, dx_sw, dx_se;   // d w / d ix
  float dy_nw, dy_ne, dy_sw, dy_se;   // d w / d iy
};

__device__ __forceinline__ BilinearD bilinear_clamped(float gx, float gy, int W, int H) {
  float ix = unnormalize(gx, W), iy = unnormalize(gy, H);
  float x0f = floorf(ix), y0f = floorf(iy);
  float wx1 = ix - x0f, wx0 = (x0f + 1.f) - ix, wy1 = iy - y0f, wy0 = (y0f + 1.f) - iy;
  int x0 = (int)x0f, y0 = (int)y0f;
  int cx0 = min(max(x0, 0), W - 1), cx1 = min(max(x0 + 1, 0), W - 1);
  int cy0 = min(max(y0, 0), H - 1), cy1 = min(max(y0 + 1, 0), H - 1);
  BilinearD b;
  b.o00 = cy0 * W + cx0; b.o01 = cy0 * W + cx1; b.o10 = cy1 * W + cx0; b.o11 = cy1 * W + cx1;
  b.nw = wx0 * wy0; b.ne = wx1 * wy0; b.sw = wx0 * wy1; b.se = wx1 * wy1;
  b.dx_nw = -wy0; b.dx_ne = wy0; b.dx_sw = -wy1; b.dx_se = wy1;
  b.dy_nw = -wx0; b.dy_ne = -wx1; b.dy_sw = wx0; b.dy_se = wx1;
  return b;
}

struct LinearD {
  int o0, o1;
  float w0, w1;
};

__device__ __forceinline__ LinearD linear_clamped(float gy, int D) {
  float iy = unnormalize(gy, D);
  float y0f = floorf(iy);
  int y0 = (int)y0f;
  LinearD l;
  l.w0 = (y0f + 1.f) - iy; l.w1 = iy - y0f;
  l.o0 = min(max(y0, 0), D - 1); l.o1 = min(max(y0 + 1, 0), D - 1);
  return l;
}

__device__ __forceinline__ float4 f4_comb4(float4 a, float4 b, float4 c, float4 d, float wa, float wb, float wc, float wd) {
  float4 r;
  r.x = a.x * wa + b.x * wb + c.x * wc + d.x * wd;
  r.y = a.y * wa + b.y * wb + c.y * wc + d.y * wd;
  r.z = a.z * wa + b.z * wb + c.z * wc + d.z * wd;
  r.w = a.w * wa + b.w * wb + c.w * wc + d.w * wd;
  return r;
}
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 f4_mul(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4_sub(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float f4_dot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// ------------------------------------------------------------------------------------------------------------------
// appearance products, forward / backward (zero-padding sampler = F.grid_sample)
// ------------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void app_products_kernel(TirField f, const float* __restrict__ xn, int64_t n, float* __restrict__ out) {
  const int64_t total = n * 3;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / 3;
    const int k = (int)(t - i * 3);
    const float x[3] = {xn[i * 3], xn[i * 3 + 1], xn[i * 3 + 2]};
    const int m0 = kMat0[k], m1 = kMat1[k], v = kVec[k];
    const Bilinear b = bilinear_setup(x[m0], x[m1], f.grid[m0], f.grid[m1]);
    const Linear1 l = linear_setup(x[v], f.grid[v]);
    const float* P = f.aplane[k];
    const float* L = f.aline[k];
    float* o = out + i * (3 * C) + k * C;
#pragma unroll 4
    for (int c = 0; c < C; c += 4) {
      const float4 pv = bilerp4(ldg4(P + (size_t)b.o00 * C + c), ldg4(P + (size_t)b.o01 * C + c),
                                ldg4(P + (size_t)b.o10 * C + c), ldg4(P + (size_t)b.o11 * C + c), b);
      const float4 lv = lerp4(ldg4(L + (size_t)l.o0 * C + c), ldg4(L + (size_t)l.o1 * C + c), l);
      *reinterpret_cast<float4*>(o + c) = make_float4(__fmul_rn(pv.x, lv.x), __fmul_rn(pv.y, lv.y),
                                                      __fmul_rn(pv.z, lv.z), __fmul_rn(pv.w, lv.w));
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// density feature + spatial gradient (clamped sampler), forward / backward
// ------------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void density_grad_kernel(TirField f, const float* __restrict__ xn, int64_t n_cap,
                                    const int64_t* __restrict__ n_dev, float* __restrict__ feat,
                                    float* __restrict__ dfdx) {
  const int64_t n = list_rows(n_cap, n_dev);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x[3] = {xn[i * 3], xn[i * 3 + 1], xn[i * 3 + 2]};
    float ft = 0.f, gr[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int m0 = kMat0[k], m1 = kMat1[k], v = kVec[k];
      const int W = f.grid[m0], H = f.grid[m1], D = f.grid[v];
      const BilinearD b = bilinear_clamped(x[m0], x[m1], W, H);
      const LinearD l = linear_clamped(x[v], D);
      const float sx = 0.5f * (W - 1), sy = 0.5f * (H - 1), sl = 0.5f * (D - 1);
      const float* P = f.dplane[k];
      const float* L = f.dline[k];
      // Per-tap channel sums first, then the weight combination: this is the grouping autograd produces for the
      // reference (grad of a broadcast weight = sum over channels), and it makes flat regions give an exact 0.
      float S[4] = {0.f, 0.f, 0.f, 0.f}, R[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < C; c += 4) {
        const float4 a = ldg4(P + (size_t)b.o00 * C + c), bb = ldg4(P + (size_t)b.o01 * C + c),
                     cc = ldg4(P + (size_t)b.o10 * C + c), d = ldg4(P + (size_t)b.o11 * C + c);
        const float4 l0 = ldg4(L + (size_t)l.o0 * C + c), l1 = ldg4(L + (size_t)l.o1 * C + c);
        const float4 lv = f4_add(f4_scale(l0, l.w0), f4_scale(l1, l.w1));
        const float4 dl = f4_sub(l1, l0);
        S[0] += f4_dot(a, lv); S[1] += f4_dot(bb, lv); S[2] += f4_dot(cc, lv); S[3] += f4_dot(d, lv);
        R[0] += f4_dot(a, dl); R[1] += f4_dot(bb, dl); R[2] += f4_dot(cc, dl); R[3] += f4_dot(d, dl);
      }
      const float wy0 = -b.dx_nw, wy1 = -b.dx_sw, wx0 = -b.dy_nw, wx1 = -b.dy_ne;
      const float s = b.nw * S[0] + b.ne * S[1] + b.sw * S[2] + b.se * S[3];
      const float s0 = wy0 * (S[1] - S[0]) + wy1 * (S[3] - S[2]);
      const float s1 = wx0 * (S[2] - S[0]) + wx1 * (S[3] - S[1]);
      const float sv = b.nw * R[0] + b.ne * R[1] + b.sw * R[2] + b.se * R[3];
      ft += s; gr[m0] += s0 * sx; gr[m1] += s1 * sy; gr[v] += sv * sl;
    }
    feat[i] = ft;
    dfdx[i * 3 + 0] = gr[0]; dfdx[i * 3 + 1] = gr[1]; dfdx[i * 3 + 2] = gr[2];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// gradient scatters of the three gathers: float4 atomics into channel-last gradient shadows, summed per run first
// ------------------------------------------------------------------------------------------------------------------
// A group of C/4 consecutive threads (one 4-channel chunk each, so a group covers whole texels and a warp's atomics fill
// whole 32-byte sectors) walks kScatterRows consecutive rows of a list for one orientation.  The valid and appearance
// lists are sorted by ray and a ray's samples are half a voxel apart, so consecutive rows often hit the same tap texel:
// each of the 6 taps keeps its open run (texel, sum so far) in registers and issues one atomic when its texel changes
// or the block ends.  The merge compares texels, not rays, so it is exact for any row order (an unsorted list only
// merges less), and a run adds as many terms into an entry as its rows would one by one.
constexpr int kScatterRows = 8;

struct TapRun {
  int key;       // texel of the open run, -1: none
  float4 acc;
};

// what one row adds to its 4 plane taps and 2 line taps; key -1: nothing (zero tap weight)
struct RowTaps {
  int key[6];
  float4 v[6];
};

__device__ __forceinline__ void run_add(TapRun& r, float* g, int C, int key, float4 v) {
  if (key < 0) return;
  if (key == r.key) {
    r.acc = f4_add(r.acc, v);
    return;
  }
  if (r.key >= 0) red4(g + (size_t)r.key * C, r.acc);
  r.key = key;
  r.acc = v;
}

// zero-padding sampler: taps with a zero weight add nothing
__device__ __forceinline__ void zero_padded_taps(const Bilinear& b, const Linear1& l, float4 gp, float4 gl, RowTaps& r) {
  r.key[0] = b.nw != 0.f ? b.o00 : -1; r.v[0] = f4_scale(gp, b.nw);
  r.key[1] = b.ne != 0.f ? b.o01 : -1; r.v[1] = f4_scale(gp, b.ne);
  r.key[2] = b.sw != 0.f ? b.o10 : -1; r.v[2] = f4_scale(gp, b.sw);
  r.key[3] = b.se != 0.f ? b.o11 : -1; r.v[3] = f4_scale(gp, b.se);
  r.key[4] = l.w0 != 0.f ? l.o0 : -1; r.v[4] = f4_scale(gl, l.w0);
  r.key[5] = l.w1 != 0.f ? l.o1 : -1; r.v[5] = f4_scale(gl, l.w1);
}

// coordinates of a point on plane k's two axes and line k's axis (kMat0 / kMat1 / kVec without an indexed local array)
struct Orient {
  float a, b, v;
};
__device__ __forceinline__ Orient orient(const float* xn, int64_t i, int k) {
  const float x0 = xn[i * 3], x1 = xn[i * 3 + 1], x2 = xn[i * 3 + 2];
  return Orient{k == 2 ? x1 : x0, k == 0 ? x1 : x2, k == 0 ? x2 : (k == 1 ? x1 : x0)};
}

// density feature backward (zero-padding sampler): d L / d feature[i] = g[i]; rows with g[i] == 0 are skipped
struct DensityRows {
  static constexpr int C = 16;
  const float* xn;
  const float* g;
  __device__ __forceinline__ bool row(const TirField& f, int64_t i, int k, int c, RowTaps& r) const {
    const float gi = g[i];
    if (gi == 0.f) return false;
    const Orient x = orient(xn, i, k);
    const Bilinear b = bilinear_setup(x.a, x.b, f.grid[kMat0[k]], f.grid[kMat1[k]]);
    const Linear1 l = linear_setup(x.v, f.grid[kVec[k]]);
    const float* P = f.dplane[k];
    const float* L = f.dline[k];
    const float4 pv = bilerp4(ldg4(P + (size_t)b.o00 * C + c), ldg4(P + (size_t)b.o01 * C + c),
                              ldg4(P + (size_t)b.o10 * C + c), ldg4(P + (size_t)b.o11 * C + c), b);
    const float4 lv = lerp4(ldg4(L + (size_t)l.o0 * C + c), ldg4(L + (size_t)l.o1 * C + c), l);
    zero_padded_taps(b, l, f4_scale(lv, gi), f4_scale(pv, gi), r);
    return true;
  }
};

// appearance products backward (zero-padding sampler): d L / d product = g0 (+ g1 + g2, heads sharing the points)
struct AppRows {
  static constexpr int C = 48;
  const float* xn;
  const float* g0;
  const float* g1;
  const float* g2;
  __device__ __forceinline__ bool row(const TirField& f, int64_t i, int k, int c, RowTaps& r) const {
    const Orient x = orient(xn, i, k);
    const Bilinear b = bilinear_setup(x.a, x.b, f.grid[kMat0[k]], f.grid[kMat1[k]]);
    const Linear1 l = linear_setup(x.v, f.grid[kVec[k]]);
    const float* P = f.aplane[k];
    const float* L = f.aline[k];
    const int64_t go_off = i * (3 * C) + k * C + c;
    float4 gv = *reinterpret_cast<const float4*>(g0 + go_off);
    if (g1) gv = f4_add(gv, *reinterpret_cast<const float4*>(g1 + go_off));
    if (g2) gv = f4_add(gv, *reinterpret_cast<const float4*>(g2 + go_off));
    const float4 pv = bilerp4(ldg4(P + (size_t)b.o00 * C + c), ldg4(P + (size_t)b.o01 * C + c),
                              ldg4(P + (size_t)b.o10 * C + c), ldg4(P + (size_t)b.o11 * C + c), b);
    const float4 lv = lerp4(ldg4(L + (size_t)l.o0 * C + c), ldg4(L + (size_t)l.o1 * C + c), l);
    zero_padded_taps(b, l, f4_mul(gv, lv), f4_mul(gv, pv), r);   // d/d plane value, d/d line value
    return true;
  }
};

// backward of density_grad_kernel (clamped sampler) from g_feat and / or g_dfdx (NULL: zero); every tap adds
struct DensityGradRows {
  static constexpr int C = 16;
  const float* xn;
  const float* g_feat;
  const float* g_dfdx;
  __device__ __forceinline__ bool row(const TirField& f, int64_t i, int k, int c, RowTaps& r) const {
    const Orient x = orient(xn, i, k);
    const int m0 = kMat0[k], m1 = kMat1[k], v = kVec[k];
    const int W = f.grid[m0], H = f.grid[m1], D = f.grid[v];
    const BilinearD b = bilinear_clamped(x.a, x.b, W, H);
    const LinearD l = linear_clamped(x.v, D);
    const float sx = 0.5f * (W - 1), sy = 0.5f * (H - 1), sl = 0.5f * (D - 1);
    const float gf = g_feat ? g_feat[i] : 0.f;
    const float g0 = g_dfdx ? g_dfdx[i * 3 + m0] * sx : 0.f;
    const float g1 = g_dfdx ? g_dfdx[i * 3 + m1] * sy : 0.f;
    const float gv = g_dfdx ? g_dfdx[i * 3 + v] * sl : 0.f;
    // coefficient of P_t: lv*(gf*w_t + g0*dwx_t + g1*dwy_t) + dl*(gv*w_t)
    const float a_nw = gf * b.nw + g0 * b.dx_nw + g1 * b.dy_nw, a_ne = gf * b.ne + g0 * b.dx_ne + g1 * b.dy_ne;
    const float a_sw = gf * b.sw + g0 * b.dx_sw + g1 * b.dy_sw, a_se = gf * b.se + g0 * b.dx_se + g1 * b.dy_se;
    const float* P = f.dplane[k];
    const float* L = f.dline[k];
    const float4 a = ldg4(P + (size_t)b.o00 * C + c), bb = ldg4(P + (size_t)b.o01 * C + c),
                 cc = ldg4(P + (size_t)b.o10 * C + c), d = ldg4(P + (size_t)b.o11 * C + c);
    const float4 l0 = ldg4(L + (size_t)l.o0 * C + c), l1 = ldg4(L + (size_t)l.o1 * C + c);
    const float4 pv = f4_comb4(a, bb, cc, d, b.nw, b.ne, b.sw, b.se);
    const float4 px = f4_comb4(a, bb, cc, d, b.dx_nw, b.dx_ne, b.dx_sw, b.dx_se);
    const float4 py = f4_comb4(a, bb, cc, d, b.dy_nw, b.dy_ne, b.dy_sw, b.dy_se);
    const float4 lv = f4_add(f4_scale(l0, l.w0), f4_scale(l1, l.w1));
    const float4 dl = f4_sub(l1, l0);
    r.key[0] = b.o00; r.v[0] = f4_add(f4_scale(lv, a_nw), f4_scale(dl, gv * b.nw));
    r.key[1] = b.o01; r.v[1] = f4_add(f4_scale(lv, a_ne), f4_scale(dl, gv * b.ne));
    r.key[2] = b.o10; r.v[2] = f4_add(f4_scale(lv, a_sw), f4_scale(dl, gv * b.sw));
    r.key[3] = b.o11; r.v[3] = f4_add(f4_scale(lv, a_se), f4_scale(dl, gv * b.se));
    // coefficient of L_u: pv*(gf*wl_u -/+ gv) + wl_u*(g0*px + g1*py)
    const float4 q = f4_add(f4_scale(px, g0), f4_scale(py, g1));
    r.key[4] = l.o0; r.v[4] = f4_add(f4_scale(pv, gf * l.w0 - gv), f4_scale(q, l.w0));
    r.key[5] = l.o1; r.v[5] = f4_add(f4_scale(pv, gf * l.w1 + gv), f4_scale(q, l.w1));
    return true;
  }
};

// threads of a scatter over n rows: one group of C/4 per (orientation, block of kScatterRows rows)
inline int64_t scatter_threads(int64_t n, int C) { return 3 * ((n + kScatterRows - 1) / kScatterRows) * (C / 4); }

// grid-stride over the (orientation, row block, chunk) threads t0, t0 + stride, ... of a list of n rows
template <class Rows>
__device__ __forceinline__ void scatter_rows(const TirField& f, const Rows& rows, const GradPtrs& g, int64_t n,
                                             int64_t t0, int64_t stride) {
  constexpr int C = Rows::C, Q = C / 4;
  const int64_t blocks = (n + kScatterRows - 1) / kScatterRows;
  const int64_t total = blocks * 3 * Q;
  for (int64_t t = t0; t < total; t += stride) {
    const int64_t grp = t / Q;
    const int c = (int)(t - grp * Q) * 4;
    const int k = (int)(grp / blocks);
    const int64_t i0 = (grp - k * blocks) * kScatterRows;
    const int64_t i1 = i0 + kScatterRows < n ? i0 + kScatterRows : n;
    float* gp = (k == 0 ? g.plane[0] : k == 1 ? g.plane[1] : g.plane[2]) + c;   // no indexed copy of g
    float* gl = (k == 0 ? g.line[0] : k == 1 ? g.line[1] : g.line[2]) + c;
    TapRun run[6];
#pragma unroll
    for (int u = 0; u < 6; ++u) run[u] = TapRun{-1, make_float4(0.f, 0.f, 0.f, 0.f)};
    for (int64_t i = i0; i < i1; ++i) {
      RowTaps r;
      if (!rows.row(f, i, k, c, r)) continue;
#pragma unroll
      for (int u = 0; u < 6; ++u) run_add(run[u], u < 4 ? gp : gl, C, r.key[u], r.v[u]);
    }
#pragma unroll
    for (int u = 0; u < 6; ++u)
      if (run[u].key >= 0) red4((u < 4 ? gp : gl) + (size_t)run[u].key * C, run[u].acc);
  }
}

__global__ void __launch_bounds__(128, 4) density_bwd_kernel(TirField f, DensityRows rows, int64_t n_cap,
                                                          const int64_t* __restrict__ n_dev, GradPtrs g) {
  scatter_rows(f, rows, g, list_rows(n_cap, n_dev), blockIdx.x * (int64_t)blockDim.x + threadIdx.x,
               (int64_t)gridDim.x * blockDim.x);
}

// the scatters of one appearance list (AppScatterJob) in one launch: job j runs on its own range of job[j].ctas CTAs
struct AppScatterLaunch {
  AppScatterJob job[kMaxAppScatterJobs];
  int n_jobs;
  int64_t n_cap;
  const int64_t* n_dev;
};

__global__ void __launch_bounds__(128, 4) app_scatter_kernel(TirField f, AppScatterLaunch p) {
  int b = blockIdx.x, j = 0;
  while (j + 1 < p.n_jobs && b >= p.job[j].ctas) b -= p.job[j].ctas, ++j;
  const AppScatterJob& J = p.job[j];
  const int64_t n = list_rows(p.n_cap, p.n_dev);
  const int64_t t0 = b * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)J.ctas * blockDim.x;
  if (J.density_grad)
    scatter_rows(f, DensityGradRows{J.xn, J.g[0], J.g[1]}, J.out, n, t0, stride);
  else
    scatter_rows(f, AppRows{J.xn, J.g[0], J.g[1], J.g[2]}, J.out, n, t0, stride);
}

// ------------------------------------------------------------------------------------------------------------------
// ray-sorted valid sample lists (sample_ray + alpha-mask filter), one warp per ray
// ------------------------------------------------------------------------------------------------------------------
template <bool FILL>
__global__ void valid_samples_kernel(TirField f, TirMarchCfg cfg, const float* __restrict__ rays_o,
                                     const float* __restrict__ rays_d, int64_t n_rays, int32_t* __restrict__ counts,
                                     const int64_t* __restrict__ offsets, int32_t* __restrict__ out_ray,
                                     int32_t* __restrict__ out_sample, float* __restrict__ out_xn,
                                     float* __restrict__ out_z, float* __restrict__ out_dist,
                                     unsigned long long* counters, int64_t capacity, int stride) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (ray >= n_rays) return;
  const float ox = rays_o[ray * stride], oy = rays_o[ray * stride + 1], oz = rays_o[ray * stride + 2];
  const float dx = rays_d[ray * stride], dy = rays_d[ray * stride + 1], dz = rays_d[ray * stride + 2];
  const int N = cfg.n_samples;
  float tmin = 0.f, jit = 0.f;
  if (cfg.sampling == TIR_SAMPLE_STEP) {
    const float vx = dx == 0.f ? 1e-6f : dx, vy = dy == 0.f ? 1e-6f : dy, vz = dz == 0.f ? 1e-6f : dz;
    const float ax = __fdiv_rn(__fsub_rn(f.aabb_hi[0], ox), vx), bx = __fdiv_rn(__fsub_rn(f.aabb_lo[0], ox), vx);
    const float ay = __fdiv_rn(__fsub_rn(f.aabb_hi[1], oy), vy), by = __fdiv_rn(__fsub_rn(f.aabb_lo[1], oy), vy);
    const float az = __fdiv_rn(__fsub_rn(f.aabb_hi[2], oz), vz), bz = __fdiv_rn(__fsub_rn(f.aabb_lo[2], oz), vz);
    tmin = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz));
    tmin = fminf(fmaxf(tmin, cfg.near), cfg.far);
    jit = cfg.jitter ? cfg.jitter[ray] : 0.f;
  }
  auto z_of = [&](int s) -> float {
    if (cfg.sampling == TIR_SAMPLE_STEP) return __fadd_rn(tmin, __fmul_rn(cfg.step, __fadd_rn((float)s, jit)));
    return cfg.z_table[s];
  };
  // occupancy bricks read through L1 (4 KB at 256^3): a per-CTA copy would cost more than the 8 rays of a CTA read
  const CellBricks bricks = cell_bricks(f, f.amask ? global_bricks(f, cfg) : nullptr);
  int64_t pos = FILL ? offsets[ray] : 0;
  int cnt = 0;
  unsigned long long c_mask = 0;
  for (int base = 0; base < N; base += 32) {
    const int s = base + lane;
    bool valid = false;
    float z = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
    if (s < N) {
      z = z_of(s);
      const float px = __fadd_rn(ox, __fmul_rn(dx, z)), py = __fadd_rn(oy, __fmul_rn(dy, z)),
                  pz = __fadd_rn(oz, __fmul_rn(dz, z));
      const bool out = (f.aabb_lo[0] > px) | (px > f.aabb_hi[0]) | (f.aabb_lo[1] > py) | (py > f.aabb_hi[1]) |
                       (f.aabb_lo[2] > pz) | (pz > f.aabb_hi[2]);
      if (!out || (cfg.flags & TIR_MARCH_NO_BBOX)) {
        valid = true;
        if (f.amask) { c_mask += 1; valid = alpha_mask_positive(f, px, py, pz, bricks); }
        nx = __fsub_rn(__fmul_rn(__fsub_rn(px, f.aabb_lo[0]), f.inv_aabb[0]), 1.f);
        ny = __fsub_rn(__fmul_rn(__fsub_rn(py, f.aabb_lo[1]), f.inv_aabb[1]), 1.f);
        nz = __fsub_rn(__fmul_rn(__fsub_rn(pz, f.aabb_lo[2]), f.inv_aabb[2]), 1.f);
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if (FILL && valid && (pos + __popc(m & ((1u << lane) - 1u)) < capacity)) {
      const int64_t o = pos + __popc(m & ((1u << lane) - 1u));
      out_ray[o] = (int32_t)ray; out_sample[o] = s;
      out_xn[o * 3] = nx; out_xn[o * 3 + 1] = ny; out_xn[o * 3 + 2] = nz;
      out_z[o] = z;
      out_dist[o] = (s + 1 < N) ? __fsub_rn(z_of(s + 1), z) : 0.f;
    }
    pos += __popc(m);
    cnt += __popc(m);
  }
  if (!FILL) {
    if (lane == 0) counts[ray] = cnt;
    c_mask = warp_sum_u64(c_mask);
    if (lane == 0 && counters) {
      if (c_mask) atomicAdd(counters + TIR_CNT_MASK, c_mask);
      if (cnt) atomicAdd(counters + TIR_CNT_DENSITY, (unsigned long long)cnt);
      atomicAdd(counters + TIR_CNT_RAYS, 1ull);
    }
  }
}

// raw2alpha over ray segments, sequential like torch.cumprod: one thread per ray.
__global__ void composite_fwd_kernel(const float* __restrict__ sigma, const float* __restrict__ dist,
                                     const int64_t* __restrict__ offsets, int64_t n_rays, float scale,
                                     float* __restrict__ weight, float* __restrict__ trans,
                                     float* __restrict__ t_last, int64_t limit, const float* __restrict__ z,
                                     float* __restrict__ acc, float* __restrict__ depth) {
  const int64_t ray = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  float T = 1.f, a = 0.f, d = 0.f;
  const int64_t e_ = offsets[ray + 1] < limit ? offsets[ray + 1] : limit;
  for (int64_t i = offsets[ray]; i < e_; ++i) {
    const float alpha = __fsub_rn(1.f, expf(__fmul_rn(-sigma[i], __fmul_rn(dist[i], scale))));
    const float w = __fmul_rn(alpha, T);
    weight[i] = w;
    trans[i] = T;
    a += w;
    if (z) d = fmaf(w, z[i], d);
    T = __fmul_rn(T, __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f));
  }
  if (t_last) t_last[ray] = T;
  if (acc) acc[ray] = a;                 // acc_map = sum_s weight          (tensorBase:974)
  if (depth) depth[ray] = d;             // depth_map = sum_s weight * z    (tensorBase:975)
}

__global__ void composite_bwd_kernel(const float* __restrict__ sigma, const float* __restrict__ dist,
                                     const int64_t* __restrict__ offsets, int64_t n_rays, float scale,
                                     const float* __restrict__ weight, const float* __restrict__ trans,
                                     const float* __restrict__ g_weight, float* __restrict__ g_sigma,
                                     int64_t limit, const float* __restrict__ z, const float* __restrict__ g_acc,
                                     const float* __restrict__ g_depth) {
  const int64_t ray = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  const int64_t b = offsets[ray], e = offsets[ray + 1] < limit ? offsets[ray + 1] : limit;
  float suffix = 0.f;   // sum_{j>i} g_j * w_j
  const float ga = g_acc ? g_acc[ray] : 0.f, gd = (g_depth && z) ? g_depth[ray] : 0.f;
  for (int64_t i = e - 1; i >= b; --i) {
    const float d = dist[i] * scale;
    const float ex = expf(-sigma[i] * d);
    const float alpha = 1.f - ex;
    const float om = (1.f - alpha) + 1e-10f;
    const float gw = (g_weight ? g_weight[i] : 0.f) + ga + (z ? gd * z[i] : 0.f);   // d/d weight_i incl. acc / depth
    const float g_alpha = gw * trans[i] - suffix / om;
    g_sigma[i] = g_alpha * d * ex;
    suffix += gw * weight[i];
  }
}

inline int blocks_for(int64_t n, int threads, int cap = 0) {
  if (cap <= 0) cap = num_sms() * 16;
  int64_t b = (n + threads - 1) / threads;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

namespace tir {
int launch_valid_samples(const TirField& f, const TirMarchCfg& cfg, const float* rays, int64_t n_rays, bool fill,
                         int32_t* counts, const int64_t* offsets, int32_t* out_ray, int32_t* out_sample, float* out_xn,
                         float* out_z, float* out_dist, uint64_t* counters, int64_t capacity, cudaStream_t stream) {
  if (n_rays <= 0) return TIR_OK;
  const int threads = 256;
  const unsigned blocks = (unsigned)((n_rays * 32 + threads - 1) / threads);
  if (fill)
    valid_samples_kernel<true><<<blocks, threads, 0, stream>>>(f, cfg, rays, rays + 3, n_rays, nullptr, offsets, out_ray,
                                                               out_sample, out_xn, out_z, out_dist, nullptr, capacity, 6);
  else
    valid_samples_kernel<false><<<blocks, threads, 0, stream>>>(f, cfg, rays, rays + 3, n_rays, counts, nullptr, nullptr,
                                                                nullptr, nullptr, nullptr, nullptr,
                                                                (unsigned long long*)counters, 0, 6);
  return (int)cudaGetLastError();
}
int launch_density_bwd(const TirField& f, const float* xn, int64_t n, const int64_t* n_dev, const float* g_feature,
                       const GradPtrs& g, cudaStream_t stream) {
  if (n <= 0) return TIR_OK;
  if (f.dC != 16) return TIR_ERR_SHAPE;
  density_bwd_kernel<<<blocks_for(scatter_threads(n, 16), 128), 128, 0, stream>>>(f, DensityRows{xn, g_feature}, n,
                                                                                  n_dev, g);
  return (int)cudaGetLastError();
}
int launch_app_scatter(const TirField& f, AppScatterJob* jobs, int n_jobs, int64_t n, const int64_t* n_dev,
                       cudaStream_t stream) {
  if (n <= 0 || n_jobs <= 0) return TIR_OK;
  if (n_jobs > kMaxAppScatterJobs) return TIR_ERR_CONFIG;
  AppScatterLaunch p{};
  int64_t threads[kMaxAppScatterJobs], sum = 0;
  for (int j = 0; j < n_jobs; ++j) {
    if (jobs[j].density_grad ? f.dC != 16 : f.aC != 48) return TIR_ERR_SHAPE;
    threads[j] = scatter_threads(n, jobs[j].density_grad ? 16 : 48);
    sum += threads[j];
  }
  const int total = blocks_for(sum, 128);
  int ctas = 0;
  for (int j = 0; j < n_jobs; ++j) {
    jobs[j].ctas = (int)((double)total * threads[j] / sum + 0.5);
    if (jobs[j].ctas < 1) jobs[j].ctas = 1;
    p.job[j] = jobs[j];
    ctas += jobs[j].ctas;
  }
  p.n_jobs = n_jobs; p.n_cap = n; p.n_dev = n_dev;
  app_scatter_kernel<<<ctas, 128, 0, stream>>>(f, p);
  return (int)cudaGetLastError();
}
int launch_density_grad(const TirField& f, const float* xn, int64_t n, const int64_t* n_dev, float* feature,
                        float* dfdx, cudaStream_t stream) {
  if (n <= 0) return TIR_OK;
  if (f.dC != 16) return TIR_ERR_SHAPE;
  density_grad_kernel<16><<<blocks_for(n, 128), 128, 0, stream>>>(f, xn, n, n_dev, feature, dfdx);
  return (int)cudaGetLastError();
}
}  // namespace tir

extern "C" int tir_vm_app_products(const TirField* field, const float* xn, int64_t n, float* out, void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xn || !out) return TIR_ERR_NULL;
  if (field->aC != 48) return TIR_ERR_SHAPE;
  app_products_kernel<48><<<blocks_for(n * 3, 128), 128, 0, (cudaStream_t)stream>>>(*field, xn, n, out);
  return (int)cudaGetLastError();
}

extern "C" int tir_vm_app_products_bwd(const TirField* field, const float* xn, int64_t n, const float* g_out,
                                       float* const* g_plane, float* const* g_line, void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xn || !g_out || !g_plane || !g_line) return TIR_ERR_NULL;
  if (field->aC != 48) return TIR_ERR_SHAPE;
  AppScatterJob j{};
  j.xn = xn; j.g[0] = g_out;
  for (int k = 0; k < 3; ++k) { j.out.plane[k] = g_plane[k]; j.out.line[k] = g_line[k]; }
  return launch_app_scatter(*field, &j, 1, n, nullptr, (cudaStream_t)stream);
}

extern "C" int tir_vm_density_bwd(const TirField* field, const float* xn, int64_t n, const float* g_feature,
                                  float* const* g_plane, float* const* g_line, void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xn || !g_feature || !g_plane || !g_line) return TIR_ERR_NULL;
  if (field->dC != 16) return TIR_ERR_SHAPE;
  GradPtrs g;
  for (int k = 0; k < 3; ++k) { g.plane[k] = g_plane[k]; g.line[k] = g_line[k]; }
  return launch_density_bwd(*field, xn, n, nullptr, g_feature, g, (cudaStream_t)stream);
}

extern "C" int tir_vm_density_grad(const TirField* field, const float* xn, int64_t n, float* feature, float* dfdx,
                                   void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xn || !feature || !dfdx) return TIR_ERR_NULL;
  if (field->dC != 16) return TIR_ERR_SHAPE;
  density_grad_kernel<16><<<blocks_for(n, 128), 128, 0, (cudaStream_t)stream>>>(*field, xn, n, nullptr, feature, dfdx);
  return (int)cudaGetLastError();
}

extern "C" int tir_vm_density_grad_bwd(const TirField* field, const float* xn, int64_t n, const float* g_feature,
                                       const float* g_dfdx, float* const* g_plane, float* const* g_line,
                                       void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xn || !g_plane || !g_line) return TIR_ERR_NULL;
  if (field->dC != 16) return TIR_ERR_SHAPE;
  AppScatterJob j{};
  j.density_grad = 1; j.xn = xn; j.g[0] = g_feature; j.g[1] = g_dfdx;
  for (int k = 0; k < 3; ++k) { j.out.plane[k] = g_plane[k]; j.out.line[k] = g_line[k]; }
  return launch_app_scatter(*field, &j, 1, n, nullptr, (cudaStream_t)stream);
}

extern "C" int tir_valid_samples_count(const TirField* field, const float* rays_o, const float* rays_d,
                                       int64_t n_rays, const TirMarchCfg* cfg, int32_t* counts, uint64_t* counters,
                                       void* stream) {
  if (n_rays <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !rays_o || !rays_d || !cfg || !counts) return TIR_ERR_NULL;
  if (n_rays <= 0) return TIR_OK;
  if (cfg->sampling == TIR_SAMPLE_TABLE && !cfg->z_table) return TIR_ERR_NULL;
  const int threads = 256;
  const int64_t blocks = (n_rays * 32 + threads - 1) / threads;
  valid_samples_kernel<false><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      *field, *cfg, rays_o, rays_d, n_rays, counts, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
      (unsigned long long*)counters, 0, 3);
  return (int)cudaGetLastError();
}

extern "C" int tir_valid_samples_fill(const TirField* field, const float* rays_o, const float* rays_d,
                                      int64_t n_rays, const TirMarchCfg* cfg, const int64_t* offsets,
                                      int32_t* out_ray, int32_t* out_sample, float* out_xn, float* out_z,
                                      float* out_dist, int64_t capacity, void* stream) {
  if (n_rays <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !rays_o || !rays_d || !cfg || !offsets || !out_ray || !out_sample || !out_xn || !out_z || !out_dist)
    return TIR_ERR_NULL;
  if (n_rays <= 0) return TIR_OK;
  const int threads = 256;
  const int64_t blocks = (n_rays * 32 + threads - 1) / threads;
  valid_samples_kernel<true><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      *field, *cfg, rays_o, rays_d, n_rays, nullptr, offsets, out_ray, out_sample, out_xn, out_z, out_dist, nullptr,
      capacity > 0 ? capacity : (int64_t)1 << 62, 3);
  return (int)cudaGetLastError();
}

extern "C" int tir_composite_fwd(const float* sigma, const float* dist, const int64_t* offsets, int64_t n_rays,
                                 float distance_scale, float* weight, float* trans, float* t_last, int64_t limit,
                                 const float* z, float* acc, float* depth, void* stream) {
  if (n_rays <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!sigma || !dist || !offsets || !weight || !trans) return TIR_ERR_NULL;
  if (n_rays <= 0) return TIR_OK;
  composite_fwd_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      sigma, dist, offsets, n_rays, distance_scale, weight, trans, t_last, limit > 0 ? limit : (int64_t)1 << 62, z, acc,
      depth);
  return (int)cudaGetLastError();
}

extern "C" int tir_composite_bwd(const float* sigma, const float* dist, const int64_t* offsets, int64_t n_rays,
                                 float distance_scale, const float* weight, const float* trans,
                                 const float* g_weight, float* g_sigma, int64_t limit, const float* z,
                                 const float* g_acc, const float* g_depth, void* stream) {
  if (n_rays <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!sigma || !dist || !offsets || !weight || !trans || !g_sigma) return TIR_ERR_NULL;
  if (n_rays <= 0) return TIR_OK;
  composite_bwd_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      sigma, dist, offsets, n_rays, distance_scale, weight, trans, g_weight, g_sigma,
      limit > 0 ? limit : (int64_t)1 << 62, z, g_acc, g_depth);
  return (int)cudaGetLastError();
}
