// Marching cubes over a dense [X,Y,Z] fp32 volume (the native path of the reference's convert_sdf_samples_to_ply,
// utils.py:165-225).  The per-cell math and every topological decision live in tir_mc_body.h.  Two calls, because the
// caller allocates the outputs once the counts are known:
//
//   tir_marching_cubes_count  one pass over the volume, coalesced along z: a CTA holds two consecutive x-planes of a
//                             (8+1) x (32+1) (y, z) tile in shared memory and walks 16 x-planes, writing per point the
//                             crossing bits of its three edges and the triangle count of the cell it starts; warp sums
//                             of both go to two int64 totals.  CUB then scans both arrays and compacts the active
//                             cells (triangle count > 0) into a list.
//   tir_marching_cubes_emit   one thread per point with crossing bits writes its vertices; one thread per active cell
//                             re-reads the cell's corners and writes its triangles at the cell's scanned offset.
//
// Vertices come out by (point linear index, axis), faces by (cell linear index, loop order): reruns are bit-identical.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "tir_device.cuh"
#include "tir_mc_body.h"

namespace {

constexpr int kTZ = 32;          // threads along z (one warp)
constexpr int kTY = 8;           // warps along y
constexpr int kXSteps = 16;      // x-planes per CTA
constexpr int kEmitThreads = 256;

struct Popc {
  __host__ __device__ __forceinline__ int operator()(uint8_t b) const { return (b & 1) + (b >> 1 & 1) + (b >> 2 & 1); }
};
struct Widen {
  __host__ __device__ __forceinline__ int operator()(uint8_t b) const { return (int)b; }
};
using BitsIt = thrust::transform_iterator<Popc, const uint8_t*, int>;
using TrisIt = thrust::transform_iterator<Widen, const uint8_t*, int>;
using CountIt = thrust::counting_iterator<int32_t>;

__global__ void __launch_bounds__(kTZ * kTY) mc_count_kernel(const float* __restrict__ vol, int X, int Y, int Z,
                                                             float level, uint8_t* __restrict__ bits,
                                                             uint8_t* __restrict__ tris,
                                                             unsigned long long* __restrict__ totals) {
  __shared__ float pl[2][kTY + 1][kTZ + 1];
  const int tz = threadIdx.x, ty = threadIdx.y;
  const int k0 = blockIdx.x * kTZ, j0 = blockIdx.y * kTY;
  const int k = k0 + tz, j = j0 + ty;
  const int i0 = blockIdx.z * kXSteps;
  const int i1 = min(i0 + kXSteps, X);
  const int tid = ty * kTZ + tz;
  auto load = [&](int buf, int i) {
    for (int t = tid; t < (kTY + 1) * (kTZ + 1); t += kTY * kTZ) {
      const int yy = t / (kTZ + 1), zz = t - yy * (kTZ + 1);
      const int jj = j0 + yy, kk = k0 + zz;
      float v = 0.f;
      if (i < X && jj < Y && kk < Z) v = __ldg(vol + ((int64_t)i * Y + jj) * Z + kk);
      pl[buf][yy][zz] = v;
    }
  };
  load(0, i0);
  unsigned nv = 0, nt = 0;
  for (int i = i0; i < i1; ++i) {
    const int cur = (i - i0) & 1;
    load(cur ^ 1, i + 1);
    __syncthreads();
    if (j < Y && k < Z) {
      const float v = pl[cur][ty][tz];
      const bool in = mc_inside(v, level);
      unsigned b = 0;
      if (i + 1 < X && mc_inside(pl[cur ^ 1][ty][tz], level) != in) b |= 1;
      if (j + 1 < Y && mc_inside(pl[cur][ty + 1][tz], level) != in) b |= 2;
      if (k + 1 < Z && mc_inside(pl[cur][ty][tz + 1], level) != in) b |= 4;
      int t = 0;
      if (i + 1 < X && j + 1 < Y && k + 1 < Z) {
        float c[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) c[q] = pl[cur ^ (q & 1)][ty + (q >> 1 & 1)][tz + (q >> 2)];
        const unsigned m = mc_cell_mask(c, level);
        if (m != 0 && m != 255) t = mc_cell_triangles(m, mc_face_decisions(c, m, level), nullptr);
      }
      const int64_t p = ((int64_t)i * Y + j) * Z + k;
      bits[p] = (uint8_t)b;
      tris[p] = (uint8_t)t;
      nv += (b & 1) + (b >> 1 & 1) + (b >> 2);
      nt += t;
    }
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
    nt += __shfl_xor_sync(0xffffffffu, nt, o);
  }
  if (tz == 0) {
    if (nv) atomicAdd(totals, (unsigned long long)nv);
    if (nt) atomicAdd(totals + 1, (unsigned long long)nt);
  }
}

struct EmitParams {
  const float* vol;
  int X, Y, Z;
  float level;
  double sp[3];
  const uint8_t* bits;
  const int32_t* voff;
  const int32_t* toff;
  const int32_t* active;
  const int32_t* n_active;
  int64_t cap_v, cap_f;
  float* verts;
  int32_t* faces;
};

__global__ void __launch_bounds__(kEmitThreads) mc_verts_kernel(const EmitParams p) {
  const int64_t n = (int64_t)p.X * p.Y * p.Z;
  const int64_t stride[3] = {(int64_t)p.Y * p.Z, (int64_t)p.Z, 1};
  for (int64_t q = (int64_t)blockIdx.x * kEmitThreads + threadIdx.x; q < n; q += (int64_t)gridDim.x * kEmitThreads) {
    const unsigned b = p.bits[q];
    if (!b) continue;
    const int64_t idx[3] = {q / stride[0], (q / p.Z) % p.Y, q % p.Z};
    const float v = __ldg(p.vol + q);
    int64_t row = p.voff[q];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!(b >> a & 1)) continue;
      if (row < p.cap_v) {
        const float vh = __ldg(p.vol + q + stride[a]);
        float* out = p.verts + row * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          out[c] = c == a ? mc_edge_coord(idx[c], v, vh, p.level, p.sp[c]) : mc_grid_coord(idx[c], p.sp[c]);
      }
      ++row;
    }
  }
}

__global__ void __launch_bounds__(kEmitThreads) mc_faces_kernel(const EmitParams p) {
  const int n_active = *p.n_active;
  const int64_t stride[3] = {(int64_t)p.Y * p.Z, (int64_t)p.Z, 1};
  for (int q = blockIdx.x * kEmitThreads + threadIdx.x; q < n_active; q += gridDim.x * kEmitThreads) {
    const int64_t cell = p.active[q];
    float c[8];
    int64_t pt[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      pt[r] = cell + (r & 1) * stride[0] + (r >> 1 & 1) * stride[1] + (r >> 2);
      c[r] = __ldg(p.vol + pt[r]);
    }
    const unsigned m = mc_cell_mask(c, p.level);
    int8_t tri[3 * MC_MAX_TRIS];
    const int nt = mc_cell_triangles(m, mc_face_decisions(c, m, p.level), tri);
    const int64_t row0 = p.toff[cell];
    for (int t = 0; t < nt; ++t) {
      if (row0 + t >= p.cap_f) break;
      for (int s = 0; s < 3; ++s) {
        const int e = tri[3 * t + s], a = e >> 2;
        const int64_t v = pt[mc_edge_corner(e)];
        p.faces[(row0 + t) * 3 + s] = p.voff[v] + __popc(p.bits[v] & ((1u << a) - 1u));
      }
    }
  }
}

// CUB temporary storage of the three device-wide passes (they run one after the other on one stream)
cudaError_t cub_temp_bytes(int n, size_t* bytes) {
  size_t a = 0, b = 0, c = 0;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, a, BitsIt(nullptr, Popc()), (int32_t*)nullptr, n);
  if (e) return e;
  e = cub::DeviceScan::ExclusiveSum(nullptr, b, TrisIt(nullptr, Widen()), (int32_t*)nullptr, n);
  if (e) return e;
  e = cub::DeviceSelect::Flagged(nullptr, c, CountIt(0), (const uint8_t*)nullptr,
                                 (int32_t*)nullptr, (int32_t*)nullptr, n);
  *bytes = a > b ? (a > c ? a : c) : (b > c ? b : c);
  return e;
}

// the scratch layout of dims that passed the entry's check
cudaError_t work_layout(int32_t X, int32_t Y, int32_t Z, McWork* w, size_t* temp) {
  const int64_t n = (int64_t)X * Y * Z;
  const cudaError_t e = cub_temp_bytes((int)n, temp);
  if (!e) *w = mc_work_layout(n, (int64_t)*temp);
  return e;
}

}  // namespace

extern "C" int tir_marching_cubes_work_size(int32_t X, int32_t Y, int32_t Z, int64_t* bytes) {
  const int rc = mc_work_size_check(X, Y, Z, bytes);
  if (rc < 0) return rc;
  McWork w;
  size_t temp = 0;
  const cudaError_t e = work_layout(X, Y, Z, &w, &temp);
  if (e) return (int)e;
  *bytes = w.total;
  return TIR_OK;
}

extern "C" int tir_marching_cubes_count(const float* volume, int32_t X, int32_t Y, int32_t Z, float level, void* work,
                                        int64_t work_bytes, int64_t* totals, void* stream) {
  const int rc = mc_count_check(volume, X, Y, Z, work, totals);
  if (rc < 0) return rc;
  McWork w;
  size_t temp = 0;
  cudaError_t e = work_layout(X, Y, Z, &w, &temp);
  if (e) return (int)e;
  if (work_bytes < w.total) return TIR_ERR_CAPACITY;
  const cudaStream_t s = (cudaStream_t)stream;
  const int n = (int)((int64_t)X * Y * Z);
  uint8_t* base = (uint8_t*)work;
  uint8_t* bits = base + w.bits;
  uint8_t* tris = base + w.tris;
  e = cudaMemsetAsync(totals, 0, 2 * sizeof(int64_t), s);
  if (e) return (int)e;
  const dim3 grid((Z + kTZ - 1) / kTZ, (Y + kTY - 1) / kTY, (X + kXSteps - 1) / kXSteps);
  mc_count_kernel<<<grid, dim3(kTZ, kTY), 0, s>>>(volume, X, Y, Z, level, bits, tris,
                                                 reinterpret_cast<unsigned long long*>(totals));
  if ((e = cudaGetLastError())) return (int)e;
  e = cub::DeviceScan::ExclusiveSum(base + w.temp, temp, BitsIt(bits, Popc()), (int32_t*)(base + w.voff), n, s);
  if (e) return (int)e;
  e = cub::DeviceScan::ExclusiveSum(base + w.temp, temp, TrisIt(tris, Widen()), (int32_t*)(base + w.toff), n, s);
  if (e) return (int)e;
  e = cub::DeviceSelect::Flagged(base + w.temp, temp, CountIt(0), (const uint8_t*)tris,
                                 (int32_t*)(base + w.active), (int32_t*)(base + w.n_active), n, s);
  return (int)e;
}

extern "C" int tir_marching_cubes_emit(const float* volume, int32_t X, int32_t Y, int32_t Z, float level, double sx,
                                       double sy, double sz, const void* work, int64_t work_bytes, int64_t n_verts,
                                       int64_t n_faces, float* verts, int32_t* faces, void* stream) {
  const int rc = mc_emit_check(volume, X, Y, Z, work, n_verts, n_faces, verts, faces);
  if (rc < 0) return rc;
  McWork w;
  size_t temp = 0;
  cudaError_t e = work_layout(X, Y, Z, &w, &temp);
  if (e) return (int)e;
  if (work_bytes < w.total) return TIR_ERR_CAPACITY;
  const uint8_t* base = (const uint8_t*)work;
  EmitParams p{};
  p.vol = volume; p.X = X; p.Y = Y; p.Z = Z; p.level = level;
  p.sp[0] = sx; p.sp[1] = sy; p.sp[2] = sz;
  p.bits = base + w.bits;
  p.voff = (const int32_t*)(base + w.voff);
  p.toff = (const int32_t*)(base + w.toff);
  p.active = (const int32_t*)(base + w.active);
  p.n_active = (const int32_t*)(base + w.n_active);
  p.cap_v = n_verts; p.cap_f = n_faces; p.verts = verts; p.faces = faces;
  const cudaStream_t s = (cudaStream_t)stream;
  int dev = 0, sms = 0;
  e = cudaGetDevice(&dev);
  if (!e) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e) return (int)e;
  const int64_t n = (int64_t)X * Y * Z;
  if (n_verts > 0) {
    const int64_t blocks = (n + kEmitThreads - 1) / kEmitThreads;
    mc_verts_kernel<<<(unsigned)(blocks < 16LL * sms ? blocks : 16LL * sms), kEmitThreads, 0, s>>>(p);
    if ((e = cudaGetLastError())) return (int)e;
  }
  if (n_faces > 0) {
    // the active-cell count stays on the device: persistent CTAs stride over the list
    const int64_t blocks = (n_faces + kEmitThreads - 1) / kEmitThreads;
    mc_faces_kernel<<<(unsigned)(blocks < 16LL * sms ? blocks : 16LL * sms), kEmitThreads, 0, s>>>(p);
    if ((e = cudaGetLastError())) return (int)e;
  }
  return TIR_OK;
}
