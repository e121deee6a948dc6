// Texture atlas of the textured glTF export (tir_atlas_texels / _encode / _corners, include/tensoir_b200.h): one
// thread per texel or per face, the layout and all per-texel math in tir_atlas_body.h.  No atomics: every output
// element has one writer, so repeated calls give identical bits.
#include "tir_device.cuh"
#include "tir_atlas_body.h"

namespace {

constexpr int kThreads = 256;

unsigned grid_for(int64_t n) {
  const int64_t blocks = (n + kThreads - 1) / kThreads;
  return (unsigned)(blocks < (1 << 20) ? blocks : (1 << 20));      // grid-stride loops cover the rest
}

__global__ void __launch_bounds__(kThreads) atlas_texels_kernel(const int32_t* __restrict__ faces,
                                                                const float* __restrict__ v, int32_t T, int32_t s,
                                                                int64_t first, int64_t n, int32_t* __restrict__ pix,
                                                                float* __restrict__ pos) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const AtTexel tx = at_texel(first + i, T, s);
    int32_t c[3];
    at_corners(faces, tx.face, c);
    float b[3], p[3];
    at_bary(s, tx.ia, tx.ja, b);
    at_point(v, c, b, p);
    pix[i] = tx.y * T + tx.x;
#pragma unroll
    for (int k = 0; k < 3; ++k) pos[i * 3 + k] = p[k];
  }
}

__global__ void __launch_bounds__(kThreads) atlas_encode_kernel(
    const int32_t* __restrict__ faces, const float* __restrict__ v, int32_t T, int32_t s, int64_t first, int64_t n,
    const float* __restrict__ albedo, const float* __restrict__ rough, const float* __restrict__ normal,
    const uint8_t* __restrict__ probed, uint32_t* __restrict__ base, uint32_t* __restrict__ mr,
    uint32_t* __restrict__ nmap) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const AtTexel tx = at_texel(first + i, T, s);
    int32_t c[3];
    at_corners(faces, tx.face, c);
    const AtFrame fr = at_frame(v, c, tx.face & 1);
    const float a[3] = {albedo[i * 3], albedo[i * 3 + 1], albedo[i * 3 + 2]};
    const float nr[3] = {normal[i * 3], normal[i * 3 + 1], normal[i * 3 + 2]};
    uint32_t w[3];
    at_encode(fr, a, rough[i], nr, probed[i] != 0, w);
    const int64_t px = (int64_t)tx.y * T + tx.x;
    base[px] = w[0];
    mr[px] = w[1];
    nmap[px] = w[2];
  }
}

__global__ void __launch_bounds__(kThreads) atlas_corners_kernel(const int32_t* __restrict__ faces,
                                                                 const float* __restrict__ v, int64_t F, int32_t T,
                                                                 int32_t s, float* __restrict__ position,
                                                                 float* __restrict__ normal,
                                                                 float* __restrict__ tangent,
                                                                 float* __restrict__ texcoord) {
  for (int64_t f = (int64_t)blockIdx.x * kThreads + threadIdx.x; f < F; f += (int64_t)gridDim.x * kThreads) {
    int32_t c[3];
    at_corners(faces, f, c);
    const AtFrame fr = at_frame(v, c, f & 1);
    float uv[3][2];
    at_corner_uv(f, T, s, uv);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int64_t r = f * 3 + k;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        position[r * 3 + d] = v[(int64_t)c[k] * 3 + d];
        normal[r * 3 + d] = fr.n[d];
        tangent[r * 4 + d] = fr.t[d];
      }
      tangent[r * 4 + 3] = fr.w;
      texcoord[r * 2] = uv[k][0];
      texcoord[r * 2 + 1] = uv[k][1];
    }
  }
}

}  // namespace

extern "C" int tir_atlas_texels(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s,
                                int64_t first, int64_t n, int32_t* pix, float* pos, void* stream) {
  const int rc = at_texels_check(faces, n_faces, v, T, s, first, n, pix, pos);
  if (rc <= 0) return rc;
  atlas_texels_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(faces, v, T, s, first, n, pix, pos);
  return (int)cudaGetLastError();
}

extern "C" int tir_atlas_encode(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s,
                                int64_t first, int64_t n, const float* albedo, const float* rough,
                                const float* normal, const uint8_t* probed, uint8_t* base_color,
                                uint8_t* metallic_roughness, uint8_t* normal_map, void* stream) {
  const int rc = at_encode_check(faces, n_faces, v, T, s, first, n, albedo, rough, normal, probed, base_color,
                                 metallic_roughness, normal_map);
  if (rc <= 0) return rc;
  atlas_encode_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(
      faces, v, T, s, first, n, albedo, rough, normal, probed, (uint32_t*)base_color, (uint32_t*)metallic_roughness,
      (uint32_t*)normal_map);
  return (int)cudaGetLastError();
}

extern "C" int tir_atlas_corners(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s,
                                 float* position, float* normal, float* tangent, float* texcoord, void* stream) {
  const int rc = at_corners_check(faces, n_faces, v, T, s, position, normal, tangent, texcoord);
  if (rc <= 0) return rc;
  atlas_corners_kernel<<<grid_for(n_faces), kThreads, 0, (cudaStream_t)stream>>>(faces, v, n_faces, T, s, position,
                                                                                  normal, tangent, texcoord);
  return (int)cudaGetLastError();
}
