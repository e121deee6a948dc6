// Layout shadows + point-wise field queries.
#include "tir_device.cuh"

using namespace tir;

extern "C" int tir_abi_version(void) { return TIR_ABI_VERSION; }

// [C][H*W] -> [H*W][C] through a padded shared tile so both sides are coalesced.
__global__ void pack_channels_last_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int HW) {
  __shared__ float tile[32][33];
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int c = c0 + r, p = p0 + threadIdx.x;
    tile[r][threadIdx.x] = (c < C && p < HW) ? in[(size_t)c * HW + p] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int p = p0 + r, c = c0 + threadIdx.x;
    if (p < HW && c < C) out[(size_t)p * C + c] = tile[threadIdx.x][r];
  }
}

__global__ void unpack_channels_last_add_kernel(const float* __restrict__ cl, float* __restrict__ nchw, int C, int HW) {
  __shared__ float tile[32][33];
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int p = p0 + r, c = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (p < HW && c < C) ? cl[(size_t)p * C + c] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int c = c0 + r, p = p0 + threadIdx.x;
    if (c < C && p < HW) nchw[(size_t)c * HW + p] += tile[threadIdx.x][r];
  }
}

extern "C" int tir_pack_channels_last(const float* nchw, float* out, int32_t C, int32_t H, int32_t W, void* stream) {
  if (!nchw || !out) return TIR_ERR_NULL;
  if (C <= 0 || H <= 0 || W <= 0) return TIR_ERR_SHAPE;
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, (C + 31) / 32), block(32, 8);
  pack_channels_last_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(nchw, out, C, HW);
  return (int)cudaGetLastError();
}

extern "C" int tir_unpack_channels_last_add(const float* cl, float* nchw, int32_t C, int32_t H, int32_t W, void* stream) {
  if (!nchw || !cl) return TIR_ERR_NULL;
  if (C <= 0 || H <= 0 || W <= 0) return TIR_ERR_SHAPE;
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, (C + 31) / 32), block(32, 8);
  unpack_channels_last_add_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(cl, nchw, C, HW);
  return (int)cudaGetLastError();
}

__global__ void pack_alpha_kernel(const float* __restrict__ vol, uint8_t* __restrict__ corners,
                                  uint8_t* __restrict__ cells, int X, int Y, int Z, int pass) {
  size_t n = (size_t)X * Y * Z;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (pass == 0) {
      corners[i] = vol[i] > 0.f ? 1 : 0;
    } else {
      int x = (int)(i % X), y = (int)((i / X) % Y), z = (int)(i / ((size_t)X * Y));
      uint8_t any = 0;
      for (int dz = 0; dz < 2; ++dz)
        for (int dy = 0; dy < 2; ++dy)
          for (int dx = 0; dx < 2; ++dx) {
            int xx = x + dx, yy = y + dy, zz = z + dz;
            if (xx < X && yy < Y && zz < Z) any |= corners[((size_t)zz * Y + yy) * X + xx];
          }
      cells[i] = any;
    }
  }
}

extern "C" int tir_pack_alpha_mask(const float* volume, uint8_t* corners, uint8_t* cells,
                                   int32_t X, int32_t Y, int32_t Z, void* stream) {
  if (!volume || !corners || !cells) return TIR_ERR_NULL;
  if (X <= 0 || Y <= 0 || Z <= 0) return TIR_ERR_SHAPE;
  size_t n = (size_t)X * Y * Z;
  int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  pack_alpha_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(volume, corners, cells, X, Y, Z, 0);
  pack_alpha_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(volume, corners, cells, X, Y, Z, 1);
  return (int)cudaGetLastError();
}

template <int C>
__global__ void density_points_kernel(TirField f, const float* __restrict__ xn, int64_t n,
                                      float* __restrict__ feature, float* __restrict__ sigma) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float ft = density_feature<C>(f, xn[i * 3 + 0], xn[i * 3 + 1], xn[i * 3 + 2]);
    if (feature) feature[i] = ft;
    if (sigma) sigma[i] = feature_to_sigma(f, ft);
  }
}

extern "C" int tir_density_points(const TirField* field, const float* xn, int64_t n, float* feature, float* sigma,
                                  void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xn) return TIR_ERR_NULL;
  const int64_t cap = (int64_t)num_sms() * 16;
  int blocks = (int)((n + 127) / 128 < cap ? (n + 127) / 128 : cap);
  if (field->dC == 16)
    density_points_kernel<16><<<blocks, 128, 0, (cudaStream_t)stream>>>(*field, xn, n, feature, sigma);
  else if (field->dC == 8)
    density_points_kernel<8><<<blocks, 128, 0, (cudaStream_t)stream>>>(*field, xn, n, feature, sigma);
  else
    return TIR_ERR_SHAPE;
  return (int)cudaGetLastError();
}

__global__ void alpha_points_kernel(TirField f, const float* __restrict__ xyz, int64_t n, uint8_t* __restrict__ mask) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    mask[i] = alpha_mask_positive(f, xyz[i * 3 + 0], xyz[i * 3 + 1], xyz[i * 3 + 2]) ? 1 : 0;
}

extern "C" int tir_alpha_mask_points(const TirField* field, const float* xyz, int64_t n, uint8_t* mask, void* stream) {
  if (n <= 0) return TIR_OK;   // empty input: nothing to do (pointers of empty tensors are NULL)
  if (!field || !xyz || !mask || !field->amask || !field->acell) return TIR_ERR_NULL;
  const int64_t cap = (int64_t)num_sms() * 8;
  int blocks = (int)((n + 255) / 256 < cap ? (n + 255) / 256 : cap);
  alpha_points_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(*field, xyz, n, mask);
  return (int)cudaGetLastError();
}

// ---- on-the-fly ray generation (SURVEY.md 8 f4): rays of (view, pixel) ids instead of fancy-indexing a precomputed
// [n_views*H*W, 6] table on the host (train_tensoIR.py:239-242; get_ray_directions + normalise + get_rays,
// dataLoader/ray_utils.py:25-43, :67-88, tensoIR_rotation_setting.py:103-114).
namespace {
__global__ void generate_rays_kernel(const float* __restrict__ c2w /* [n_views,4,4] row-major */,
                                     const int32_t* __restrict__ view, const int32_t* __restrict__ pix, int64_t n,
                                     int32_t H, int32_t W, float focal, float* __restrict__ rays) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float* M = c2w + (size_t)view[t] * 16;
  const int p = pix[t];
  const float i = (float)(p % W) + 0.5f, j = (float)(p / W) + 0.5f;
  float dx = __fdiv_rn(__fsub_rn(i, 0.5f * (float)W), focal), dy = __fdiv_rn(__fsub_rn(j, 0.5f * (float)H), focal), dz = 1.f;
  const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), 1.f));
  dx = __fdiv_rn(dx, nrm); dy = __fdiv_rn(dy, nrm); dz = __fdiv_rn(dz, nrm);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    rays[t * 6 + r] = M[r * 4 + 3];                                                    // origin = c2w[:3, 3]
    rays[t * 6 + 3 + r] = fmaf(dz, M[r * 4 + 2], fmaf(dy, M[r * 4 + 1], __fmul_rn(dx, M[r * 4 + 0])));   // d @ R^T
  }
}
}  // namespace

extern "C" int tir_generate_rays(const float* c2w, const int32_t* view_idx, const int32_t* pix_idx, int64_t n, int32_t H,
                                 int32_t W, float focal, float* rays, void* stream) {
  if (n <= 0) return TIR_OK;
  if (!c2w || !view_idx || !pix_idx || !rays) return TIR_ERR_NULL;
  if (H <= 0 || W <= 0 || !(focal > 0.f)) return TIR_ERR_CONFIG;
  generate_rays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(c2w, view_idx, pix_idx, n, H, W,
                                                                                      focal, rays);
  return (int)cudaGetLastError();
}
