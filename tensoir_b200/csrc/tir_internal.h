// Internal (non-ABI) interfaces between the translation units of libtensoir_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"

namespace tir {

// One appearance head evaluated on a list of points (the training / eval forward of the primary march).
struct HeadJobDev {
  TirMlp mlp;
  const float* xn;            // [n,3] normalised sample points
  const float* x_in;          // [n,3] 3-vector fed to the MLP, or (x_index != NULL) a table indexed by x_index
  const int32_t* x_index;     // [n] row of x_in / light_idx per sample (the sample's ray), or NULL (= row i)
  int32_t x_in_stride;        // floats between rows of x_in (3, or 6 when it points into a [n_rays,6] ray table)
  const int32_t* light_idx;   // light index per row of the x_index space (or per sample), NULL -> row 0
  int32_t light_mode;         // 0 none, 1 indexed row of mlp.light_line, 2 mean over the mlp.n_lights rows
  int32_t act;                // 0 sigmoid, 1 tanh
  float* out;                 // [n, out_stride]
  int32_t out_stride;
  float* save_x0;             // [n,144] raw plane*line products (before the light factor), or NULL
  float* save_in;             // [n,150] MLP input incl. positional encodings, or NULL
  float* save_h1;             // [n,128] post-ReLU
  float* save_h2;             // [n,128] post-ReLU
};

constexpr int kMaxHeadJobs = 4;

// Forward of up to 4 heads in ONE launch (CTAs are partitioned over the jobs).  n = rows allocated, n_dev = optional
// device pointer to the real row count (<= n).
int launch_heads_forward(const TirField& f, const HeadJobDev* jobs, int n_jobs, int64_t n, const int64_t* n_dev,
                         cudaStream_t stream);

// Backward of the same heads on the dumps of launch_heads_forward (csrc/tir_mlp_bwd.cu).
struct HeadBwdJob {
  TirMlp mlp;                 // weights (forward values)
  const int32_t* x_index;     // as in the forward (light index lookup)
  const int32_t* light_idx;
  int32_t light_mode;
  int32_t act;
  int32_t point_set;          // which x0 buffer / gx0 accumulator this head belongs to (0 or 1)
  const float* out;           // [n, out_stride] forward output
  int32_t out_stride;
  const float* g_out;         // [n, out_stride] gradient w.r.t. the output
  const float* inp;           // dumps of the forward
  const float* h1;
  const float* h2;
  float* gz1;                 // [n,128] scratch: gradient at the first hidden pre-activation
  float* gz2;                 // [n,128] scratch: gradient at the second hidden pre-activation
  float* gfeat;               // [n,32]  scratch: gradient w.r.t. the 27 basis features (row stride 32)
  float* gx0;                 // [n,144] gradient w.r.t. the raw products of this head's point set (overwritten)
  // parameter gradients, ACCUMULATED (+=): PyTorch layouts
  float* g_w0; float* g_b0; float* g_w1; float* g_b1; float* g_w2; float* g_b2;
};

struct HeadsBwdShared {
  const float* x0[2];         // raw products per point set [n,144]
  float* g_basis;             // [27,144] accumulated over all heads
  float* g_light;             // [L,144] accumulated
};

int launch_heads_backward(const TirField& f, const HeadBwdJob* jobs, int n_jobs, const HeadsBwdShared& sh, int64_t n,
                          const int64_t* n_dev, cudaStream_t stream);

// channel-last gradient buffers of the VM factors (same layout as the field's planes / lines), accumulated with atomics
struct GradPtrs {
  float* plane[3];
  float* line[3];
};

// valid-sample list passes over an interleaved [n_rays,6] ray table (origin | direction)
int launch_valid_samples(const TirField& f, const TirMarchCfg& cfg, const float* rays, int64_t n_rays, bool fill,
                         int32_t* counts, const int64_t* offsets, int32_t* out_ray, int32_t* out_sample, float* out_xn,
                         float* out_z, float* out_dist, uint64_t* counters, int64_t capacity, cudaStream_t stream);
int launch_density_bwd(const TirField& f, const float* xn, int64_t n, const int64_t* n_dev, const float* g_feature,
                       const GradPtrs& g, cudaStream_t stream);
// One scatter of an appearance-list point set into the VM-factor gradients: the appearance products' backward (g[0] +
// g[1] + g[2] when not NULL: heads evaluated at the same points share one scatter) or, with density_grad, the
// backward of the density feature and its spatial gradient (g[0] = d L / d feature, g[1] = d L / d (d f / d x_hat),
// either NULL for zero).  The jobs of one launch write disjoint gradients.
constexpr int kMaxAppScatterJobs = 3;
struct AppScatterJob {
  int density_grad;
  const float* xn;
  const float* g[3];
  GradPtrs out;
  int ctas;                   // set by launch_app_scatter
};
// all jobs over the same list length (n rows, min(*n_dev, n) when n_dev is given), CTAs split in proportion to work
int launch_app_scatter(const TirField& f, AppScatterJob* jobs, int n_jobs, int64_t n, const int64_t* n_dev,
                       cudaStream_t stream);
int launch_density_grad(const TirField& f, const float* xn, int64_t n, const int64_t* n_dev, float* feature,
                        float* dfdx, cudaStream_t stream);

// real row count of a list: min(*n_dev, n) when a device count is given
__device__ __forceinline__ int64_t list_rows(int64_t n, const int64_t* n_dev) {
  if (!n_dev) return n;
  const int64_t r = *n_dev;
  return r < n ? r : n;
}

}  // namespace tir
