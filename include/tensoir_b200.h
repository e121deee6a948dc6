/* tensoir_b200 — C ABI of the H100-native (sm_90a) TensoIR volume-rendering hot path.
 *
 * The reference (Haian-Jin/TensoIR) is 100 % Python/PyTorch and has no FFI of its own
 * (SURVEY.md §8b); this ABI is what the Python shim in tensoir_b200/ binds with ctypes, and
 * what a maintainer of the reference would bind from models/relight_utils.py and
 * models/tensorBase_*.py (stubs in INTEGRATION.md).  Each entry point cites the reference
 * function(s) it replaces (paths relative to the reference root).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller (PyTorch); nothing is allocated,
 *    freed or retained by the library; scratch buffers are passed in;
 *  - all arithmetic is fp32, indices int32, counters uint64;
 *  - `stream` is a cudaStream_t passed as void*; every call is asynchronous on it;
 *  - return value: 0 = ok, <0 = TirStatus argument error, >0 = cudaError_t passthrough;
 *  - no global state, re-entrant, never throws.
 */
#ifndef TENSOIR_B200_H
#define TENSOIR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TIR_ABI_VERSION 3

typedef enum TirStatus {
  TIR_OK = 0,
  TIR_ERR_NULL = -1,      /* required pointer is NULL */
  TIR_ERR_SHAPE = -2,     /* unsupported channel count / size */
  TIR_ERR_CONFIG = -3,    /* bad enum / config value */
  TIR_ERR_CAPACITY = -4   /* scratch buffer too small */
} TirStatus;

/* counters[] slots (uint64, accumulated with atomics; caller zeroes them) — parity and the
 * roofline are both defined on these (SURVEY.md §8d) */
enum {
  TIR_CNT_MASK = 0,      /* in-bbox samples looked up in the alpha mask      (32 B each)   */
  TIR_CNT_DENSITY = 1,   /* valid density samples                            (1152 B each) */
  TIR_CNT_APP = 2,       /* appearance samples, weight > thres               (3456 B each) */
  TIR_CNT_RAYS = 3,      /* rays marched (secondary: after the cosine test)               */
  TIR_CNT_OVERFLOW = 4,  /* app samples dropped because the sample list was full (must be 0) */
  TIR_CNT_SLOTS = 8
};

/* The VM field as the kernels see it: channel-last fp32 shadows of the reference's
 * parameters (models/tensoRF_rotated_lights.py:11-29).
 *   plane k  [G[m1]][G[m0]][C]  from density_plane[k] / app_plane[k]  ([1,C,G[m1],G[m0]])
 *   line  k  [G[v]][C]          from density_line[k]  / app_line[k]   ([1,C,G[v],1])
 * with matMode = {{0,1},{0,2},{1,2}}, vecMode = {2,1,0} (models/tensorBase_rotated_lights.py:398-399). */
typedef struct TirField {
  const float* dplane[3];
  const float* dline[3];
  const float* aplane[3];
  const float* aline[3];
  int32_t dC;              /* density channels per orientation (16)  — multiple of 4 */
  int32_t aC;              /* appearance channels per orientation (48) — multiple of 4 */
  int32_t grid[3];         /* gridSize x,y,z */
  float aabb_lo[3];
  float aabb_hi[3];
  float inv_aabb[3];       /* 2/(hi-lo) exactly as the host computed it (tensorBase:612) */
  /* alpha mask (AlphaGridMask, models/tensorBase_rotated_lights.py:100-119); amask == NULL => none */
  const uint8_t* amask;    /* [Z][Y][X] 0/1 corner occupancy */
  const uint8_t* acell;    /* [Z][Y][X] OR of the 8 corners of cell (x,y,z) (built by tir_pack_alpha_mask) */
  int32_t agrid[3];        /* X,Y,Z */
  float a_lo[3];
  float a_inv[3];          /* 1/(hi-lo)*2 as AlphaGridMask.invgridSize */
  /* world-space bounding box of the alpha-mask CELLS that have a set corner (grown by a guard band): a sample outside it
   * lies in cells whose 8 corners are all 0, so AlphaGridMask.sample_alpha is exactly 0 there and the marches skip the
   * lookup (empty-space skipping that cannot change which samples are valid).  occ_lo > occ_hi: no box (test disabled). */
  float occ_lo[3];
  float occ_hi[3];
  float density_shift;     /* -10 */
  float distance_scale;    /* 25 */
  float weight_thres;      /* rayMarch_weight_thres 1e-4 */
  int32_t softplus;        /* 1 = softplus(f+shift), 0 = relu(f) (tensorBase:813-817) */
} TirField;

/* A 3-layer MLP head (MLPRender_Fea / MLPBRDF_PEandFeature, tensorBase:122-146,:182-208) plus
 * the shared basis_mat / light_line of TensorVMSplit.  Weights in PyTorch [out,in] row-major. */
typedef struct TirMlp {
  const float* w0; const float* b0;   /* [H, in_dim], [H]  in_dim = 2*pe_x*3 + 2*pe_f*F + 3 + F */
  const float* w1; const float* b1;   /* [H, H], [H] */
  const float* w2; const float* b2;   /* [out, H], [out] */
  const float* basis;                 /* basis_mat.weight [F, 3*aC] */
  const float* light_line;            /* light_line.weight [L, 3*aC]; NULL => no light factor (tensoRF_init) */
  int32_t n_lights;
  int32_t feat_dim;                   /* F = app_dim (27) */
  int32_t hidden;                     /* featureC (128) */
  int32_t out_dim;                    /* 3 or 4 */
  int32_t pe_feat;                    /* fea_pe (2) */
  int32_t pe_x;                       /* view_pe / pos_pe (2) */
} TirMlp;

typedef enum TirSampling {
  TIR_SAMPLE_STEP = 0,   /* TensorBase.sample_ray (tensorBase:705-724): z = t_min + step*(i + jitter) */
  TIR_SAMPLE_TABLE = 1   /* sample_ray_equally (relight_utils.py:707-722): z = z_table[i], same for all rays */
} TirSampling;

typedef struct TirMarchCfg {
  int32_t sampling;        /* TirSampling */
  int32_t n_samples;
  float step;              /* stepSize (STEP) */
  float near;              /* near_far[0] (STEP: clamp of t_min) */
  float far;
  const float* z_table;    /* [n_samples] (TABLE), computed by the host exactly like the reference */
  const float* jitter;     /* [n_rays] per-ray jitter or NULL (STEP; the reference draws it on the CPU, tensorBase:717) */
  int32_t flags;           /* TIR_MARCH_NO_BBOX: skip the in-aabb test (filtering_rays samples the alpha mask for every
                              point, tensorBase:803-804) */
} TirMarchCfg;

enum {
  TIR_MARCH_NO_BBOX = 1,
  /* Production mode of the marches: work whose only effect would be on TIR_CNT_MASK / TIR_CNT_DENSITY is skipped (the
   * rest of a ray whose transmittance has underflowed to exactly 0), so those two slots count the queries actually made
   * instead of the queries the reference makes.  All outputs, the appearance list and the other counters are unchanged. */
  TIR_MARCH_LEAN_COUNTERS = 2
};

/* One compacted appearance sample produced by the march (w > weight_thres), consumed by tir_app_mlp. */
typedef struct TirAppSample {
  float xn[3];             /* normalised coords in [-1,1] */
  float weight;
  int32_t ray;
  int32_t sample;          /* index along the ray */
} TirAppSample;

int tir_abi_version(void);

/* NCHW [1,C,H,W] parameter -> channel-last [H][W][C] shadow. Replaces nothing in the reference:
 * it is the layout change that makes one bilinear tap one contiguous 4*C-byte read. */
int tir_pack_channels_last(const float* nchw, float* out, int32_t C, int32_t H, int32_t W, void* stream);
/* inverse scatter of a channel-last gradient back to NCHW (accumulating: nchw += cl) */
int tir_unpack_channels_last_add(const float* cl, float* nchw, int32_t C, int32_t H, int32_t W, void* stream);

/* float alpha_volume [Z,Y,X] (0/1) -> corner bytes + per-cell OR bytes (AlphaGridMask, tensorBase:100-119). */
int tir_pack_alpha_mask(const float* volume, uint8_t* corners, uint8_t* cells,
                        int32_t X, int32_t Y, int32_t Z, void* stream);

/* compute_densityfeature + feature2density on normalised points
 * (models/tensoRF_rotated_lights.py:95-110, tensorBase:813-817): xn [n,3] -> feature [n], sigma [n]
 * (either output may be NULL). */
int tir_density_points(const TirField* field, const float* xn, int64_t n, float* feature, float* sigma, void* stream);

/* AlphaGridMask.sample_alpha(xyz) > 0 on world-space points (tensorBase:112-116): xyz [n,3] -> mask [n] (0/1). */
int tir_alpha_mask_points(const TirField* field, const float* xyz, int64_t n, uint8_t* mask, void* stream);

/* Density-only march: sample_ray / sample_ray_equally + alpha-mask filter + compute_densityfeature +
 * feature2density + raw2alpha + compositing.  Replaces compute_transmittance
 * (models/relight_utils.py:657-705) and the density half of TensorBase.forward (tensorBase:885-921,:974-975).
 *   rays_o, rays_d [n_rays,3];  t_last [n_rays] (= nerv_vis), acc [n_rays] (nerfactor_vis = 1-acc),
 *   depth [n_rays] (sum w*z) — any output may be NULL. */
int tir_march_density(const TirField* field, const float* rays_o, const float* rays_d, int64_t n_rays,
                      const TirMarchCfg* cfg, float* t_last, float* acc, float* depth,
                      uint64_t* counters, void* stream);

/* Full radiance march over explicit rays: compute_radiance (models/relight_utils.py:777-834) and, with
 * TIR_SAMPLE_STEP, the rgb half of TensorBase_Init.forward (models/tensorBase_init.py:406-462).
 *   light_idx [n_rays] int32 or NULL; view direction fed to the MLP = rays_d.
 *   samples: scratch list [capacity] of TirAppSample; sample_count: device uint32 (caller zeroes).
 *   rgb [n_rays,3] must be zeroed by the caller (accumulated with atomics). */
int tir_march_radiance(const TirField* field, const TirMlp* mlp, const float* rays_o, const float* rays_d,
                       const int32_t* light_idx, int64_t n_rays, const TirMarchCfg* cfg,
                       float* t_last, float* acc, float* depth, float* rgb,
                       TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                       uint64_t* counters, void* stream);

/* Secondary shading of render_with_BRDF (models/relight_utils.py:428-450): for every surface point p and
 * every incident direction d with clamp(d.n,0) > 1e-6, march compute_radiance along (p, d).
 * Rays are generated on chip (no [bs,n_dirs,3] tensors).
 *   surf_xyz, normals [n_pts,3]; light_idx [n_pts]; dirs [n_dirs,3]
 *   vis [n_pts,n_dirs] (T_last, 0 where masked), indirect [n_pts,n_dirs,3] (caller zeroes both). */
int tir_secondary_radiance(const TirField* field, const TirMlp* mlp, const float* surf_xyz, const float* normals,
                           const int32_t* light_idx, int64_t n_pts, const float* dirs, int32_t n_dirs,
                           const TirMarchCfg* cfg, float* vis, float* indirect,
                           TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                           uint64_t* counters, void* stream);

/* First half of tir_secondary_radiance only (cosine test + density march + app-sample compaction); the second half is
 * tir_app_mlp on the same list.  Exposed so the two kernels can be timed / profiled separately. */
int tir_secondary_march(const TirField* field, const float* surf_xyz, const float* normals, int64_t n_pts,
                        const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg, float* vis,
                        TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                        uint64_t* counters, void* stream);

/* Appearance gather + basis_mat + MLPRender_Fea on a compacted sample list
 * (compute_appfeature tensoRF_rotated_lights.py:197-224 + MLPRender_Fea tensorBase:136-146):
 *   rgb_out[ray] += weight * sigmoid(mlp(...)) for every sample; dirs_of_ray gives the view dir.
 *   ray_dirs [n_rays,3] when dir_stride_rays = 1, or the [n_dirs,3] table with ray % n_dirs indexing
 *   when n_dirs > 0.  light_idx indexed by ray (n_dirs == 0) or by ray / n_dirs. */
int tir_app_mlp(const TirField* field, const TirMlp* mlp, const TirAppSample* samples,
                const uint32_t* sample_count, int64_t max_samples, const float* ray_dirs, int32_t n_dirs,
                const int32_t* light_idx, float* rgb_out, void* stream);

/* The two implementations behind tir_app_mlp (which dispatches to _wgmma unless the environment has TIR_MLP_LEGACY=1):
 *   _wgmma   sm_90a-native: wgmma.mma_async with the A operand and the accumulator in registers, weights resident
 *            in shared memory, two warpgroups per CTA on different 64-sample tiles (csrc/tir_mlp_wgmma.cu)
 *   _legacy  round 1: mma.sync.m16n8k16 on 64-sample tiles (csrc/tir_mlp.cu)
 * Same arguments and results (both use the error-compensated split-BF16 product with fp32 accumulation). */
int tir_app_mlp_wgmma(const TirField* field, const TirMlp* mlp, const TirAppSample* samples,
                      const uint32_t* sample_count, int64_t max_samples, const float* ray_dirs, int32_t n_dirs,
                      const int32_t* light_idx, float* rgb_out, void* stream);
int tir_app_mlp_legacy(const TirField* field, const TirMlp* mlp, const TirAppSample* samples,
                       const uint32_t* sample_count, int64_t max_samples, const float* ray_dirs, int32_t n_dirs,
                       const int32_t* light_idx, float* rgb_out, void* stream);
int tir_app_mlp_points_wgmma(const TirField* field, const TirMlp* mlp, const float* xn, const float* x_in,
                             const int32_t* light_idx, int64_t n, int32_t act, float* out, void* stream);
int tir_app_mlp_points_legacy(const TirField* field, const TirMlp* mlp, const float* xn, const float* x_in,
                              const int32_t* light_idx, int64_t n, int32_t act, float* out, void* stream);

/* Same gather+MLP on explicit points (no compositing): xn [n,3] normalised coords, x_in [n,3] the 3-vector fed
 * to the MLP next to the features (view dir for MLPRender_Fea, position for MLPBRDF_PEandFeature),
 * light_idx [n] or NULL (row 0 of mlp->light_line, e.g. the mean-light row of compute_intrinfeature),
 * act 0 = sigmoid, 1 = tanh -> out [n,out_dim].  Mirrors renderModule*(compute_*feature(...)). */
int tir_app_mlp_points(const TirField* field, const TirMlp* mlp, const float* xn, const float* x_in,
                       const int32_t* light_idx, int64_t n, int32_t act, float* out, void* stream);

/* tir_app_mlp_points that also dumps the activations a host-side backward needs (training forward of the primary
 * MLP heads): save_xl [n, 3*aC] light-scaled products, save_in [n, in_dim] MLP input incl. positional encoding,
 * save_h1 / save_h2 [n, hidden] post-ReLU hidden layers; any of them may be NULL. */
int tir_app_mlp_points_save(const TirField* field, const TirMlp* mlp, const float* xn, const float* x_in,
                            const int32_t* light_idx, int64_t n, int32_t act, float* out, float* save_xl,
                            float* save_in, float* save_h1, float* save_h2, void* stream);

/* Shading epilogue of render_with_BRDF (models/relight_utils.py:452-475) with GGX_specular (:17-50):
 *   rgb[i] = sum_l (albedo_i/pi + GGX_il) * (vis_il * direct[light_i][l] + indirect_il) * clamp(dir_l . n_i, 0) * weight_l
 * normal/albedo/rough/fresnel/view [bs,3], light_idx [bs], dirs [n_dirs,3], weight [n_dirs] (solid angles),
 * direct [n_lights,n_dirs,3] (SG environment light), vis [bs,n_dirs], indirect [bs,n_dirs,3] -> rgb [bs,3] (linear). */
int tir_shade_fwd(const float* normal, const float* albedo, const float* rough, const float* fresnel,
                  const float* view, const int32_t* light_idx, int64_t bs, const float* dirs, const float* weight,
                  int32_t n_dirs, const float* direct, int32_t n_lights, const float* vis, const float* indirect,
                  float* rgb, void* stream);
/* analytic backward: g_rgb [bs,3] -> g_normal, g_albedo, g_rough, g_fresnel [bs,3] (overwritten) and g_direct
 * [n_lights,n_dirs,3] (accumulated, caller zeroes). */
int tir_shade_bwd(const float* normal, const float* albedo, const float* rough, const float* fresnel,
                  const float* view, const int32_t* light_idx, int64_t bs, const float* dirs, const float* weight,
                  int32_t n_dirs, const float* direct, int32_t n_lights, const float* vis, const float* indirect,
                  const float* g_rgb, float* g_normal, float* g_albedo, float* g_rough, float* g_fresnel,
                  float* g_direct, void* stream);

/* The same quadrature over a WHOLE ray batch masked by acc_mask (renderer.py:99-106): rows with mask == 0 shade to the
 * constant 1 (white) and contribute no gradient; rows with mask != 0 are shaded, clipped to [0,1] and (srgb != 0)
 * converted with linear2srgb_torch (relight_utils.py:476-481, :489-515) inside the kernel.  The surface hits are never
 * compacted into a list: tir_hits_prepare builds the surface points (rays_o + depth * rays_d, relight_utils.py:412) and
 * zeroes the normals of non-hit rays, which makes tir_secondary_radiance skip all of their directions.
 *   rays [n,6], mask [n] (0/1), normal/albedo/fresnel [n,3], rough1 [n,1], view direction = -rays_d;
 *   lin [n,3] = linear value before clip / sRGB (written by the forward, read by the backward). */
int tir_hits_prepare(const float* rays, const float* depth, const float* normal, const uint8_t* mask, int64_t n,
                     float* surf_xyz, float* normal_masked, void* stream);
int tir_shade_hits_fwd(const float* rays, const uint8_t* mask, const float* normal, const float* albedo,
                       const float* rough1, const float* fresnel, const int32_t* light_idx, int64_t n,
                       const float* dirs, const float* weight, int32_t n_dirs, const float* direct, int32_t n_lights,
                       const float* vis, const float* indirect, int32_t srgb, float* rgb, float* lin, void* stream);
int tir_shade_hits_bwd(const float* rays, const uint8_t* mask, const float* normal, const float* albedo,
                       const float* rough1, const float* fresnel, const int32_t* light_idx, int64_t n,
                       const float* dirs, const float* weight, int32_t n_dirs, const float* direct, int32_t n_lights,
                       const float* vis, const float* indirect, int32_t srgb, const float* lin, const float* g_rgb,
                       float* g_normal, float* g_albedo, float* g_rough1, float* g_fresnel, float* g_direct,
                       void* stream);

/* ---- modular, autograd-facing half of the primary march (training needs gradients) --------------------- */

/* plane*line products of the appearance tensors on normalised points: xn [n,3] -> out [n, 3*aC]
 * (first half of compute_{app,both,intrin}feature, models/tensoRF_rotated_lights.py:141-153). */
int tir_vm_app_products(const TirField* field, const float* xn, int64_t n, float* out, void* stream);
/* backward of the above into channel-last gradient shadows g_plane[k] [H][W][aC], g_line[k] [D][aC] (accumulating;
 * replaces grid_sampler_2d_backward, SURVEY.md a20). */
int tir_vm_app_products_bwd(const TirField* field, const float* xn, int64_t n, const float* g_out,
                            float* const* g_plane, float* const* g_line, void* stream);
/* backward of tir_density_points' feature output (compute_densityfeature, tensoRF:95-110). */
int tir_vm_density_bwd(const TirField* field, const float* xn, int64_t n, const float* g_feature,
                       float* const* g_plane, float* const* g_line, void* stream);
/* density feature and its analytic spatial gradient d f / d x_hat [n,3] with the clamped-index sampler
 * (compute_densityfeature_with_xyz_grad tensoRF:113-129 + grid_sample relight_utils.py:57-107; feeds
 * compute_derived_normals tensorBase:839-856 without an autograd.grad round trip). */
int tir_vm_density_grad(const TirField* field, const float* xn, int64_t n, float* feature, float* dfdx, void* stream);
/* backward of both outputs (g_feature / g_dfdx may be NULL) — the reference's double backward. */
int tir_vm_density_grad_bwd(const TirField* field, const float* xn, int64_t n, const float* g_feature,
                            const float* g_dfdx, float* const* g_plane, float* const* g_line, void* stream);

/* sample_ray + in-bbox + alpha-mask filter (tensorBase:705-724, :892-897) as a ray-sorted list, two passes:
 * count -> (host cumsum) -> fill.  Row order equals the reference's xyz_sampled[ray_valid]. */
int tir_valid_samples_count(const TirField* field, const float* rays_o, const float* rays_d, int64_t n_rays,
                            const TirMarchCfg* cfg, int32_t* counts, uint64_t* counters, void* stream);
int tir_valid_samples_fill(const TirField* field, const float* rays_o, const float* rays_d, int64_t n_rays,
                           const TirMarchCfg* cfg, const int64_t* offsets, int32_t* out_ray, int32_t* out_sample,
                           float* out_xn, float* out_z, float* out_dist, int64_t capacity /* 0 = unbounded; rows past
                           it are dropped (static-capacity lists for CUDA-graph capture) */, void* stream);

/* raw2alpha (tensorBase:21-28) over ray segments of a valid-sample list, sequential like torch.cumprod:
 * weight[i] = alpha_i * T_i, trans[i] = T_i (exclusive), t_last[ray]. */
int tir_composite_fwd(const float* sigma, const float* dist, const int64_t* offsets, int64_t n_rays,
                      float distance_scale, float* weight, float* trans, float* t_last,
                      int64_t limit /* 0 = none; list rows >= limit are ignored */,
                      const float* z /* [n_valid] or NULL */, float* acc /* [n_rays] sum w, or NULL */,
                      float* depth /* [n_rays] sum w*z, or NULL */, void* stream);
int tir_composite_bwd(const float* sigma, const float* dist, const int64_t* offsets, int64_t n_rays,
                      float distance_scale, const float* weight, const float* trans, const float* g_weight,
                      float* g_sigma, int64_t limit, const float* z, const float* g_acc /* [n_rays] or NULL */,
                      const float* g_depth /* [n_rays] or NULL */, void* stream);

/* ---- fused end of the primary march (tensorBase_rotated_lights.py:930-1036) --------------------------------- */

/* Per appearance sample: BRDF split, relative-smoothness costs (:858-863), normals_diff / orientation terms (:952-961),
 * weighting and the per-ray sums torch.sum(weight[..., None] * x, -2) (:974-975) of 14 channels
 *   [rgb 3 | normal 3 | albedo 3 | roughness | albedo cost | roughness cost | normals_diff | orientation].
 * w [n], ray [n] int64 (ray of each sample), rgb / vn [n,3], brdf / brdfj [n,4] (BRDF head at x and at x + noise),
 * dn [n,3] derived normals or NULL (then the last two channels are 0), viewdirs [n_rays,3]
 * -> packed [n_rays,14], accumulated with atomics (caller zeroes). */
int tir_tail_fwd(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                 const float* brdfj, const float* vn, const float* dn, const float* viewdirs, float* packed,
                 void* stream);
/* analytic backward: g_packed [n_rays,14] -> per-sample gradients (g_dn may be NULL when dn is). */
int tir_tail_bwd(int64_t n, const float* w, const int64_t* ray, const float* rgb, const float* brdf,
                 const float* brdfj, const float* vn, const float* dn, const float* viewdirs, const float* g_packed,
                 float* g_w, float* g_rgb, float* g_brdf, float* g_brdfj, float* g_vn, float* g_dn, void* stream);

/* per-ray maps of the 12-tuple (or their gradients) */
typedef struct TirRayMaps {
  float* rgb;      /* [n,3] sRGB */
  float* depth;    /* [n]   */
  float* normal;   /* [n,3] unit */
  float* albedo;   /* [n,3] */
  float* rough;    /* [n]   */
  float* fresnel;  /* [n,3] */
  float* nd;       /* [n] normals_diff_map */
  float* no;       /* [n] normals_orientation_loss_map */
} TirRayMaps;

/* Per ray: background compositing with (1 - acc) when bg != 0 (:1004-1012), clamps, linear2srgb_torch
 * (relight_utils.py:489-515), safe_l2_normalize of the normal map, acc_mask = acc > 0.5, and the two scalar
 * smoothness losses mean(albedo cost), mean(roughness cost) accumulated into losses[2] (caller zeroes).
 * packed [n,14] from tir_tail_fwd, acc / depth [n] from tir_composite_fwd, rays [n,6]. */
int tir_epilogue_fwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                     float fresnel0, int32_t bg, const TirRayMaps* out, uint8_t* acc_mask, float* losses,
                     void* stream);
/* analytic backward; every pointer in g_out and the two scalar-loss gradients may be NULL. */
int tir_epilogue_bwd(int64_t n, const float* packed, const float* acc, const float* depth, const float* rays,
                     float fresnel0, int32_t bg, const TirRayMaps* g_out, const float* g_loss_albedo,
                     const float* g_loss_rough, float* g_packed, float* g_acc, float* g_depth, void* stream);

/* ---- fused primary march: TensorBase.forward (models/tensorBase_rotated_lights.py:868-1036) with is_relight=True as
 * three calls that chain every kernel of the path on the caller's stream, without host synchronisation:
 *   tir_primary_march     sample_ray + aabb / alpha-mask filter -> ray-sorted valid list -> compute_densityfeature ->
 *                         feature2density -> raw2alpha / acc / depth -> per-ray counts of the appearance samples
 *   tir_primary_heads     appearance list (weight > rayMarch_weight_thres) -> the appearance heads (radiance, BRDF,
 *                         BRDF at jittered points, predicted normal) -> derived normals -> per-sample costs and the 14
 *                         composited channels -> per-ray epilogue (background, clamps, sRGB, normalise, acc_mask)
 *   tir_primary_backward  the whole backward of both (SURVEY.md a20), gradients ACCUMULATED into caller-zeroed buffers
 * All lists live in caller-allocated scratch of static capacity; their real lengths stay on the device
 * (work->offsets[n_rays], work->a_offsets[n_rays]); rows that do not fit are dropped and flagged in work->status, so the
 * caller can size the lists exactly (count pass + host read between the calls) or statically (CUDA-graph capture). */
#define TIR_MAX_HEADS 4

typedef struct TirHeadJob {
  TirMlp mlp;                 /* light_line = the full [n_lights,3*aC] table (or NULL) */
  int32_t point_set;          /* 0: appearance samples, 1: the same samples jittered by 0.01*N(0,1) (tensorBase:937) */
  int32_t x_in;               /* 0: view direction of the sample's ray, 1: the (normalised) sample point itself */
  int32_t light_mode;         /* 0 none, 1 light_line[light_idx[ray]], 2 mean over the lights (compute_intrinfeature) */
  int32_t act;                /* 0 sigmoid, 1 tanh */
  int32_t role;               /* TIR_HEAD_RGB / _BRDF / _BRDF_JITTER / _NORMAL */
} TirHeadJob;
enum { TIR_HEAD_RGB = 0, TIR_HEAD_BRDF = 1, TIR_HEAD_BRDF_JITTER = 2, TIR_HEAD_NORMAL = 3 };
enum { TIR_NORMALS_DERIVED_PLUS_PREDICTED = 0, TIR_NORMALS_PREDICTED = 1, TIR_NORMALS_DERIVED = 2 };

typedef struct TirPrimaryWork {
  int64_t cap_valid, cap_app;
  /* per ray */
  int32_t* counts;            /* [n_rays] valid samples */
  int64_t* offsets;           /* [n_rays+1] exclusive scan; offsets[n_rays] = real length of the valid list */
  float* t_last; float* acc; float* depth;          /* [n_rays] */
  int32_t* a_counts; int64_t* a_offsets;            /* appearance samples per ray, scan */
  float* packed;              /* [n_rays,14] composited channels */
  /* valid list [cap_valid] */
  int32_t* v_ray; int32_t* v_sample; float* v_xn; float* v_z; float* v_dist;
  float* v_feat; float* v_sigma; float* v_weight; float* v_trans;
  /* appearance list [cap_app] */
  int64_t* a_src;             /* row of the valid list */
  int32_t* a_ray; float* a_w; float* a_xn; float* a_xj;
  const float* noise;         /* [cap_app,3] N(0,1) draws for the jittered points */
  float* x0[2];               /* raw plane*line products per point set [cap_app,3*aC] (NULL: not saved, no backward) */
  float* inp[TIR_MAX_HEADS]; float* h1[TIR_MAX_HEADS]; float* h2[TIR_MAX_HEADS];   /* activation dumps (or NULL) */
  float* out[TIR_MAX_HEADS];  /* [cap_app,4] head outputs */
  float* dn_feat; float* dn_dfdx;                   /* derived-normal inputs [cap_app], [cap_app,3] */
  int64_t* status;            /* [4]: real valid count, real appearance count, overflow flag (0/1), reserved */
} TirPrimaryWork;

typedef struct TirPrimaryBwdWork {
  float* g_packed; float* g_acc; float* g_depth;    /* [n_rays,14], [n_rays], [n_rays] */
  float* g_weight; float* g_feat;                   /* [cap_valid] */
  float* g_out[TIR_MAX_HEADS];                      /* [cap_app,4] */
  float* gz1[TIR_MAX_HEADS]; float* gz2[TIR_MAX_HEADS];   /* [cap_app,hidden] */
  float* gfeat[TIR_MAX_HEADS];                      /* [cap_app,32] */
  float* gx0[TIR_MAX_HEADS];                        /* [cap_app,3*aC] */
  float* g_dn_feat; float* g_dn_dfdx;               /* [cap_app], [cap_app,3] */
} TirPrimaryBwdWork;

typedef struct TirPrimaryGrads {      /* accumulated (+=); the caller zeroes them (they may be the .grad tensors) */
  float* dplane[3]; float* dline[3]; float* aplane[3]; float* aline[3];   /* channel-last, like TirField */
  float* basis; float* light_line;
  float* w0[TIR_MAX_HEADS]; float* b0[TIR_MAX_HEADS]; float* w1[TIR_MAX_HEADS]; float* b1[TIR_MAX_HEADS];
  float* w2[TIR_MAX_HEADS]; float* b2[TIR_MAX_HEADS];   /* per job; jobs of the same module share buffers */
} TirPrimaryGrads;

int tir_primary_march(const TirField* field, const float* rays /* [n_rays,6] origin | direction */, int64_t n_rays,
                      const TirMarchCfg* cfg, const TirPrimaryWork* work, uint64_t* counters, void* stream);
/* appearance list of the march (rows of the valid list with weight > rayMarch_weight_thres, in list order): fills
 * work->a_src / a_ray / a_w / a_xn; its real length is work->a_offsets[n_rays].  Separate so that the caller can draw the
 * jitter noise (work->noise) for exactly these rows before tir_primary_heads. */
int tir_primary_app_list(const TirField* field, int64_t n_rays, const TirPrimaryWork* work, void* stream);
int tir_primary_heads(const TirField* field, const TirHeadJob* jobs, int32_t n_jobs, int32_t normals_kind,
                      const float* rays, const int32_t* light_idx /* [n_rays] */, int64_t n_rays,
                      const TirPrimaryWork* work, float fresnel0, int32_t white_bg, const TirRayMaps* out,
                      uint8_t* acc_mask, float* losses /* [2] */, uint64_t* counters, void* stream);
int tir_primary_backward(const TirField* field, const TirHeadJob* jobs, int32_t n_jobs, int32_t normals_kind,
                         const float* rays, const int32_t* light_idx, int64_t n_rays, const TirPrimaryWork* work,
                         const TirPrimaryBwdWork* bwork, float fresnel0, int32_t white_bg,
                         const TirRayMaps* g_maps /* gradients of the maps, members may be NULL */,
                         const float* g_acc_map /* [n_rays] or NULL */, const float* g_loss_albedo,
                         const float* g_loss_rough, const TirPrimaryGrads* grads, void* stream);

/* ---- optimiser pass (SURVEY.md 8 f3): torch.optim.Adam's update for a list of dense fp32 tensors in ONE launch, with
 * the L1 regulariser's gradient (l1 * sign(param), density_L1 of tensoRF_rotated_lights.py:74-78) folded in, the
 * gradient cleared for the next accumulation, and a device-side skip flag (found_inf != 0: parameters, moments and the
 * step counter stay untouched, gradients are still cleared).  table / chunk_prefix / state live in device memory:
 * chunk_prefix[k] = first chunk (of tir_adam_chunk_elems() elements) of tensor k, state = {step, 1-beta1^t,
 * sqrt(1-beta2^t), skipped}. */
typedef struct TirAdamTensor {
  float* p; float* g; float* m; float* v;   /* parameter, gradient, exp_avg, exp_avg_sq: same dense layout, n elements */
  int64_t n;
  const float* lr_dev;                      /* learning rate in device memory (CUDA-graph replay), or NULL -> lr */
  float lr;
  float l1;                                 /* coefficient of sign(param) added to the gradient (0: none) */
} TirAdamTensor;
int tir_adam_chunk_elems(void);
int tir_adam_step(const TirAdamTensor* table_dev, int32_t n_tensors, const int64_t* chunk_prefix_dev,
                  int64_t total_chunks, float* state_dev, float beta1, float beta2, float eps,
                  const float* found_inf_dev, int32_t clear_grad, void* stream);

/* Total-variation regulariser of up to TIR_TV_MAX_PLANES VM planes in one launch (SURVEY.md 8 f3): TVLoss (utils.py:143-162)
 * as summed by TV_loss_density / TV_loss_app (tensoRF_rotated_lights.py:80-92).  x / grad: the storage of a [1,C,H,W]
 * parameter, channel_last != 0: [H][W][C], else [C][H][W].
 *   tir_tv_loss:     out[0] = sum_planes scale_h * sum (x[h+1]-x[h])^2 + scale_w * sum (x[w+1]-x[w])^2   (out is overwritten)
 *   tir_tv_loss_bwd: grad += gout[0] * d out / d x      (gout in device memory: the weight decays every iteration)
 * The caller folds 2 * TVLoss_weight * 1e-2 / count_h (count_w) into the scales. */
#define TIR_TV_MAX_PLANES 3
typedef struct TirTvPlane {
  const float* x;
  float* grad;                 /* only read by tir_tv_loss_bwd */
  int32_t H, W, C;
  int32_t channel_last;
  float scale_h, scale_w;
} TirTvPlane;
int tir_tv_loss(const TirTvPlane* planes, int32_t n_planes, float* out, void* stream);
int tir_tv_loss_bwd(const TirTvPlane* planes, int32_t n_planes, const float* gout, void* stream);

/* On-the-fly ray generation from (view, pixel) ids (SURVEY.md 8 f4) instead of indexing a [n_views*H*W, 6] host table
 * (train_tensoIR.py:239-242): directions ((i+0.5-W/2)/f, (j+0.5-H/2)/f, 1) normalised and rotated by c2w[:3,:3], origin
 * c2w[:3,3] (dataLoader/ray_utils.py:25-43, :67-88).  c2w [n_views,4,4] row-major, pix = j*W + i -> rays [n,6]. */
int tir_generate_rays(const float* c2w, const int32_t* view_idx, const int32_t* pix_idx, int64_t n, int32_t H, int32_t W,
                      float focal, float* rays, void* stream);

/* Test-view metrics of one rendered view (renderer.py:211-501, utils.py:93-139) from the device maps the renderer
 * returns, [H*W,3] in row-major pixel order.  out[TIR_EVAL_N_OUT] (fp64, device, overwritten):
 *   0 sum (clamp01(rgb) - gt_rgb)^2              1 sum (clamp01(rgb_brdf) - gt_rgb)^2          (over H*W*3)
 *   2 sum (gt_albedo^g - single_aligned^g)^2      3 sum (gt_albedo^g - three_aligned^g)^2       (g = 1/2.2)
 *   4 sum over all pixels of the normal angular error in degrees
 *   5..8 SSIM of rgb/gt_rgb, rgb_brdf/gt_rgb, single_aligned/gt_albedo, three_aligned/gt_albedo (mean over the
 *        (H-10)*(W-10)*3 valid windows; needs H, W >= 11 and ssim != 0, else 0; 7 and 8 need the albedo terms)
 * Terms whose inputs are NULL are skipped and left 0.  The aligned albedo maps (clamp(ratio * albedo, 0, 1) inside
 * gt_mask, 1 outside; ratio[0] for the single-channel and ratio[1..3] for the three-channel variant, in device memory)
 * are written to aligned_single / aligned_three.  Every reduction is fixed-order (per-block fp64 partials in `work`,
 * then one ordered pass): two calls on the same inputs return bit-identical outputs.  work holds
 * tir_eval_work_size(H, W) doubles. */
#define TIR_EVAL_N_OUT 9
typedef struct TirEvalView {
  int32_t H, W;
  int32_t ssim;                           /* != 0: compute the four SSIMs */
  int32_t reserved;
  const float* rgb;                       /* required */
  const float* rgb_brdf;                  /* required */
  const float* gt_rgb;                    /* required */
  const float* albedo;                    /* albedo terms: albedo, gt_albedo, gt_mask, ratio, aligned_* all set, */
  const float* gt_albedo;                 /*   or albedo and gt_albedo both NULL                                   */
  const uint8_t* gt_mask;                 /* [H*W] bool */
  const float* ratio;                     /* [4]: single-channel ratio, three-channel ratio */
  float* aligned_single;                  /* [H*W,3] out */
  float* aligned_three;                   /* [H*W,3] out */
  const float* normal;                    /* normal term: both set, or both NULL */
  const float* gt_normal;
} TirEvalView;
int tir_eval_work_size(int32_t H, int32_t W, int64_t* n_doubles);
int tir_eval_view(const TirEvalView* view, double* work, int64_t work_cap, double* out, void* stream);

/* Metrics of P image pairs (relight_importance.py:216-219): a, b [P,H,W,3] fp32, out[P,2] (fp64, device, overwritten)
 * = per pair the squared-error sum over H*W*3 ((a-b)^2 in fp32, summed in fp64) and the mean SSIM of utils.rgb_ssim
 * (the same pass and the same fixed-order partials as tir_eval_view, so a pair gives the same bits through either
 * entry point).  Needs H, W >= 11.  work holds tir_eval_pairs_work_size(P, H, W) doubles. */
int tir_eval_pairs_work_size(int32_t P, int32_t H, int32_t W, int64_t* n_doubles);
int tir_eval_pairs(const float* a, const float* b, int32_t P, int32_t H, int32_t W, double* work, int64_t work_cap,
                   double* out, void* stream);

/* ---- relighting under environment maps (scripts/relight_importance.py:99-181, Environment_Light of
 * models/relight_utils.py:110-205) ------------------------------------------------------------------------------------
 * One chunk of n primary rays, L environment maps, S importance samples per surface hit, in two calls around the
 * existing density march (tir_march_density with the 96-sample equal-z table over [0.05, 1.5]):
 *   tir_relight_sample  per (map, ray, sample) of a hit ray (acc > acc_mask_threshold): bin = upper bound of u in the
 *                       map's CDF, clamped to H*W-1 (torch.searchsorted(cdf, u, right=True).clamp(max=H*W-1)); the
 *                       sample is appended to the visibility list (origin o + depth*d, direction hdr_dir[bin]) when
 *                       cosine = dir . normal (raw normal) > 1e-6.  bin[L,n,S] and pos[L,n,S] (list row, or -1) are
 *                       written for every slot (bin 0 / pos -1 on non-hit rays).  The list length is accumulated in
 *                       *count (device, caller zeroes); rows past `capacity` are not written (pos -1) but counted.
 *   tir_relight_shade   one warp per (map, ray): mean over S of (albedo*rescale/pi + GGX) * vis * rgb[bin] * cosine /
 *                       pdf_return[bin] with vis = vis_list[pos] (vis_kind 0, nerv: the march's t_last) or
 *                       1 - vis_list[pos] (vis_kind 1, nerfactor: the march's acc), 0 where pos < 0; clamp, sRGB.
 *                       Non-hit rays are white.  The background of every ray is the bilinear (align_corners, zero
 *                       padding) lookup of get_light, clamped and sRGB; with_bg = acc_t*without_bg + (1-acc_t)*bg with
 *                       acc_t = acc > 0.9 ? acc : 0.  Rows are written at [l, row0 + i] of [L, out_rows, 3] maps.
 * Every reduction is in a fixed order (no float atomics): repeated calls give identical bits. */
#define TIR_RELIGHT_MAX_LIGHTS 16
typedef struct TirEnvMap {
  int32_t H, W;
  const float* rgb;         /* [H*W,3] hdr_rgbs */
  const float* dir;         /* [H*W,3] hdr_dir */
  const float* pdf_return;  /* [H*W]   hdr_pdf_return */
  const double* cdf;        /* [H*W]   normalised cumulative sum of hdr_pdf_sample (last entry 1) */
} TirEnvMap;
int tir_relight_sample(const TirEnvMap* envs /* host array [n_lights] */, int32_t n_lights, const float* rays,
                       const float* depth, const float* normal, const float* acc, int64_t n, int32_t n_samples,
                       float acc_mask_threshold, const double* u /* [L,n,S] */, int32_t* bin, int32_t* pos,
                       float* list_o, float* list_d /* [capacity,3] */, int64_t capacity, int64_t* count,
                       void* stream);
int tir_relight_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                      const float* albedo, const float* rough, int32_t rough_stride /* 1: [n,1], 3: [n,3] */,
                      const float* fresnel, const float* acc, int64_t n, int32_t n_samples, float acc_mask_threshold,
                      const float* rescale /* [3] */, const int32_t* bin, const int32_t* pos, const float* vis_list,
                      int32_t vis_kind, float* with_bg, float* without_bg, int64_t out_rows, int64_t row0,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TENSOIR_B200_H */
