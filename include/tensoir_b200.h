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
 *  - no global state, re-entrant, never throws; the one exception is the work counter of the dense secondary march
 *    (tir_secondary_march / tir_secondary_radiance), see there.
 */
#ifndef TENSOIR_B200_H
#define TENSOIR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TIR_ABI_VERSION 4

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
  const uint8_t* acell;    /* [Z][Y][X] OR of the 8 corners of cell (x,y,z) (built by tir_pack_alpha_mask), followed
                              by the occupancy bricks: at byte offset X*Y*Z rounded up to 16, one bit per brick of
                              E^3 cells = the OR of acell over the brick, brick (bx,by,bz) at bit (bz*BY + by)*BX + bx
                              of little-endian uint32 words, BX = ceil(X/E) etc.  E is the smallest power of two >= 8
                              that keeps BX*BY*BZ <= 65536 (8 KB).  Read only when cfg.flags has
                              TIR_MARCH_CELL_BRICKS; tir_alpha_cells_bytes gives the size of the whole buffer. */
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
  TIR_MARCH_LEAN_COUNTERS = 2,
  /* field.acell is followed by the occupancy bricks tir_pack_alpha_mask builds (see TirField.acell): a sample strictly
   * inside a cell of an empty brick is rejected without reading acell.  Same valid samples, same counters. */
  TIR_MARCH_CELL_BRICKS = 4
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

/* float alpha_volume [Z,Y,X] (0/1) -> corner bytes + per-cell OR bytes (AlphaGridMask, tensorBase:100-119) + the
 * occupancy bricks behind the cell bytes.  corners holds X*Y*Z bytes, cells tir_alpha_cells_bytes(X, Y, Z) bytes. */
int tir_pack_alpha_mask(const float* volume, uint8_t* corners, uint8_t* cells,
                        int32_t X, int32_t Y, int32_t Z, void* stream);
int tir_alpha_cells_bytes(int32_t X, int32_t Y, int32_t Z, int64_t* n_bytes);

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
 * Rays are generated on chip (no [bs,n_dirs,3] tensors).  Point-major: a CTA marches all directions of one surface
 * point before it takes the next one from a per-device work counter, which the launch leaves at zero when it ends, so
 * two of these calls must not run concurrently on different streams of one device.
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

/* The density feature of compute_densityfeature (models/tensoRF_rotated_lights.py:95-110) sampled at the density-grid
 * vertices of a sub-box [lo, lo+n) of the grid, stored [z][y][x] with x fastest (n[0]*n[1]*n[2] floats):
 *   D[x,y,z] = sum_k sum_c plane_k[c](x_{m0}, x_{m1}) * line_k[c](x_v)
 * For every orientation k, bilinear(plane) * linear(line) uses separable weights, so the feature at any point is the
 * trilinear interpolation of D with the same taps and the same zero padding.  The secondary march reads 8 floats of D
 * per sample instead of 6 taps x 3 orientations x C channels of the factors.  D is a function of the live density
 * factors: rebuild it (tir_density_volume_build) before every march that reads it, never keep it across a parameter
 * update. */
typedef struct TirDensityVolume {
  float* data;
  int32_t lo[3];           /* first density-grid vertex x,y,z of the box */
  int32_t n[3];            /* vertices along x,y,z; 0 along any axis = empty box */
} TirDensityVolume;

/* Host-only (no device access, no stream).  The box every valid sample of the secondary march reads: the density-grid
 * vertices whose trilinear taps a point inside the occupied-cell box field->occ_lo/occ_hi can touch (computed with the
 * kernels' own coordinate arithmetic), grown by one vertex on each side against rounding and clamped to the grid.  The
 * whole grid when the field has no alpha mask or no box (occ_lo > occ_hi); an empty box (some n == 0) when the
 * occupied-cell box does not meet the grid.  TIR_ERR_SHAPE when a grid size is < 1. */
int tir_density_volume_extent(const TirField* field, int32_t lo[3], int32_t n[3]);

/* Fills vol->data over the box vol->lo / vol->n from the density factors of `field` (plane and line rows are read once
 * per tile of vertices; per vertex the channels of an orientation are summed in channel order, then the three
 * orientations in order 0,1,2, as the factor path sums them).  TIR_ERR_CAPACITY when capacity (floats) is smaller than
 * n[0]*n[1]*n[2]; TIR_ERR_SHAPE when the box leaves the grid or dC != 16. */
int tir_density_volume_build(const TirField* field, TirDensityVolume* vol, int64_t capacity, void* stream);

/* tir_secondary_march / tir_secondary_radiance with the density of every sample read from `vol` (built from the same
 * field by tir_density_volume_build over the box tir_density_volume_extent gives): 8 trilinear corner reads instead of
 * the 18-tap factor gather.  Same samples, masks, counters and outputs as the factor path up to the rounding of the
 * density feature.  The factor-path entry points above stay the reference. */
int tir_secondary_radiance_vol(const TirField* field, const TirMlp* mlp, const float* surf_xyz, const float* normals,
                               const int32_t* light_idx, int64_t n_pts, const float* dirs, int32_t n_dirs,
                               const TirMarchCfg* cfg, const TirDensityVolume* vol, float* vis, float* indirect,
                               TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                               uint64_t* counters, void* stream);
int tir_secondary_march_vol(const TirField* field, const float* surf_xyz, const float* normals, int64_t n_pts,
                            const float* dirs, int32_t n_dirs, const TirMarchCfg* cfg, const TirDensityVolume* vol,
                            float* vis, TirAppSample* samples, uint32_t* sample_count, int64_t capacity,
                            uint64_t* counters, void* stream);

/* Appearance gather + basis_mat + MLPRender_Fea on a compacted sample list
 * (compute_appfeature tensoRF_rotated_lights.py:197-224 + MLPRender_Fea tensorBase:136-146):
 *   rgb_out[ray] += weight * sigmoid(mlp(...)) for every sample; mlp->out_dim must be 3.
 *   The view dir of a sample is ray_dirs[ray] ([n_rays,3]) when n_dirs == 0, or the [n_dirs,3] table row ray % n_dirs
 *   when n_dirs > 0.  light_idx indexed by ray (n_dirs == 0) or by ray / n_dirs.
 * Runs the sm_90a wgmma kernel (csrc/tir_mlp_wgmma.cu): A operand and accumulator in registers, split-BF16 weights
 * resident in shared memory, three warpgroups per CTA on different 64-sample tiles. */
int tir_app_mlp(const TirField* field, const TirMlp* mlp, const TirAppSample* samples,
                const uint32_t* sample_count, int64_t max_samples, const float* ray_dirs, int32_t n_dirs,
                const int32_t* light_idx, float* rgb_out, void* stream);

/* The same gather + MLP on explicit points (no compositing): xn [n,3] normalised coords, x_in [n,3] the 3-vector fed
 * to the MLP next to the features (view dir for MLPRender_Fea, position for MLPBRDF_PEandFeature),
 * light_idx [n] or NULL (row 0 of mlp->light_line, e.g. the mean-light row of compute_intrinfeature),
 * act 0 = sigmoid, 1 = tanh -> out [n,out_dim].  Mirrors renderModule*(compute_*feature(...)).
 * Optionally dumps the activations a host-side backward needs (training forward of the primary MLP heads):
 * save_xl [n, 3*aC] light-scaled products, save_in [n, in_dim] MLP input incl. positional encoding,
 * save_h1 / save_h2 [n, hidden] post-ReLU hidden layers; any of them may be NULL.
 * Runs the split-BF16 mma.sync kernel of the primary heads (csrc/tir_mlp.cu). */
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

/* TensorBase.forward with is_relight=False (tensorBase_rotated_lights.py:868-986, the radiance-only warm-up phase of
 * training) on the same march, appearance list and scratch: after tir_primary_march + tir_primary_app_list,
 *   tir_primary_radiance           ONE head (role TIR_HEAD_RGB, point_set 0, x_in 0: renderModule on the view
 *                                  direction) into work->out[0], then per ray rgb_map = sum w * rgb and, when
 *                                  white_bg != 0, rgb_map += 1 - acc, depth_map = depth + (1 - acc) * rays[..., 5].
 *                                  No clamp, no sRGB (the reference's radiance branch has neither).  rgb_map [n_rays,3],
 *                                  depth_map [n_rays]; acc stays in work->acc.  work->noise, a_xj, packed, dn_* unused.
 *   tir_primary_radiance_backward  epilogue -> per-sample tail -> head dgrad / wgrad (job slot 0 of bwork and grads) ->
 *                                  appearance scatter -> compositing -> density scatter.  g_rgb_map [n_rays,3],
 *                                  g_depth_map, g_acc_map [n_rays] may each be NULL (zero).  grads ACCUMULATED.
 * Saving the activations for the backward needs work->x0[0], inp[0], h1[0], h2[0]; x0[1] is never read. */
int tir_primary_radiance(const TirField* field, const TirHeadJob* job, const float* rays, const int32_t* light_idx,
                         int64_t n_rays, const TirPrimaryWork* work, int32_t white_bg, float* rgb_map,
                         float* depth_map, void* stream);
int tir_primary_radiance_backward(const TirField* field, const TirHeadJob* job, const float* rays,
                                  const int32_t* light_idx, int64_t n_rays, const TirPrimaryWork* work,
                                  const TirPrimaryBwdWork* bwork, int32_t white_bg, const float* g_rgb_map,
                                  const float* g_depth_map, const float* g_acc_map, const TirPrimaryGrads* grads,
                                  void* stream);

/* ---- optimiser pass (SURVEY.md 8 f3): torch.optim.Adam's update for a list of dense fp32 tensors in ONE launch, with
 * the L1 regulariser's gradient (l1 * sign(param), density_L1 of tensoRF_rotated_lights.py:74-78) folded in, the
 * gradient cleared for the next accumulation, and a device-side skip flag (found_inf != 0: parameters, moments and the
 * step counts stay untouched, gradients are still cleared).  Every tensor has its own step count (torch.optim.Adam's
 * per-parameter state["step"]), advanced by one per call.  table / chunk_prefix / bias live in device memory:
 * chunk_prefix[k] = first chunk (of tir_adam_chunk_elems() elements) of tensor k; bias: 2 * n_tensors floats of scratch
 * (tensor k's 1-beta1^t and sqrt(1-beta2^t)). */
typedef struct TirAdamTensor {
  float* p; float* g; float* m; float* v;   /* parameter, gradient, exp_avg, exp_avg_sq: same dense layout, n elements */
  int64_t n;
  const float* lr_dev;                      /* learning rate in device memory (CUDA-graph replay), or NULL -> lr */
  float lr;
  float l1;                                 /* coefficient of sign(param) added to the gradient (0: none) */
  float* step;                              /* this tensor's step count: one float in device memory */
} TirAdamTensor;
int tir_adam_chunk_elems(void);
int tir_adam_step(const TirAdamTensor* table_dev, int32_t n_tensors, const int64_t* chunk_prefix_dev,
                  int64_t total_chunks, float* bias_dev, float beta1, float beta2, float eps,
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

/* ---- relighting with multiple importance sampling: GGX-lobe samples combined with environment-map samples ----------
 * An opt-in estimator of the same chunk (tir_relight_shade's is the default).  For a hit ray i and map l:
 *
 *   linear[l,i] = sum over the S_l light samples of map l and the S_b BRDF samples of ray i of
 *                 f(w) * V(w) * E_l(w) * cos(w) / (S_l * p_light_l(w) + S_b * p_brdf(w))
 *
 * an unbiased estimate of the integral of f V E cos over the sphere, with f tir_relight_shade's BRDF, cos the raw-normal
 * cosine (a sample with cos <= 1e-6 contributes 0 and is not marched), V the march's visibility as tir_relight_shade
 * reads it, and E_l map l taken as piecewise constant over its lat-long texels.  Light samples: a texel from the fp64
 * CDF, then a point uniform in its solid angle, p_light = P_texel / dOmega_texel (exact solid angle).  BRDF samples,
 * one set per ray shared by every map: with probability 1/2 a GGX visible-normal half vector (alpha = mean(r)^2, about
 * the view-side normal) reflected, else a cosine-weighted direction; p_brdf = 1/2 G1(V) D(h) / (4 NoV) + 1/2 max(Np.w,
 * 0) / pi.  E and p_light of every sample come from the texel of its direction as rounded.  Definitions in
 * csrc/tir_mis_body.h.  Slots: the L*n*S_l light slots (map, ray, sample) first, then the n*S_b BRDF slots (ray,
 * sample).
 *   tir_relight_mis_sample  one thread per slot of a hit ray (acc > acc_mask_threshold), u_light [L,n,S_l,3] and
 *                           u_brdf [n,S_b,3] fp64 (u_brdf may be NULL when S_b = 0): dir [slots,3] and pos [slots]
 *                           (list row, or -1) for every slot (zeros and -1 on non-hit rays); the marched slots'
 *                           (surface point, direction) are appended to list_o / list_d; count and capacity as in
 *                           tir_relight_sample.
 *   tir_march_density       on the list, by the caller, with relight()'s table.
 *   tir_relight_mis_shade   one warp per (map, ray), lanes over the map's light slots and then the ray's BRDF slots:
 *                           linear as above in a fixed order, without_bg = sRGB(clamp(linear)), white on non-hit rays;
 *                           with_bg as tir_relight_shade.  linear_out (NULL allowed) [L,out_rows,3] gets the un-toned
 *                           sum, 0 on non-hit rays.  Rows are written at [l, row0 + i] of [L, out_rows, 3] maps.
 * Repeated calls on the same list give identical bits.  TIR_ERR_SHAPE for n < 0, S_l < 1, S_b < 0, a stride other than
 * 1 or 3, more than TIR_RELIGHT_MAX_LIGHTS maps, capacity outside [0, INT32_MAX] or output rows out of range;
 * TIR_ERR_CONFIG for an unknown vis_kind; TIR_ERR_NULL for a missing input. */
int tir_relight_mis_sample(const TirEnvMap* envs /* host array [n_lights] */, int32_t n_lights, const float* rays,
                           const float* depth, const float* normal, const float* albedo, const float* rough,
                           int32_t rough_stride /* 1: [n,1], 3: [n,3] */, const float* fresnel, const float* acc,
                           int64_t n, int32_t S_l, int32_t S_b, float acc_mask_threshold, const double* u_light,
                           const double* u_brdf, float* dir, int32_t* pos, float* list_o,
                           float* list_d /* [capacity,3] */, int64_t capacity, int64_t* count, void* stream);
int tir_relight_mis_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                          const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                          const float* acc, int64_t n, int32_t S_l, int32_t S_b, float acc_mask_threshold,
                          const float* rescale /* [3] */, const float* dir, const int32_t* pos, const float* vis_list,
                          int32_t vis_kind, float* with_bg, float* without_bg, float* linear_out /* or NULL */,
                          int64_t out_rows, int64_t row0, void* stream);

/* ---- material editing: the BRDF parameters of n surface points, edited by a table of rules, for tir_relight_shade
 * (or any other consumer) ----------------------------------------------------------------------------------------------
 * The point of row i is points[i] when `points` is given, else rays[i].o + depth[i] * rays[i].d rounded as
 * tir_relight_sample rounds it (the same bits as the visibility list's origin).  a0 = albedo[i] * scale (one fp32
 * multiply per channel) is the unedited scaled albedo.
 *   Rows with acc[i] > acc_threshold are edited: the rules are visited in order; rule k selects the row when the point
 *   lies inside its box (box_lo <= p <= box_hi on every axis, when TIR_EDIT_BOX) and max_c |a0[c] - key[c]| <= key_tol
 *   (when TIR_EDIT_KEY); a rule with neither flag selects every row.  A selecting rule applies its albedo, roughness and
 *   fresnel ops to the running values (SET: the rule's value, MUL: value * rule's value, fp32), each op followed by a
 *   clamp of the value it wrote: albedo and fresnel to [0, 1], roughness to [TIR_EDIT_ROUGH_MIN, TIR_EDIT_ROUGH_MAX]
 *   (the model's valid_brdf * 0.9 + 0.09 range); the roughness value applies to every channel of a [n,3] roughness.
 *   Selection always tests the unedited a0.  sel[i] gets bit k when rule k selected the row.
 *   Every other row is passed through: albedo_out = a0, roughness and fresnel copied, sel = 0.
 * Outputs are out of place: albedo_out [n,3], rough_out [n,rough_stride], fresnel_out [n,3], sel [n] int32.  Since
 * albedo_out already holds the scale, pass rescale (1,1,1) to tir_relight_shade: an edit table without rules then
 * shades to the same bits as the unedited call with rescale = scale.  One thread per row, no atomics: reruns are
 * bit-identical.  TIR_ERR_SHAPE for n < 0, more than TIR_EDIT_MAX_RULES rules or a stride other than 1 or 3;
 * TIR_ERR_CONFIG for an unknown op or flag. */
#define TIR_EDIT_MAX_RULES 16
#define TIR_EDIT_ROUGH_MIN 0.09f
#define TIR_EDIT_ROUGH_MAX 0.99f
enum { TIR_EDIT_NONE = 0, TIR_EDIT_SET = 1, TIR_EDIT_MUL = 2 };
enum { TIR_EDIT_BOX = 1, TIR_EDIT_KEY = 2 };
typedef struct TirEditRule {
  int32_t flags;                                  /* TIR_EDIT_BOX | TIR_EDIT_KEY */
  int32_t albedo_op, rough_op, fresnel_op;        /* TIR_EDIT_NONE / SET / MUL */
  float box_lo[3], box_hi[3];
  float key[3], key_tol;
  float albedo[3], rough, fresnel[3];
} TirEditRule;
int tir_material_edit(const TirEditRule* rules /* host array [n_rules] */, int32_t n_rules, const float* rays,
                      const float* depth, const float* points /* [n,3] or NULL: use rays and depth */,
                      const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                      const float* acc, int64_t n, float acc_threshold, const float* scale /* [3] */,
                      float* albedo_out, float* rough_out, float* fresnel_out, int32_t* sel, void* stream);

/* ---- relighting under analytic lights: directional, point and spot lights with marched shadows -----------------------
 * One chunk of n primary rays under one setup of up to TIR_LIGHTS_MAX lights, light j with K_j area samples, in two
 * calls around tir_march_density (as tir_relight_sample / tir_relight_shade are).  The slots of a chunk are laid out
 * light-major: slot(j, i, s) = n * (K_0 + ... + K_{j-1}) + i * K_j + s, so lights of one setup may have different K.
 *   tir_lights_sample  per slot of a hit ray (acc > acc_mask_threshold), from the surface point p = o + depth*d: the
 *                      unit direction L towards the light sample and the falloff.  A light without extent, or with
 *                      K = 1, is sampled at its centre and reads no uniform; otherwise (u[slot][0], u[slot][1]) is
 *                      mapped to the unit disc (concentric map; the disc's axes are the orthonormal basis of Duff et
 *                      al. 2017 around its normal) and the sample lies
 *                        directional: at dir + extent * disc on the plane tangent to dir (extent = tan of the angular
 *                                     radius), L its normalisation, falloff 1;
 *                        point, spot: at pos + extent * disc on the disc of the sphere that faces p, L = (q - p)/d,
 *                                     falloff = cone / d^2, cone = 1 for a point light and, for a spot, 1 where
 *                                     c = -L . dir >= cos_inner, 0 where c <= cos_outer and smoothstep of
 *                                     (c - cos_outer) / (cos_inner - cos_outer) between.
 *                      The slot joins the shadow-ray list (origin p, direction L) when L . normal (raw normal) > 1e-6
 *                      and falloff > 0.  L [slots,3], falloff [slots] and pos [slots] (list row, or -1) are written for
 *                      every slot (zeros and -1 on non-hit rays); count and capacity as in tir_relight_sample.
 *   tir_lights_shade   one warp per ray: linear = sum over lights, in order, of power_j * mean over the light's K slots
 *                      of (albedo*rescale/pi + GGX) * vis * falloff * cosine, vis as in tir_relight_shade (0 where
 *                      pos < 0).  without_bg = sRGB(clamp(linear)), white on non-hit rays; with_bg = acc_t*without_bg +
 *                      (1-acc_t)*background with acc_t = acc > 0.9 ? acc : 0.  `linear` (may be NULL) gets the un-toned
 *                      sum, 0 on non-hit rays.  Rows are written at [row0 + i] of [out_rows,3] maps.
 * A point or spot light must lie outside the model's aabb: a shadow ray then leaves the box before it reaches the light,
 * so tir_march_density, which has one far for all rays, is exact for it.  Every reduction is in a fixed order (no float
 * atomics): repeated calls give identical bits.  TIR_ERR_SHAPE for n < 0, more than TIR_LIGHTS_MAX lights, K outside
 * [1, TIR_LIGHT_SAMPLES_MAX], more than INT32_MAX slots, a stride other than 1 or 3 or rows out of range;
 * TIR_ERR_CONFIG for an unknown type or vis_kind. */
#define TIR_LIGHTS_MAX 16
#define TIR_LIGHT_SAMPLES_MAX 1024
enum { TIR_LIGHT_DIRECTIONAL = 0, TIR_LIGHT_POINT = 1, TIR_LIGHT_SPOT = 2 };
typedef struct TirLight {
  int32_t type, n_samples;
  float dir[3];                /* unit; directional: towards the light; spot: axis, light -> target */
  float pos[3];                /* point, spot */
  float power[3];              /* irradiance facing the light (directional) or radiant intensity (point, spot) */
  float extent;                /* directional: tan(angular radius); point, spot: sphere radius */
  float cos_inner, cos_outer;  /* spot */
} TirLight;
int tir_lights_sample(const TirLight* lights /* host array [n_lights] */, int32_t n_lights, const float* rays,
                      const float* depth, const float* normal, const float* acc, int64_t n,
                      float acc_mask_threshold, const double* u /* [slots,2] */, float* L, float* falloff,
                      int32_t* pos, float* list_o, float* list_d /* [capacity,3] */, int64_t capacity, int64_t* count,
                      void* stream);
int tir_lights_shade(const TirLight* lights, int32_t n_lights, const float* rays, const float* normal,
                     const float* albedo, const float* rough, int32_t rough_stride /* 1: [n,1], 3: [n,3] */,
                     const float* fresnel, const float* acc, int64_t n, float acc_mask_threshold,
                     const float* rescale /* [3] */, const float* background /* [3] */, const float* L,
                     const float* falloff, const int32_t* pos, const float* vis_list, int32_t vis_kind, float* with_bg,
                     float* without_bg, float* linear /* or NULL */, int64_t out_rows, int64_t row0, void* stream);

/* ---- light transport to the texels of an environment map (inverse lighting) -----------------------------------------
 * With geometry and materials fixed, relight()'s shading is linear in the environment map: for one surface hit its
 * estimator has expectation sum_k f_k * vis_k * cos_k * L_k * dOmega_k over the map's K = H*W texels, with
 * dOmega_k = pdf / pdf_return = 2 pi^2 sin(theta_k) / (H W).  These two calls write that linear map, the transport
 * T[c, i, k], around tir_march_density (relight()'s 96-sample equal-z table over [0.05, 1.5]):
 *   tir_transport_sample  per (ray, texel) of a hit ray (acc > acc_mask_threshold): the texel's direction dirs[k] joins
 *                         the visibility list (origin o + depth*d, direction dirs[k]) when dirs[k] . normal (raw normal)
 *                         > 1e-6, as a sample of tir_relight_sample does.  pos[n,K] (list row, or -1) is written for
 *                         every (ray, texel), -1 on non-hit rays; count and capacity as in tir_relight_sample.
 *   tir_transport_build   one warp per ray, lanes over the texels: T[c, i, k] = (albedo*rescale/pi + GGX)_c * vis *
 *                         cosine * dOmega[k], the per-sample term of tir_relight_shade with unit radiance and the solid
 *                         angle in place of 1 / pdf_return; vis as in tir_relight_shade; 0 where pos < 0 and on rows
 *                         with acc <= acc_mask_threshold.  T is [3, n, K] fp32: one contiguous [n, K] matrix per channel.
 * No reduction, no float atomics: repeated calls on the same list give identical bits.  TIR_ERR_SHAPE for K outside
 * [1, TIR_TRANSPORT_MAX_TEXELS], n < 0, n*K > INT32_MAX, capacity outside [0, INT32_MAX] or a stride other than 1 or 3;
 * TIR_ERR_CONFIG for an unknown vis_kind. */
#define TIR_TRANSPORT_MAX_TEXELS 2048
int tir_transport_sample(const float* dirs /* [K,3] */, int32_t K, const float* rays, const float* depth,
                         const float* normal, const float* acc, int64_t n, float acc_mask_threshold, int32_t* pos,
                         float* list_o, float* list_d /* [capacity,3] */, int64_t capacity, int64_t* count,
                         void* stream);
int tir_transport_build(const float* dirs, const float* domega /* [K] */, int32_t K, const float* rays,
                        const float* normal, const float* albedo, const float* rough,
                        int32_t rough_stride /* 1: [n,1], 3: [n,3] */, const float* fresnel, const float* acc,
                        int64_t n, float acc_mask_threshold, const float* rescale /* [3] */, const int32_t* pos,
                        const float* vis_list, int32_t vis_kind, float* T /* [3,n,K] */, void* stream);

/* ---- one bounce of indirect light for relighting under environment maps ----------------------------------------------
 * For a hit primary ray i (acc > acc_mask_threshold) and map l:
 *
 *   linear[l,i] = (1/S)  * sum_s direct_s                  (exactly tir_relight_shade's sum, same order, same bits)
 *               + (1/K)  * sum_k T[i,k] * w[i,k] * Lo[l, h(i,k)]
 *   without_bg  = tone(linear),  with_bg = rl_composite(...)  (as tir_relight_shade)
 *
 * with K cosine-weighted directions per hit (Malley's method on lt_disc and lt_frame of the normalised normal), their
 * throughput T = (albedo*rescale/pi + GGX) * cosine / pdf, the secondary march's occlusion weight w = 1 - vis, and Lo
 * the un-toned direct light of map l at the secondary hit x = p + (depth / acc) * omega seen from -omega (definitions
 * in csrc/tir_indirect_body.h).  One bounce only; cosine sampling only.  Around the existing calls:
 *   tir_indirect_sample   per (ray, slot), u [n,K,2] fp64: dir [n,K,3], T [n,K,3] and pos [n,K] (secondary-list row or
 *                         -1) for every slot (zeros and -1 on non-hit rays and on slots with cosine or z <= 1e-6); the
 *                         marched slots' (surface point, direction) are appended to list_o / list_d; count and
 *                         capacity as in tir_relight_sample.
 *   tir_march_density     on the list, with relight()'s table: t_last, acc, depth per list row.
 *   tir_indirect_hits     per slot, through pos: a secondary hit when w > 1e-3 and acc > 0, with w = 1 - t_last
 *                         (vis_kind 0, nerv) or 1 - (1 - acc) (vis_kind 1, nerfactor).  The hits are compacted in slot
 *                         order (a scan, not an append): hit_rays [m_h,6] = (x, omega), xn [m_h,3] = (x - aabb[0:3]) *
 *                         aabb[3:6] - 1 (aabb: host [6] = lo, inverse half extent), w [m_h], hit [n,K] (row or -1).
 *                         *count (device) is set to m_h; rows past capacity are not written (hit -1) but counted.
 *                         work: tir_indirect_hits_work_size bytes of device scratch (TIR_ERR_CAPACITY when smaller).
 *   tir_relight_sample    + tir_march_density on the hits (rays = hit_rays, depth 0), S2 samples per hit.
 *   tir_indirect_radiance one warp per (map, hit): Lo[l, row0 + h] of [L, out_rows, 3] = mean over S2 of rl_contrib
 *                         with the view direction -omega, un-toned; vis as in tir_relight_shade.
 *   tir_indirect_shade    one warp per (map, ray): tir_relight_shade's outputs with the indirect sum added before the
 *                         tone map on rays with at least one hit slot (other rows have tir_relight_shade's bits).
 *                         Lo [L, m_h, 3]; indirect (NULL allowed) [L, out_rows, 3] receives the un-toned indirect term.
 * Fixed-order sums and a stable hit list: repeated calls give identical bits.  TIR_ERR_SHAPE for n < 0, K outside
 * [1, 1024], S2 outside [1, 1024], n*K > INT32_MAX, more than TIR_RELIGHT_MAX_LIGHTS maps, capacity outside
 * [0, INT32_MAX], a stride other than 1 or 3 or output rows out of range; TIR_ERR_CONFIG for an unknown vis_kind. */
int tir_indirect_sample(const float* rays, const float* depth, const float* normal, const float* albedo,
                        const float* rough, int32_t rough_stride, const float* fresnel, const float* acc, int64_t n,
                        int32_t K, float acc_mask_threshold, const float* rescale /* [3] */, const double* u,
                        float* dir, float* T, int32_t* pos, float* list_o, float* list_d /* [capacity,3] */,
                        int64_t capacity, int64_t* count, void* stream);
int tir_indirect_hits_work_size(int64_t n, int32_t K, int64_t* bytes);
int tir_indirect_hits(int64_t n, int32_t K, const int32_t* pos, const float* list_o, const float* list_d,
                      const float* t_last, const float* acc, const float* depth, int32_t vis_kind,
                      const float* aabb /* host [6] */, float* hit_rays, float* xn, float* w, int32_t* hit,
                      int64_t capacity, int64_t* count, void* work, int64_t work_bytes, void* stream);
int tir_indirect_radiance(const TirEnvMap* envs, int32_t n_lights, const float* hit_rays, const float* normal,
                          const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                          int64_t m, int32_t n_samples, const float* rescale, const int32_t* bin, const int32_t* pos,
                          const float* vis_list, int32_t vis_kind, float* Lo, int64_t out_rows, int64_t row0,
                          void* stream);
int tir_indirect_shade(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* normal,
                       const float* albedo, const float* rough, int32_t rough_stride, const float* fresnel,
                       const float* acc, int64_t n, int32_t n_samples, float acc_mask_threshold,
                       const float* rescale, const int32_t* bin, const int32_t* pos, const float* vis_list,
                       int32_t vis_kind, int32_t K, const float* T, const int32_t* hit, const float* w,
                       const float* Lo, int64_t m_h, float* with_bg, float* without_bg, float* indirect,
                       int64_t out_rows, int64_t row0, void* stream);

/* ---- camera-path frames: rotated environment maps and a shadow-catching ground plane ---------------------------------
 * Conventions.  Cameras are camera-to-world matrices in the OpenCV convention (x right, y down, z forward), as the
 * datasets (transform_matrix @ blender2opencv) and tir_generate_rays use.  A map rotated by angle a turns about world +z
 * with R(a) = [[cos a, -sin a, 0], [sin a, cos a, 0], [0, 0, 1]] (the reference's light_rotation matrix): the radiance
 * arriving from world direction w is E(w @ R(a)), w a row vector, as the reference lights with
 * init_light_directions @ rotation_matrix.  The object under a rotated map is shaded by tir_relight_sample and
 * tir_relight_shade with the map's dir table replaced by dir @ R(a)^T (bins, rgb, pdf_return and cdf unchanged), which
 * rotates their estimator exactly.
 *
 * The ground is the plane z = ground_z with normal +z, a shadow catcher: it receives the object's shadow but does not
 * occlude or light the object.  Primary ray i has a ground point p = o + t d when d.z < 0 and t > 0 (never for a NaN
 * ground_z); p.z is ground_z.
 *   tir_ground_sample   per (map, ray, slot) of a ray with a ground point, u [L,n,S] fp64: bin = rl_bin of u in the
 *                       map's CDF (as tir_relight_sample), w = dir[bin] of the (rotated) table, and
 *                         pos = -1          when w.z <= 1e-6: the slot counts nowhere;
 *                         pos = -2          when the shadow ray p + t w (t >= 0) misses the box [box_lo, box_hi]
 *                                           (host [3] each; lo > hi on an axis: empty): unoccluded, not marched;
 *                         pos = list row    otherwise: (p + max(t_enter - TIR_PATH_SHADOW_NEAR, 0) w, w) is appended,
 *                                           so a march whose first sample is at TIR_PATH_SHADOW_NEAR starts at the box
 *                                           entry.
 *                       Rays without a ground point get bin 0, pos -1 in every slot.  count and capacity as in
 *                       tir_relight_sample.  The box is the model's occupied-cell box (TirField.occ_lo/occ_hi, where
 *                       the march finds every valid sample), or its aabb without an alpha mask: a shadow ray that misses
 *                       it would march through no valid sample and see t_last 1, acc 0.
 *   tir_march_density   on the list, by the caller, with a table from TIR_PATH_SHADOW_NEAR out past the box diagonal.
 *   tir_path_composite  one warp per (map, pixel): r_c = sum E_c cos V / pdf / sum E_c cos / pdf over the ray's slots
 *                       with pos != -1 (fixed lane order), E = rgb[bin], cos = w.z, pdf = pdf_return[bin], V = 1 for
 *                       pos -2 and the march's visibility as tir_relight_shade reads it for pos >= 0; r clamped to
 *                       [0, 1], 1 when the denominator is 0 and on rays without a ground point.  bg = get_light at
 *                       d @ rot (rot = R(a), host [9] row-major, shared by the call's maps) times r per channel;
 *                       with_bg = acc_t*without_bg + (1-acc_t)*sRGB(clamp(bg)), acc_t = acc > 0.9 ? acc : 0, with
 *                       without_bg read from the same rows (tir_relight_shade's output).  shadow (NULL allowed) gets r.
 *                       Rows are [l, row0 + i] of [L, out_rows, 3] maps.  With a NaN ground_z and rot the identity,
 *                       with_bg has tir_relight_shade's bits; bin, pos and vis_list are then not read and may be NULL.
 * The ratio is differential rendering with a diffuse receiver: both sums use the same samples, so an unoccluded point
 * gets exactly 1.  Repeated calls on the same list give identical bits.  TIR_ERR_SHAPE for n < 0, S < 0 (S < 1 for the
 * composite with a ground), more than TIR_RELIGHT_MAX_LIGHTS maps, capacity outside [0, INT32_MAX] or output rows out of
 * range; TIR_ERR_CONFIG for an unknown vis_kind; TIR_ERR_NULL for a missing input. */
#define TIR_PATH_SHADOW_NEAR 0.05f
int tir_ground_sample(const TirEnvMap* envs /* host array [n_lights] */, int32_t n_lights, const float* rays, int64_t n,
                      float ground_z, const float* box_lo /* host [3] */, const float* box_hi /* host [3] */,
                      int32_t n_samples, const double* u /* [L,n,S] */, int32_t* bin, int32_t* pos, float* list_o,
                      float* list_d /* [capacity,3] */, int64_t capacity, int64_t* count, void* stream);
int tir_path_composite(const TirEnvMap* envs, int32_t n_lights, const float* rays, const float* acc, int64_t n,
                       const float* rot /* host [9] */, float ground_z, const int32_t* bin, const int32_t* pos,
                       const float* vis_list, int32_t vis_kind, int32_t n_samples, const float* without_bg,
                       float* with_bg, float* shadow /* or NULL */, int64_t out_rows, int64_t row0, void* stream);

/* The same ground under one setup of analytic lights (the TirLight table of tir_lights_sample; the object shaded by
 * tir_lights_sample / tir_lights_shade).  Slots are laid out light-major as tir_lights_sample's, slot(j, i, s) =
 * n * (K_0 + ... + K_{j-1}) + i * K_j + s, and read their uniforms under the same rule.
 *   tir_ground_lights_sample   per slot of a ray with a ground point p: L and falloff of the light sample seen from p
 *                              (as tir_lights_sample, spot cone and 1/d^2 included), g = falloff * L.z (the slot's
 *                              unshadowed irradiance weight on the +z receiver), and
 *                                pos = -1        when L.z <= 1e-6 or g <= 0: the slot counts nowhere;
 *                                pos = -2        when the shadow ray p + t L misses the box, or, for a point or spot
 *                                                light, enters it at t_enter >= |q - p|, the distance to the light
 *                                                sample q: unoccluded, not marched;
 *                                pos = list row  otherwise, appended as by tir_ground_sample.
 *                              Rays without a ground point get g 0, pos -1 in every slot.  The box must lie inside the
 *                              model's aabb (the occupied-cell box clipped to it) and every point or spot light sample
 *                              outside the aabb: then a shadow ray that enters the box before the light also leaves it
 *                              before the light, every valid march sample lies between p and the light, and the distance
 *                              cull is exact.
 *   tir_march_density          on the list, by the caller, as for tir_ground_sample.
 *   tir_path_lights_composite  one warp per pixel: r_c = sum_j power_jc / K_j * sum_s g V  /  sum_j power_jc / K_j *
 *                              sum_s g over the slots with pos != -1 (per light, lanes in a fixed order and the xor
 *                              butterfly; lights in order), V as for tir_path_composite; r clamped to [0, 1], 1 when
 *                              the denominator is 0 and on rays without a ground point.  bg_c = background_c where
 *                              r_c == 1, else sRGB(clamp(background_linear_c * r_c)): background is the setup's display
 *                              colour (host [3]), background_linear its linear value (host [3]), so the shadow darkens
 *                              linear light.  with_bg = acc_t*without_bg + (1-acc_t)*bg, acc_t as in tir_lights_shade,
 *                              without_bg read from the same rows (tir_lights_shade's output).  shadow (NULL allowed)
 *                              gets r.  Rows are [row0 + i] of [out_rows, 3] maps.  With a NaN ground_z, with_bg has
 *                              tir_lights_shade's bits; g, pos and vis_list are then not read and may be NULL.
 * Both sums of the ratio use the same expressions in the same order, so an unoccluded point gets exactly 1.  Repeated
 * calls on the same list give identical bits.  TIR_ERR_SHAPE for n < 0, more than TIR_LIGHTS_MAX lights, K outside
 * [1, TIR_LIGHT_SAMPLES_MAX], more than INT32_MAX slots, capacity outside [0, INT32_MAX] or output rows out of range;
 * TIR_ERR_CONFIG for an unknown light type or vis_kind; TIR_ERR_NULL for a missing input. */
int tir_ground_lights_sample(const TirLight* lights /* host array [n_lights] */, int32_t n_lights, const float* rays,
                             int64_t n, float ground_z, const float* box_lo /* host [3] */,
                             const float* box_hi /* host [3] */, const double* u /* [slots,2] */, float* g /* [slots] */,
                             int32_t* pos /* [slots] */, float* list_o, float* list_d /* [capacity,3] */,
                             int64_t capacity, int64_t* count, void* stream);
int tir_path_lights_composite(const TirLight* lights, int32_t n_lights, const float* rays, const float* acc, int64_t n,
                              float ground_z, const float* background /* host [3] */,
                              const float* background_linear /* host [3] */, const float* g, const int32_t* pos,
                              const float* vis_list, int32_t vis_kind, const float* without_bg, float* with_bg,
                              float* shadow /* or NULL */, int64_t out_rows, int64_t row0, void* stream);

/* ---- mesh export: marching cubes over a dense volume (utils.py:165-225, skimage.measure.marching_cubes on
 * TensorBase.getDenseAlpha(), tensorBase_rotated_lights.py:737-753) ---------------------------------------------------
 * volume [X,Y,Z] fp32 C-contiguous, X, Y, Z >= 2 and X*Y*Z <= INT32_MAX (TIR_ERR_SHAPE otherwise).  A point is inside
 * iff v > level; the topology, vertex placement and winding are documented in csrc/tir_mc_body.h.
 *   tir_marching_cubes_work_size  bytes of the caller's scratch `work` for an X x Y x Z volume;
 *   tir_marching_cubes_count      totals[2] (device, int64, overwritten) = vertex and triangle counts; fills `work`;
 *   tir_marching_cubes_emit       with the same volume, level and work: verts [n_verts,3] fp32 = (axis0, axis1, axis2)
 *                                 coordinates scaled by (sx, sy, sz), faces [n_faces,3] int32.  n_verts / n_faces are
 *                                 the counts read back from totals; a count above INT32_MAX is TIR_ERR_SHAPE.
 * Vertices are ordered by (grid-point linear index, axis), faces by (cell linear index, loop order): reruns are
 * bit-identical. */
int tir_marching_cubes_work_size(int32_t X, int32_t Y, int32_t Z, int64_t* bytes);
int tir_marching_cubes_count(const float* volume, int32_t X, int32_t Y, int32_t Z, float level, void* work,
                             int64_t work_bytes, int64_t* totals, void* stream);
int tir_marching_cubes_emit(const float* volume, int32_t X, int32_t Y, int32_t Z, float level, double sx, double sy,
                            double sz, const void* work, int64_t work_bytes, int64_t n_verts, int64_t n_faces,
                            float* verts, int32_t* faces, void* stream);

/* ---- textured glTF export: the texture atlas of a marching-cubes mesh (tensoir_b200/gltf.py) -----------------------
 * faces [F,3] int32 in marching_cubes' winding (reversed here, as the PLY writes them), v [V,3] fp32 the field
 * positions of the vertices, a T x T atlas (T a power of two in [256, 8192]) of s x s cells (s in [6, 64],
 * floor(T/s)^2 >= ceil(F/2)); the layout, the no-bleed guarantee, the probe points, the tangent frames and the
 * encoding are documented in csrc/tir_atlas_body.h.  Texels are numbered face-major, F * s(s-1)/2 in all (int64).
 *   tir_atlas_texels   texels [first, first+n): pix [n] int32 = row * T + column, pos [n,3] fp32 the texel's point on
 *                      its face (clamped barycentrics of its corners' v);
 *   tir_atlas_encode   the same texels with their probe results (albedo [n,3], rough [n], normal [n,3], probed [n]
 *                      uint8): one RGBA8 word per texel into base_color, metallic_roughness and normal_map [T,T,4];
 *                      other texels are not written;
 *   tir_atlas_corners  per face corner, unwelded (row 3f+k = corner k of face f): position [3F,3] = v, normal [3F,3]
 *                      and tangent [3F,4] the face's frame, texcoord [3F,2] its UV.
 * One thread per texel / face, no atomics: repeated calls give identical bits.  n = 0 (F = 0 for the corners) is a
 * no-op; TIR_ERR_SHAPE for a negative size, a layout outside the ranges above or a texel range past the last texel. */
int tir_atlas_texels(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s, int64_t first,
                     int64_t n, int32_t* pix, float* pos, void* stream);
int tir_atlas_encode(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s, int64_t first,
                     int64_t n, const float* albedo, const float* rough, const float* normal, const uint8_t* probed,
                     uint8_t* base_color, uint8_t* metallic_roughness, uint8_t* normal_map, void* stream);
int tir_atlas_corners(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s, float* position,
                      float* normal, float* tangent, float* texcoord, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TENSOIR_B200_H */
