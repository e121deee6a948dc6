// The texture atlas of the textured glTF export (tensoir_b200/gltf.py): its layout, the probe point of every texel,
// the per-face tangent frames and the bytes of the three images.  Shared by the CUDA kernels (tir_atlas.cu) and the
// host twin (tests/host_atlas.cpp), so that both give identical bits; every fp32 product, sum and quotient goes
// through the exactly rounded ev_* helpers of tir_eval_body.h, in a fixed order, never fused.
//
// Faces.  Face f's corners c0, c1, c2 are faces[f] reversed (the PLY's winding, mesh.face_records): the right-hand
// normal of (c0, c1, c2) points out of the dense region.  v [V,3] are the field positions of mesh.asset_surface.
//
// Image.  T x T texels, T a power of two in [256, 8192].  Texel (i, j) is column i and row j; row 0 is the top row of
// the PNG; its centre has UV ((i + 0.5) / T, (j + 0.5) / T) (glTF's top-left origin).
//
// Cells.  Faces 2c (face A) and 2c+1 (face B) share cell c, an s x s block with its origin at texel
// (s (c mod P), s (c div P)), P = floor(T / s).  s is the largest value <= 64 with P^2 >= ceil(F/2) (chosen by
// gltf.atlas_cell_size; the entry points accept any s in [6, 64] whose cells fit).  In cell-local texel-centre
// coordinates, with L = s - 3:
//   face A: c0, c1, c2 at (0, 0), (L, 0), (0, L);           owns the texels with i + j <= s - 2;
//   face B: c0, c1, c2 at (s-1, s-1), (2, s-1), (s-1, 2);   owns the texels with i + j >= s,
// so B is A turned by 180 degrees, (i, j) -> (s-1-i, s-1-j), and the diagonal i + j = s - 1 belongs to neither.  Each
// face owns q = s (s-1) / 2 texels, F q in all.
//
// No-bleed guarantee.  A bilinear lookup (no mipmaps) at any point of a face's UV triangle gives non-zero weight only
// to texels that face owns.  In A's frame a point (x, y) of the triangle has x, y >= 0 and x + y <= L; the texels with
// non-zero weight are (floor(x) + dx, floor(y) + dy) with dx = 1 only when x is not an integer, and the same for y.
// They have i, j >= 0 and i + j <= L + 1 = s - 2: when both fractions are non-zero, floor(x) + floor(y) < x + y <= L,
// so floor(x) + floor(y) <= L - 1.  So no texel of another cell, no texel of the other face and no diagonal texel is
// read.  Mipmaps average across cells and break the guarantee.
//
// Texel -> probe point.  A texel's barycentrics are its position in A's frame (B's texels turned into it) over the
// triangle, clamped to the triangle's nearest point in texel units: inside, (1 - (x+y)/L, x/L, y/L); beyond the
// hypotenuse (x + y = L + 1 for owned texels) the point ((x - y + L) / 2, (y - x + L) / 2), clamped to [0, L] along it.
// All of them are integer numerators over 2L, divided once: a corner texel has b = (1, 0, 0) exactly and lands on its
// vertex bit for bit.  The position is (b0 v[c0] + b1 v[c1]) + b2 v[c2].
//
// Tangent frame of a face (glTF NORMAL and TANGENT, and the normal map's basis).  N = normalize(e1 x e2) with
// e1 = v[c1] - v[c0], e2 = v[c2] - v[c0]; dP/du is e1 on face A and -e1 on face B (and dP/dv is +-e2), so
// T = normalize(dP/du - (dP/du . N) N), and w = +-1 makes cross(N, T) w point along -dP/dv, the image's "up" (glTF's +Y
// for normal maps).  A face whose fp32 cross product has zero length (or a zero tangent) is degenerate and gets
// N = (0,0,1), T = (1,0,0), w = 1.
//
// Encoding (RGBA8, alpha 255; unowned texels keep the caller's defaults).
//   base colour        the sRGB OETF of the linear albedo (IEC 61966-2-1), rounded to the nearest 8-bit code: the
//                      code is the number of thresholds EOTF((k - 0.5) / 255), k = 1..255, at or below the albedo,
//                      each threshold rounded up to fp32 (so the comparison is exact for an fp32 albedo);
//   metallic-roughness R = 255, G = roughness, B = 0 (metallic 0); glTF and tir_ggx.h both use alpha = roughness^2;
//   normal             the normal in (T, cross(N, T) w, N), normalised, as x 0.5 + 0.5 (a negative z as it is);
// where an fp32 value v in [0, 1] becomes floor(v 255 + 0.5) (clamped to [0, 1] first, NaN as 0) and a texel that is
// not probed encodes probe()'s fallback material, albedo 0 and roughness 1.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/tensoir_b200.h"
#include "tir_eval_body.h"

#if defined(__CUDACC__)
#define AT_HD __host__ __device__ __forceinline__
#define AT_D __device__ __forceinline__      // reads the sRGB table, which lives in device memory
#define AT_TABLE __device__ const            // global memory: the bisection's indices diverge across a warp
#else
#define AT_HD inline
#define AT_D inline
#define AT_TABLE static const
#endif

#define AT_T_MIN 256
#define AT_T_MAX 8192
#define AT_S_MIN 6
#define AT_S_MAX 64

// texels owned by each face of a cell of size s
AT_HD int at_face_texels(int s) { return s * (s - 1) / 2; }

// TIR_OK when F faces fit a T x T atlas of cells of size s
inline int at_validate_layout(int64_t F, int32_t T, int32_t s) {
  if (F < 0 || F > INT32_MAX) return TIR_ERR_SHAPE;
  if (T < AT_T_MIN || T > AT_T_MAX || (T & (T - 1))) return TIR_ERR_SHAPE;
  if (s < AT_S_MIN || s > AT_S_MAX) return TIR_ERR_SHAPE;
  const int64_t P = T / s;
  return P * P >= (F + 1) / 2 ? TIR_OK : TIR_ERR_SHAPE;
}

// TIR_OK for a texel range [first, first + n) inside the F q texels of the layout
inline int at_validate_range(int64_t F, int32_t s, int64_t first, int64_t n) {
  if (first < 0 || n < 0) return TIR_ERR_SHAPE;
  return first + n <= F * at_face_texels(s) ? TIR_OK : TIR_ERR_SHAPE;
}

// The whole argument check of each entry, run by tir_atlas.cu and its host build before their launch / loop:
// 1 run, 0 nothing to do, < 0 TirStatus
inline int at_texels_check(const int32_t* faces, int64_t F, const float* v, int32_t T, int32_t s, int64_t first,
                           int64_t n, const int32_t* pix, const float* pos) {
  int rc = at_validate_layout(F, T, s);
  if (!rc) rc = at_validate_range(F, s, first, n);
  if (rc || n == 0) return rc;
  if (!faces || !v || !pix || !pos) return TIR_ERR_NULL;
  return 1;
}

inline int at_encode_check(const int32_t* faces, int64_t F, const float* v, int32_t T, int32_t s, int64_t first,
                           int64_t n, const float* albedo, const float* rough, const float* normal,
                           const uint8_t* probed, const uint8_t* base_color, const uint8_t* metallic_roughness,
                           const uint8_t* normal_map) {
  int rc = at_validate_layout(F, T, s);
  if (!rc) rc = at_validate_range(F, s, first, n);
  if (rc || n == 0) return rc;
  if (!faces || !v || !albedo || !rough || !normal || !probed || !base_color || !metallic_roughness || !normal_map)
    return TIR_ERR_NULL;
  return 1;
}

inline int at_corners_check(const int32_t* faces, int64_t F, const float* v, int32_t T, int32_t s,
                            const float* position, const float* normal, const float* tangent, const float* texcoord) {
  const int rc = at_validate_layout(F, T, s);
  if (rc || F == 0) return rc;
  if (!faces || !v || !position || !normal || !tangent || !texcoord) return TIR_ERR_NULL;
  return 1;
}

// Texel t of the face-major enumeration: face t / q, then its owned texels by anti-diagonal d = i + j of A's frame
// and by i along it.  -> face, A-frame (ia, ja), image texel (x, y).
struct AtTexel {
  int64_t face;
  int ia, ja;
  int x, y;
};

AT_HD AtTexel at_texel(int64_t t, int32_t T, int32_t s) {
  const int q = at_face_texels(s);
  AtTexel r;
  r.face = t / q;
  const int k = (int)(t - r.face * q);
  int d = (int)((sqrtf(8.f * (float)k + 1.f) - 1.f) * 0.5f);
  while ((d + 1) * (d + 2) / 2 <= k) ++d;
  while (d * (d + 1) / 2 > k) --d;
  r.ia = k - d * (d + 1) / 2;
  r.ja = d - r.ia;
  const bool b = r.face & 1;
  const int64_t c = r.face >> 1;
  const int P = T / s;
  r.x = (int)(c % P) * s + (b ? s - 1 - r.ia : r.ia);
  r.y = (int)(c / P) * s + (b ? s - 1 - r.ja : r.ja);
  return r;
}

// the UVs of face f's corners c0, c1, c2: texel centres ((x + 0.5) / T, (y + 0.5) / T), exact in fp32
AT_HD void at_corner_uv(int64_t f, int32_t T, int32_t s, float uv[3][2]) {
  const int L = s - 3, P = T / s;
  const int64_t c = f >> 1;
  const int ox = (int)(c % P) * s, oy = (int)(c / P) * s;
  const int ca[3][2] = {{0, 0}, {L, 0}, {0, L}};
  for (int k = 0; k < 3; ++k) {
    const int x = ox + ((f & 1) ? s - 1 - ca[k][0] : ca[k][0]);
    const int y = oy + ((f & 1) ? s - 1 - ca[k][1] : ca[k][1]);
    uv[k][0] = ev_div(ev_add((float)x, 0.5f), (float)T);
    uv[k][1] = ev_div(ev_add((float)y, 0.5f), (float)T);
  }
}

// the corners c0, c1, c2 of face f (faces[f] reversed)
AT_HD void at_corners(const int32_t* faces, int64_t f, int32_t c[3]) {
  c[0] = faces[f * 3 + 2];
  c[1] = faces[f * 3 + 1];
  c[2] = faces[f * 3 + 0];
}

// clamped barycentrics of A-frame texel (ia, ja)
AT_HD void at_bary(int s, int ia, int ja, float b[3]) {
  const int L = s - 3;
  int n1, n2;
  if (ia + ja <= L) {
    n1 = 2 * ia;
    n2 = 2 * ja;
  } else {
    n1 = ia - ja + L;
    n1 = n1 < 0 ? 0 : (n1 > 2 * L ? 2 * L : n1);
    n2 = 2 * L - n1;
  }
  const float den = (float)(2 * L);
  b[0] = ev_div((float)(2 * L - n1 - n2), den);
  b[1] = ev_div((float)n1, den);
  b[2] = ev_div((float)n2, den);
}

// the field position of barycentrics b on corners c of positions v
AT_HD void at_point(const float* v, const int32_t c[3], const float b[3], float p[3]) {
  for (int k = 0; k < 3; ++k)
    p[k] = ev_add(ev_add(ev_mul(b[0], v[(int64_t)c[0] * 3 + k]), ev_mul(b[1], v[(int64_t)c[1] * 3 + k])),
                  ev_mul(b[2], v[(int64_t)c[2] * 3 + k]));
}

AT_HD void at_cross(const float a[3], const float b[3], float c[3]) {
  c[0] = ev_sub(ev_mul(a[1], b[2]), ev_mul(a[2], b[1]));
  c[1] = ev_sub(ev_mul(a[2], b[0]), ev_mul(a[0], b[2]));
  c[2] = ev_sub(ev_mul(a[0], b[1]), ev_mul(a[1], b[0]));
}

AT_HD float at_dot(const float a[3], const float b[3]) {
  return ev_add(ev_add(ev_mul(a[0], b[0]), ev_mul(a[1], b[1])), ev_mul(a[2], b[2]));
}

// a / |a| -> false (a untouched) when |a| is 0 or not finite
AT_HD bool at_unit(float a[3]) {
  const float len = sqrtf(at_dot(a, a));
  if (!(len > 0.f) || !(len < INFINITY)) return false;
  for (int k = 0; k < 3; ++k) a[k] = ev_div(a[k], len);
  return true;
}

struct AtFrame {
  float n[3], t[3], w;
  bool degenerate;
};

// the tangent frame of face f (side = f & 1)
AT_HD AtFrame at_frame(const float* v, const int32_t c[3], bool side) {
  AtFrame fr;
  float e1[3], e2[3];
  for (int k = 0; k < 3; ++k) {
    e1[k] = ev_sub(v[(int64_t)c[1] * 3 + k], v[(int64_t)c[0] * 3 + k]);
    e2[k] = ev_sub(v[(int64_t)c[2] * 3 + k], v[(int64_t)c[0] * 3 + k]);
  }
  at_cross(e1, e2, fr.n);
  bool ok = at_unit(fr.n);
  if (ok) {
    float du[3], dv[3];
    for (int k = 0; k < 3; ++k) {
      du[k] = side ? -e1[k] : e1[k];
      dv[k] = side ? -e2[k] : e2[k];
    }
    const float d = at_dot(du, fr.n);
    for (int k = 0; k < 3; ++k) fr.t[k] = ev_sub(du[k], ev_mul(d, fr.n[k]));
    ok = at_unit(fr.t);
    if (ok) {
      float bt[3];
      at_cross(fr.n, fr.t, bt);
      fr.w = at_dot(bt, dv) > 0.f ? -1.f : 1.f;
    }
  }
  fr.degenerate = !ok;
  if (!ok) {
    fr.n[0] = 0.f; fr.n[1] = 0.f; fr.n[2] = 1.f;
    fr.t[0] = 1.f; fr.t[1] = 0.f; fr.t[2] = 0.f;
    fr.w = 1.f;
  }
  return fr;
}

// floor(clamp(v, 0, 1) 255 + 0.5), NaN as 0
AT_HD uint32_t at_unorm8(float v) {
  v = v > 0.f ? (v < 1.f ? v : 1.f) : 0.f;
  return (uint32_t)ev_add(ev_mul(v, 255.f), 0.5f);
}

// fp32 thresholds of the sRGB codes 1..255: EOTF((k - 0.5) / 255) rounded up to fp32
AT_TABLE float kAtSrgbThreshold[255] = {
    1.517635e-04f, 4.552905e-04f, 7.588175e-04f, 1.0623445e-03f, 1.3658715e-03f, 1.6693985e-03f, 1.9729256e-03f,
    2.2764525e-03f, 2.5799794e-03f, 2.8835065e-03f, 3.188301e-03f, 3.5092595e-03f, 3.848315e-03f, 4.2057484e-03f,
    4.581833e-03f, 4.9768374e-03f, 5.3910245e-03f, 5.824651e-03f, 6.2779696e-03f, 6.7512277e-03f, 7.2446684e-03f,
    7.758531e-03f, 8.2930485e-03f, 8.848454e-03f, 9.424971e-03f, 1.00228265e-02f, 1.0642237e-02f, 1.1283422e-02f,
    1.19465925e-02f, 1.263196e-02f, 1.3339732e-02f, 1.4070112e-02f, 1.4823304e-02f, 1.5599503e-02f, 1.639891e-02f,
    1.7221717e-02f, 1.8068116e-02f, 1.8938296e-02f, 1.9832443e-02f, 2.0750746e-02f, 2.1693384e-02f, 2.2660539e-02f,
    2.3652392e-02f, 2.4669116e-02f, 2.5710888e-02f, 2.6777884e-02f, 2.7870271e-02f, 2.8988222e-02f, 3.0131903e-02f,
    3.1301484e-02f, 3.2497123e-02f, 3.371899e-02f, 3.4967244e-02f, 3.6242045e-02f, 3.7543554e-02f, 3.887193e-02f,
    4.022732e-02f, 4.160989e-02f, 4.3019786e-02f, 4.4457164e-02f, 4.5922175e-02f, 4.7414966e-02f, 4.893569e-02f,
    5.0484486e-02f, 5.206151e-02f, 5.36669e-02f, 5.5300802e-02f, 5.696336e-02f, 5.8654718e-02f, 6.0375012e-02f,
    6.2124386e-02f, 6.3902974e-02f, 6.571092e-02f, 6.754836e-02f, 6.941541e-02f, 7.131224e-02f, 7.323896e-02f,
    7.519571e-02f, 7.718262e-02f, 7.919982e-02f, 8.124745e-02f, 8.3325624e-02f, 8.543449e-02f, 8.757416e-02f,
    8.974477e-02f, 9.1946445e-02f, 9.41793e-02f, 9.644348e-02f, 9.8739095e-02f, 1.0106628e-01f, 1.0342514e-01f,
    1.05815805e-01f, 1.0823841e-01f, 1.1069305e-01f, 1.1317987e-01f, 1.1569897e-01f, 1.1825049e-01f, 1.2083452e-01f,
    1.234512e-01f, 1.2610064e-01f, 1.2878296e-01f, 1.3149826e-01f, 1.3424668e-01f, 1.370283e-01f, 1.3984329e-01f,
    1.4269169e-01f, 1.4557366e-01f, 1.4848931e-01f, 1.5143874e-01f, 1.5442206e-01f, 1.574394e-01f, 1.6049084e-01f,
    1.635765e-01f, 1.666965e-01f, 1.6985095e-01f, 1.7303993e-01f, 1.7626357e-01f, 1.7952198e-01f, 1.8281525e-01f,
    1.861435e-01f, 1.8950684e-01f, 1.9290535e-01f, 1.9633916e-01f, 1.9980836e-01f, 2.0331305e-01f, 2.0685335e-01f,
    2.1042934e-01f, 2.1404114e-01f, 2.1768886e-01f, 2.2137257e-01f, 2.250924e-01f, 2.2884843e-01f, 2.3264077e-01f,
    2.3646952e-01f, 2.4033478e-01f, 2.4423665e-01f, 2.4817522e-01f, 2.521506e-01f, 2.5616285e-01f, 2.6021212e-01f,
    2.642985e-01f, 2.6842204e-01f, 2.725829e-01f, 2.767811e-01f, 2.8101683e-01f, 2.852901e-01f, 2.8960103e-01f,
    2.9394975e-01f, 2.983363e-01f, 3.027608e-01f, 3.0722338e-01f, 3.1172407e-01f, 3.1626296e-01f, 3.208402e-01f,
    3.2545584e-01f, 3.3011e-01f, 3.3480275e-01f, 3.395342e-01f, 3.4430438e-01f, 3.4911346e-01f, 3.539615e-01f,
    3.5884857e-01f, 3.637748e-01f, 3.6874023e-01f, 3.73745e-01f, 3.7878916e-01f, 3.8387278e-01f, 3.88996e-01f,
    3.941589e-01f, 3.9936155e-01f, 4.0460402e-01f, 4.0988642e-01f, 4.1520885e-01f, 4.2057136e-01f, 4.2597407e-01f,
    4.3141705e-01f, 4.3690038e-01f, 4.4242412e-01f, 4.4798842e-01f, 4.5359334e-01f, 4.5923892e-01f, 4.6492532e-01f,
    4.7065255e-01f, 4.7642073e-01f, 4.8222995e-01f, 4.8808026e-01f, 4.9397177e-01f, 4.9990457e-01f, 5.0587875e-01f,
    5.1189435e-01f, 5.179514e-01f, 5.240502e-01f, 5.301906e-01f, 5.363727e-01f, 5.4259676e-01f, 5.488627e-01f,
    5.5517066e-01f, 5.615207e-01f, 5.6791294e-01f, 5.743474e-01f, 5.8082414e-01f, 5.8734334e-01f, 5.9390503e-01f,
    6.005093e-01f, 6.0715616e-01f, 6.1384577e-01f, 6.2057817e-01f, 6.273534e-01f, 6.3417166e-01f, 6.4103293e-01f,
    6.479373e-01f, 6.548849e-01f, 6.6187567e-01f, 6.6890985e-01f, 6.759874e-01f, 6.8310845e-01f, 6.902731e-01f,
    6.974814e-01f, 7.047334e-01f, 7.1202916e-01f, 7.193689e-01f, 7.2675246e-01f, 7.341801e-01f, 7.4165183e-01f,
    7.4916774e-01f, 7.567279e-01f, 7.643323e-01f, 7.719812e-01f, 7.796745e-01f, 7.8741235e-01f, 7.951948e-01f,
    8.030219e-01f, 8.1089383e-01f, 8.188106e-01f, 8.267722e-01f, 8.3477885e-01f, 8.4283054e-01f, 8.509273e-01f,
    8.590693e-01f, 8.672565e-01f, 8.754891e-01f, 8.837671e-01f, 8.9209056e-01f, 9.004596e-01f, 9.088742e-01f,
    9.1733456e-01f, 9.258407e-01f, 9.343926e-01f, 9.429904e-01f, 9.516342e-01f, 9.6032405e-01f, 9.6906e-01f,
    9.7784215e-01f, 9.8667055e-01f, 9.9554527e-01f};

// the 8-bit sRGB code of linear value c (NaN and c < threshold[1] give 0)
AT_D uint32_t at_srgb8(float c) {
  int lo = 0, hi = 255;           // code = number of thresholds <= c, found by bisection
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (c >= kAtSrgbThreshold[mid - 1]) lo = mid;
    else hi = mid - 1;
  }
  return (uint32_t)lo;
}

AT_HD uint32_t at_rgba(uint32_t r, uint32_t g, uint32_t b) { return r | g << 8 | b << 16 | 0xFF000000u; }

// the three RGBA8 words of one texel: base colour, metallic-roughness and normal
AT_D void at_encode(const AtFrame& fr, const float albedo[3], float rough, const float normal[3], bool probed,
                     uint32_t out[3]) {
  const float a0 = probed ? albedo[0] : 0.f, a1 = probed ? albedo[1] : 0.f, a2 = probed ? albedo[2] : 0.f;
  out[0] = at_rgba(at_srgb8(a0), at_srgb8(a1), at_srgb8(a2));
  out[1] = at_rgba(255u, at_unorm8(probed ? rough : 1.f), 0u);
  float bt[3], local[3], unit[3];
  at_cross(fr.n, fr.t, bt);
  for (int k = 0; k < 3; ++k) bt[k] = ev_mul(bt[k], fr.w);
  local[0] = at_dot(normal, fr.t);
  local[1] = at_dot(normal, bt);
  local[2] = at_dot(normal, fr.n);
  ev_normalize(local, unit);
  uint32_t e[3];
  for (int k = 0; k < 3; ++k) e[k] = at_unorm8(ev_add(ev_mul(unit[k], 0.5f), 0.5f));
  out[2] = at_rgba(e[0], e[1], e[2]);
}
