// Host twin of csrc/tir_atlas.cu for the CPU tests of tensoir_b200/gltf.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (the at_*_check functions) and per-texel / per-face math
// of csrc/tir_atlas_body.h, with plain loops instead of kernels.  "Device" pointers are host pointers here.
#include <string.h>
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_atlas_body.h"

extern "C" int tir_atlas_texels(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s,
                                int64_t first, int64_t n, int32_t* pix, float* pos, void*) {
  const int rc = at_texels_check(faces, n_faces, v, T, s, first, n, pix, pos);
  if (rc <= 0) return rc;
  for (int64_t i = 0; i < n; ++i) {
    const AtTexel tx = at_texel(first + i, T, s);
    int32_t c[3];
    at_corners(faces, tx.face, c);
    float b[3];
    at_bary(s, tx.ia, tx.ja, b);
    at_point(v, c, b, pos + i * 3);
    pix[i] = tx.y * T + tx.x;
  }
  return TIR_OK;
}

extern "C" int tir_atlas_encode(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s,
                                int64_t first, int64_t n, const float* albedo, const float* rough,
                                const float* normal, const uint8_t* probed, uint8_t* base_color,
                                uint8_t* metallic_roughness, uint8_t* normal_map, void*) {
  const int rc = at_encode_check(faces, n_faces, v, T, s, first, n, albedo, rough, normal, probed, base_color,
                                 metallic_roughness, normal_map);
  if (rc <= 0) return rc;
  uint8_t* img[3] = {base_color, metallic_roughness, normal_map};
  for (int64_t i = 0; i < n; ++i) {
    const AtTexel tx = at_texel(first + i, T, s);
    int32_t c[3];
    at_corners(faces, tx.face, c);
    const AtFrame fr = at_frame(v, c, tx.face & 1);
    uint32_t w[3];
    at_encode(fr, albedo + i * 3, rough[i], normal + i * 3, probed[i] != 0, w);
    const int64_t px = (int64_t)tx.y * T + tx.x;
    for (int k = 0; k < 3; ++k) memcpy(img[k] + px * 4, &w[k], 4);
  }
  return TIR_OK;
}

extern "C" int tir_atlas_corners(const int32_t* faces, int64_t n_faces, const float* v, int32_t T, int32_t s,
                                 float* position, float* normal, float* tangent, float* texcoord, void*) {
  const int rc = at_corners_check(faces, n_faces, v, T, s, position, normal, tangent, texcoord);
  if (rc <= 0) return rc;
  for (int64_t f = 0; f < n_faces; ++f) {
    int32_t c[3];
    at_corners(faces, f, c);
    const AtFrame fr = at_frame(v, c, f & 1);
    float uv[3][2];
    at_corner_uv(f, T, s, uv);
    for (int k = 0; k < 3; ++k) {
      const int64_t r = f * 3 + k;
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
  return TIR_OK;
}

// the frame of face f for the tangent-frame tests: n[3], t[3], w; returns 1 for a degenerate face
extern "C" int at_host_frame(const int32_t* faces, int64_t f, const float* v, float* out) {
  int32_t c[3];
  at_corners(faces, f, c);
  const AtFrame fr = at_frame(v, c, f & 1);
  for (int d = 0; d < 3; ++d) {
    out[d] = fr.n[d];
    out[3 + d] = fr.t[d];
  }
  out[6] = fr.w;
  return fr.degenerate ? 1 : 0;
}
