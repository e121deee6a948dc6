// Host twin of csrc/tir_mesh.cu for the CPU tests of tensoir_b200/mesh.py: the SAME C-ABI signatures
// (include/tensoir_b200.h), the library's own argument checks (the mc_*_check functions), scratch layout and per-cell /
// per-vertex math of csrc/tir_mc_body.h, with plain loops instead of kernels.  The scratch has no CUB part here, so its
// size check is this build's own.  "Device" pointers are host pointers here.  mc_host_cell exposes the polygonisation
// of one cell for the all-configurations test.
#include <string.h>
#include "../include/tensoir_b200.h"
#include "../tensoir_b200/csrc/tir_mc_body.h"

extern "C" int mc_host_cell(int32_t mask, int32_t connected, int8_t* tri) {
  return mc_cell_triangles((unsigned)mask, (unsigned)connected, tri);
}

extern "C" int mc_host_face_connected(float v00, float v10, float v01, float v11, float level) {
  return mc_face_connected(v00, v10, v01, v11, level) ? 1 : 0;
}

extern "C" int tir_marching_cubes_work_size(int32_t X, int32_t Y, int32_t Z, int64_t* bytes) {
  const int rc = mc_work_size_check(X, Y, Z, bytes);
  if (rc < 0) return rc;
  *bytes = mc_work_layout((int64_t)X * Y * Z, 0).total;
  return TIR_OK;
}

static void corners(const float* vol, int64_t cell, int32_t Y, int32_t Z, float c[8], int64_t pt[8]) {
  for (int r = 0; r < 8; ++r) {
    pt[r] = cell + (r & 1) * (int64_t)Y * Z + (r >> 1 & 1) * (int64_t)Z + (r >> 2);
    c[r] = vol[pt[r]];
  }
}

extern "C" int tir_marching_cubes_count(const float* volume, int32_t X, int32_t Y, int32_t Z, float level, void* work,
                                        int64_t work_bytes, int64_t* totals, void*) {
  const int rc = mc_count_check(volume, X, Y, Z, work, totals);
  if (rc < 0) return rc;
  const int64_t n = (int64_t)X * Y * Z;
  const McWork w = mc_work_layout(n, 0);
  if (work_bytes < w.total) return TIR_ERR_CAPACITY;
  uint8_t* base = (uint8_t*)work;
  uint8_t* bits = base + w.bits;
  uint8_t* tris = base + w.tris;
  int32_t* voff = (int32_t*)(base + w.voff);
  int32_t* toff = (int32_t*)(base + w.toff);
  int32_t* active = (int32_t*)(base + w.active);
  int64_t nv = 0, nt = 0, na = 0;
  for (int32_t i = 0; i < X; ++i)
    for (int32_t j = 0; j < Y; ++j)
      for (int32_t k = 0; k < Z; ++k) {
        const int64_t p = ((int64_t)i * Y + j) * Z + k;
        const bool in = mc_inside(volume[p], level);
        unsigned b = 0;
        if (i + 1 < X && mc_inside(volume[p + (int64_t)Y * Z], level) != in) b |= 1;
        if (j + 1 < Y && mc_inside(volume[p + Z], level) != in) b |= 2;
        if (k + 1 < Z && mc_inside(volume[p + 1], level) != in) b |= 4;
        int t = 0;
        if (i + 1 < X && j + 1 < Y && k + 1 < Z) {
          float c[8];
          int64_t pt[8];
          corners(volume, p, Y, Z, c, pt);
          const unsigned m = mc_cell_mask(c, level);
          if (m != 0 && m != 255) t = mc_cell_triangles(m, mc_face_decisions(c, m, level), nullptr);
        }
        bits[p] = (uint8_t)b;
        tris[p] = (uint8_t)t;
        voff[p] = (int32_t)nv;            // the device scans are int32 too; emit rejects totals above INT32_MAX
        toff[p] = (int32_t)nt;
        if (t) active[na++] = (int32_t)p;
        nv += (b & 1) + (b >> 1 & 1) + (b >> 2);
        nt += t;
      }
  *(int32_t*)(base + w.n_active) = (int32_t)na;
  totals[0] = nv;
  totals[1] = nt;
  return TIR_OK;
}

extern "C" int tir_marching_cubes_emit(const float* volume, int32_t X, int32_t Y, int32_t Z, float level, double sx,
                                       double sy, double sz, const void* work, int64_t work_bytes, int64_t n_verts,
                                       int64_t n_faces, float* verts, int32_t* faces, void*) {
  const int rc = mc_emit_check(volume, X, Y, Z, work, n_verts, n_faces, verts, faces);
  if (rc < 0) return rc;
  const int64_t n = (int64_t)X * Y * Z;
  const McWork w = mc_work_layout(n, 0);
  if (work_bytes < w.total) return TIR_ERR_CAPACITY;
  const uint8_t* base = (const uint8_t*)work;
  const uint8_t* bits = base + w.bits;
  const int32_t* voff = (const int32_t*)(base + w.voff);
  const int32_t* toff = (const int32_t*)(base + w.toff);
  const int32_t* active = (const int32_t*)(base + w.active);
  const int32_t n_active = *(const int32_t*)(base + w.n_active);
  const double sp[3] = {sx, sy, sz};
  const int64_t stride[3] = {(int64_t)Y * Z, (int64_t)Z, 1};
  for (int64_t q = 0; q < n; ++q) {
    const unsigned b = bits[q];
    if (!b) continue;
    const int64_t idx[3] = {q / stride[0], (q / Z) % Y, q % Z};
    int64_t row = voff[q];
    for (int a = 0; a < 3; ++a) {
      if (!(b >> a & 1)) continue;
      if (row < n_verts)
        for (int c = 0; c < 3; ++c)
          verts[row * 3 + c] = c == a ? mc_edge_coord(idx[c], volume[q], volume[q + stride[a]], level, sp[c])
                                      : mc_grid_coord(idx[c], sp[c]);
      ++row;
    }
  }
  for (int32_t q = 0; q < n_active; ++q) {
    float c[8];
    int64_t pt[8];
    corners(volume, active[q], Y, Z, c, pt);
    const unsigned m = mc_cell_mask(c, level);
    int8_t tri[3 * MC_MAX_TRIS];
    const int nt = mc_cell_triangles(m, mc_face_decisions(c, m, level), tri);
    const int64_t row0 = toff[active[q]];
    for (int t = 0; t < nt && row0 + t < n_faces; ++t)
      for (int s = 0; s < 3; ++s) {
        const int e = tri[3 * t + s], a = e >> 2;
        const int64_t v = pt[mc_edge_corner(e)];
        faces[(row0 + t) * 3 + s] = voff[v] + __builtin_popcount(bits[v] & ((1u << a) - 1u));
      }
  }
  return TIR_OK;
}
