// Per-cell math of the marching-cubes surface extraction (tir_marching_cubes_*, csrc/tir_mesh.cu), the native path
// of the reference's mesh export (utils.py:165-225, skimage.measure.marching_cubes on getDenseAlpha()).  Shared by the
// CUDA kernels and by a host build (tests/host_mesh.cpp) that the CPU tests drive through the same C ABI.
//
// Decisions, fixed here for both builds:
//  - Layout.  The volume is [X,Y,Z] fp32, C-contiguous (what getDenseAlpha returns): point (i,j,k) is element
//    (i*Y + j)*Z + k, and array axis 0 is x.  Vertex coordinates come out in (axis0, axis1, axis2) order.  X, Y and Z are
//    independent (never assumed equal).  Cell (i,j,k) spans points (i..i+1, j..j+1, k..k+1) and is numbered by the
//    linear index of its lowest point.
//  - Inside test.  A point is inside iff v > level, so a NaN point is outside.
//  - Vertices.  One per grid edge whose endpoints lie on different sides; the cells around an edge share its vertex.
//    Vertices are numbered by (linear index of the edge's lower point, axis of the edge).
//  - Vertex position.  t = (level - v_lo) / (v_hi - v_lo) with v_lo the endpoint of lower index; the coordinate along the
//    edge is (i + t) * spacing, the other two are i * spacing.  Evaluated in fp64 with every operation rounded on its own
//    (no FMA contraction) and rounded to fp32 once, so the device and a host build agree bit for bit.  An edge with a
//    NaN endpoint gets a NaN coordinate.
//  - Face ambiguity.  A face whose inside corners lie on one diagonal only is resolved with the asymptotic decider:
//    the saddle value of the bilinear face interpolant, (v00 v11 - v10 v01) / (v00 + v11 - v10 - v01), against level;
//    saddle > level connects the inside corners across the face.  It is evaluated in fp32 with the four values in a
//    canonical order, v_uw for the offsets (u, w) along the face's two axes (lower axis first) in global grid
//    coordinates, so the two cells that share the face take the same decision and the mesh stays watertight.
//    This is the decider skimage's Lewiner method applies to faces.
//  - Triangles.  Each face gives 0, 1 or 2 segments between its crossed edges.  Walking the face's corners
//    counter-clockwise about the cell's outward face normal, a crossed edge is an entry (outside -> inside) or an exit;
//    every segment runs from an entry to an exit, which puts the inside corners on its right.  A two-crossing face has
//    one segment; on an ambiguous face an entry pairs with the next exit of the walk when the inside corners are
//    separated and with the previous one when they are connected.  Each crossed edge of the cell borders two of its
//    faces and is the entry of one and the exit of the other, so the segments chain into closed loops, each followed
//    from its lowest edge id.  A loop of k vertices becomes k-2 triangles, in clipping order, by ear clipping: cut off the
//    first vertex after the loop's first one whose two neighbours may be joined (mc_chord_allowed), until three
//    remain.  Where every join is allowed this is the fan from the loop's first vertex.  The rule keeps the mesh
//    closed: a join inside a face shared with a neighbour is open to only one of the two cells (a fan alone would
//    let both cells of an ambiguous face join the same two vertices).  Checked for every loop of every
//    (corner pattern, face decisions) configuration by the CPU tests.  No triangle table.
//  - No interior ambiguity test.  The tunnel configurations Lewiner's method resolves inside a cube are not resolved:
//    the loops follow from the face decisions alone.  This is an intentional topological difference from skimage.
//  - Winding.  skimage.measure.marching_cubes's default (gradient_direction='descent', object above level): a
//    triangle's right-hand normal points toward higher values, into the dense region.  Each triangle is written
//    against its loop's direction.  The reference's convert_sdf_samples_to_ply reverses the faces ("inverse face
//    orientation"), so the PLY it writes, and tensoir_b200.mesh writes, faces out of the dense region.
//
// Corner c of a cell has offsets (c & 1, c >> 1 & 1, c >> 2) along axes (0, 1, 2).  Edge e runs along axis a = e >> 2
// from the corner with offsets (e & 1, e >> 1 & 1) along the other two axes, the lower axis first.  Face f = 2*axis +
// side lies at offset `side` along `axis`.
#pragma once
#include <stdint.h>
#include "tir_eval_body.h"     // ev_mul / ev_add / ev_sub / ev_div: fp32, exactly rounded, never fused

#if defined(__CUDACC__)
#define MC_HD __host__ __device__ __forceinline__
#else
#define MC_HD inline
#endif

#define MC_MAX_TRIS 12         // a cell has at most 12 crossed edges in at least one loop: <= 10 triangles

MC_HD bool mc_inside(float v, float level) { return v > level; }

// the two axes other than a, lower first
MC_HD int mc_axis_u(int a) { return a == 0 ? 1 : 0; }
MC_HD int mc_axis_w(int a) { return a == 2 ? 1 : 2; }

// lower corner of edge e
MC_HD int mc_edge_corner(int e) {
  const int a = e >> 2;
  return ((e & 1) << mc_axis_u(a)) | (((e >> 1) & 1) << mc_axis_w(a));
}
// the edge along `axis` that starts at `corner` (whose bit `axis` is 0)
MC_HD int mc_edge_id(int axis, int corner) {
  return axis * 4 + ((corner >> mc_axis_u(axis)) & 1) + (((corner >> mc_axis_w(axis)) & 1) << 1);
}
// the two faces edge e borders (s = 0: the one across the edge's lower other axis)
MC_HD int mc_edge_face(int e, int s) {
  const int a = e >> 2;
  return s == 0 ? 2 * mc_axis_u(a) + (e & 1) : 2 * mc_axis_w(a) + ((e >> 1) & 1);
}
// May a triangle edge join the vertices of edges a and b (not neighbours in their loop)?  Edges that lie in one cell
// face may be joined only by the cell on one side of that face: in a low-side face (side 0) only edges meeting at a
// corner, in a high-side face only parallel edges.  The neighbour sees the face from the other side, so the two cells
// never produce the same edge.  Edges without a common face lie in no other cell together.
MC_HD bool mc_chord_allowed(int a, int b) {
  const unsigned fa = (1u << mc_edge_face(a, 0)) | (1u << mc_edge_face(a, 1));
  const unsigned fb = (1u << mc_edge_face(b, 0)) | (1u << mc_edge_face(b, 1));
  const unsigned common = fa & fb;
  if (!common) return true;
  const bool low = (common & 0x15u) != 0;      // faces 0, 2, 4
  const bool parallel = (a >> 2) == (b >> 2);
  return low ? !parallel : parallel;
}
// corner of face f at offsets (du, dw) along the face's two axes
MC_HD int mc_face_corner(int f, int du, int dw) {
  const int a = f >> 1;
  return ((f & 1) << a) | (du << mc_axis_u(a)) | (dw << mc_axis_w(a));
}

// fp64 operations exactly rounded, never fused
MC_HD double mc_dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
MC_HD double mc_dsub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
MC_HD double mc_dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
MC_HD double mc_ddiv(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// coordinate of a vertex along its edge's axis: (i + t) * spacing, t = (level - v_lo) / (v_hi - v_lo)
MC_HD float mc_edge_coord(int64_t i, float v_lo, float v_hi, float level, double spacing) {
  const double t = mc_ddiv(mc_dsub((double)level, (double)v_lo), mc_dsub((double)v_hi, (double)v_lo));
  return (float)mc_dmul(mc_dadd((double)i, t), spacing);
}
// coordinate along the other two axes: i * spacing
MC_HD float mc_grid_coord(int64_t i, double spacing) { return (float)mc_dmul((double)i, spacing); }

// asymptotic decider on one face, values in canonical order: true = the inside corners are connected
MC_HD bool mc_face_connected(float v00, float v10, float v01, float v11, float level) {
  const float num = ev_sub(ev_mul(v00, v11), ev_mul(v10, v01));
  const float den = ev_sub(ev_sub(ev_add(v00, v11), v10), v01);
  return ev_div(num, den) > level;
}

// bit c = corner c is inside
MC_HD unsigned mc_cell_mask(const float c[8], float level) {
  unsigned m = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) m |= (unsigned)mc_inside(c[q], level) << q;
  return m;
}

// bit f = face f is ambiguous and its inside corners are connected
MC_HD unsigned mc_face_decisions(const float c[8], unsigned mask, float level) {
  unsigned d = 0;
  for (int f = 0; f < 6; ++f) {
    const int q00 = mc_face_corner(f, 0, 0), q10 = mc_face_corner(f, 1, 0);
    const int q01 = mc_face_corner(f, 0, 1), q11 = mc_face_corner(f, 1, 1);
    const unsigned i00 = mask >> q00 & 1, i10 = mask >> q10 & 1, i01 = mask >> q01 & 1, i11 = mask >> q11 & 1;
    if (i00 == i11 && i10 == i01 && i00 != i10 && mc_face_connected(c[q00], c[q10], c[q01], c[q11], level))
      d |= 1u << f;
  }
  return d;
}

// Polygonise one cell from its inside mask and face decisions.  Returns the number of triangles; when tri != nullptr,
// writes their edge ids (3 per triangle, wound as documented above).
MC_HD int mc_cell_triangles(unsigned mask, unsigned connected, int8_t* tri) {
  int8_t next[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) next[e] = -1;
  for (int f = 0; f < 6; ++f) {
    const int a = f >> 1, side = f & 1;
    // counter-clockwise about the outward normal: (0,0) (1,0) (1,1) (0,1) in (u,w) when u x w points outward
    const bool uw = (a == 1) != (side == 1);
    int q[4];
    q[0] = mc_face_corner(f, 0, 0);
    q[1] = uw ? mc_face_corner(f, 1, 0) : mc_face_corner(f, 0, 1);
    q[2] = mc_face_corner(f, 1, 1);
    q[3] = uw ? mc_face_corner(f, 0, 1) : mc_face_corner(f, 1, 0);
    int ce[4];
    bool entry[4];
    int n = 0;
    for (int t = 0; t < 4; ++t) {
      const int c0 = q[t], c1 = q[(t + 1) & 3];
      const unsigned i0 = mask >> c0 & 1, i1 = mask >> c1 & 1;
      if (i0 == i1) continue;
      const int d = c0 ^ c1;
      ce[n] = mc_edge_id(d == 1 ? 0 : (d == 2 ? 1 : 2), c0 & c1);
      entry[n] = i1 != 0;
      ++n;
    }
    if (n == 2) {
      const int k = entry[0] ? 0 : 1;
      next[ce[k]] = (int8_t)ce[1 - k];
    } else if (n == 4) {
      const bool conn = (connected >> f) & 1;
      for (int k = 0; k < 4; ++k)
        if (entry[k]) next[ce[k]] = (int8_t)ce[conn ? (k + 3) & 3 : (k + 1) & 3];
    }
  }
  int nt = 0;
  unsigned seen = 0;
  for (int e = 0; e < 12; ++e) {
    if (next[e] < 0 || (seen >> e & 1)) continue;
    int8_t loop[12];
    int k = 0;
    for (int cur = e; cur >= 0 && !(seen >> cur & 1) && k < 12; cur = next[cur]) {
      seen |= 1u << cur;
      loop[k++] = (int8_t)cur;
    }
    // ear clipping: cut off the first vertex after loop[0] whose two neighbours may be joined, until 3 are left
    while (k >= 3) {
      int i = 1;
      if (k > 3)
        while (i < k && !mc_chord_allowed(loop[i - 1], loop[(i + 1) % k])) ++i;
      if (i == k) i = 1;       // never taken: every loop of every configuration has an allowed ear (CPU tests)
      if (tri) {
        tri[3 * nt] = loop[i - 1];              // against the loop: normal toward higher values
        tri[3 * nt + 1] = loop[(i + 1) % k];
        tri[3 * nt + 2] = loop[i];
      }
      ++nt;
      for (int m = i; m + 1 < k; ++m) loop[m] = loop[m + 1];
      --k;
    }
  }
  return nt;
}

// Scratch of tir_marching_cubes_* for N = X*Y*Z points: per point the crossing bits (bit a: the edge along axis a
// from this point is crossed) and the triangle count of the cell it starts, their exclusive scans (int32), the list of
// active cells and its length, then `extra` bytes (the device build's CUB temporary storage).  Offsets are 256-aligned.
struct McWork {
  int64_t bits, tris, voff, toff, active, n_active, temp, total;
};
MC_HD int64_t mc_align(int64_t b) { return (b + 255) & ~(int64_t)255; }
MC_HD McWork mc_work_layout(int64_t n, int64_t extra) {
  McWork w;
  w.bits = 0;
  w.tris = w.bits + mc_align(n);
  w.voff = w.tris + mc_align(n);
  w.toff = w.voff + mc_align(4 * n);
  w.active = w.toff + mc_align(4 * n);
  w.n_active = w.active + mc_align(4 * n);
  w.temp = w.n_active + 256;
  w.total = w.temp + mc_align(extra);
  return w;
}

// argument checks shared by both builds: 1 = run, <0 = TirStatus
MC_HD int mc_validate_dims(int32_t X, int32_t Y, int32_t Z) {
  if (X < 2 || Y < 2 || Z < 2) return TIR_ERR_SHAPE;
  if ((int64_t)X * Y * Z > (int64_t)INT32_MAX) return TIR_ERR_SHAPE;    // the scans index points with int32
  return 1;
}

// The null and dims checks of each entry, run by tir_mesh.cu and its host build before their scratch-size check
// (the CUB scratch differs between the builds): 1 run, < 0 TirStatus
inline int mc_work_size_check(int32_t X, int32_t Y, int32_t Z, const int64_t* bytes) {
  if (!bytes) return TIR_ERR_NULL;
  return mc_validate_dims(X, Y, Z);
}

inline int mc_count_check(const float* volume, int32_t X, int32_t Y, int32_t Z, const void* work,
                          const int64_t* totals) {
  if (!volume || !work || !totals) return TIR_ERR_NULL;
  return mc_validate_dims(X, Y, Z);
}

inline int mc_emit_check(const float* volume, int32_t X, int32_t Y, int32_t Z, const void* work, int64_t n_verts,
                         int64_t n_faces, const float* verts, const int32_t* faces) {
  if (!volume || !work) return TIR_ERR_NULL;
  if (n_verts < 0 || n_faces < 0) return TIR_ERR_SHAPE;
  if (n_verts > INT32_MAX || n_faces > INT32_MAX) return TIR_ERR_SHAPE;   // vertex ids and offsets are int32
  if ((n_verts > 0 && !verts) || (n_faces > 0 && !faces)) return TIR_ERR_NULL;
  return mc_validate_dims(X, Y, Z);
}
