"""numpy restatement of the marching-cubes conventions of csrc/tir_mc_body.h (the native mesh export), for the CPU
tests.  Written from the documented rules, not from the C++: the cell topology is derived geometrically (outward face
normals and a cross-product test for the counter-clockwise walk) and cached per (inside mask, face decisions)
configuration; everything else is vectorised over points and active cells.

  * inside iff v > level (NaN is outside);
  * one vertex per crossed grid edge, numbered by (point linear index, axis);
  * position along the edge (i + t) * spacing, t = (level - v_lo) / (v_hi - v_lo), in float64, rounded to float32 once;
  * asymptotic decider on ambiguous faces, saddle = (v00 v11 - v10 v01) / (v00 + v11 - v10 - v01) > level in float32
    with the values in global (u, w) order -- float32 because that is what the kernels evaluate, so that this
    restatement takes the same decision on near-ties;
  * segments from entry to exit crossings of the counter-clockwise walk about the outward normal, an entry paired with
    the next exit (inside corners separated) or the previous one (connected); loops followed from their lowest edge
    id and cut into triangles by ear clipping: the first vertex after the loop's first whose neighbours may be
    joined (chord_allowed) goes first, until three remain; each triangle is written against the loop's direction,
    so its right-hand normal points toward higher values (skimage's default winding);
  * edge ids: axis * 4 + offset along the lower other axis + 2 * offset along the higher one.
"""
from __future__ import annotations

import functools
import itertools

import numpy as np

CORNERS = [np.array([c & 1, c >> 1 & 1, c >> 2 & 1]) for c in range(8)]


def _others(a):
    return [b for b in range(3) if b != a]


def _corner_id(off):
    return int(off[0]) + 2 * int(off[1]) + 4 * int(off[2])


def _edge_id(c0, c1):
    """edge between two corners that differ along one axis"""
    d = np.abs(CORNERS[c1] - CORNERS[c0])
    a = int(np.argmax(d))
    lo = np.minimum(CORNERS[c0], CORNERS[c1])
    u, w = _others(a)
    return 4 * a + int(lo[u]) + 2 * int(lo[w])


def _face_walk(a, side):
    """the face's four corners, counter-clockwise about the cell's outward normal"""
    u, w = _others(a)
    n = np.zeros(3)
    n[a] = 1 if side else -1
    quad = [(0, 0), (1, 0), (1, 1), (0, 1)]
    pts = []
    for du, dw in quad:
        off = np.zeros(3, dtype=int)
        off[a], off[u], off[w] = side, du, dw
        pts.append(off)
    p = [q.astype(float) for q in pts]
    if np.dot(np.cross(p[1] - p[0], p[2] - p[1]), n) < 0:
        pts = [pts[0], pts[3], pts[2], pts[1]]
    return [_corner_id(q) for q in pts]


FACES = [(a, side) for a in range(3) for side in (0, 1)]       # face f = 2 * axis + side


def _edge_faces(e):
    """the faces (2 * axis + side) that contain both corners of edge e"""
    a = e // 4
    u, w = _others(a)
    lo = np.zeros(3, dtype=int)
    lo[u], lo[w] = e & 1, (e >> 1) & 1
    hi = lo.copy()
    hi[a] = 1
    return {2 * b + int(lo[b]) for b in range(3) if lo[b] == hi[b]}


def chord_allowed(a, b):
    """a triangle edge between the vertices of edges a and b: inside a low-side face only between edges that meet at
    a corner, inside a high-side face only between parallel edges (the neighbour sees the face from the other side)"""
    common = _edge_faces(a) & _edge_faces(b)
    if not common:
        return True
    (f,) = common
    parallel = a // 4 == b // 4
    return parallel if f % 2 else not parallel


@functools.lru_cache(maxsize=None)
def cell_triangles(mask, connected):
    """Triangles of one cell as tuples of edge ids."""
    inside = [(mask >> c) & 1 for c in range(8)]
    nxt = {}
    for f, (a, side) in enumerate(FACES):
        walk = _face_walk(a, side)
        cross = []                       # (edge, is_entry) in walk order
        for t in range(4):
            c0, c1 = walk[t], walk[(t + 1) % 4]
            if inside[c0] != inside[c1]:
                cross.append((_edge_id(c0, c1), bool(inside[c1])))
        if len(cross) == 2:
            ent = [e for e, is_in in cross if is_in][0]
            ext = [e for e, is_in in cross if not is_in][0]
            nxt[ent] = ext
        elif len(cross) == 4:
            conn = (connected >> f) & 1
            for k, (e, is_in) in enumerate(cross):
                if is_in:
                    nxt[e] = cross[(k - 1) % 4][0] if conn else cross[(k + 1) % 4][0]
    tris, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        cur = nxt[e]
        while cur != e:
            loop.append(cur)
            cur = nxt[cur]
        seen.update(loop)
        while len(loop) > 3:
            i = next(i for i in range(1, len(loop)) if chord_allowed(loop[i - 1], loop[(i + 1) % len(loop)]))
            tris.append((loop[i - 1], loop[(i + 1) % len(loop)], loop[i]))
            del loop[i]
        tris.append((loop[0], loop[2], loop[1]))
    return tuple(tris)


def _decider(v00, v10, v01, v11, level):
    f = np.float32
    with np.errstate(all="ignore"):
        num = f(v00) * f(v11) - f(v10) * f(v01)
        den = ((f(v00) + f(v11)) - f(v10)) - f(v01)
        return (num / den) > f(level)


def marching_cubes(vol, level, spacing=(1.0, 1.0, 1.0)):
    """(verts [V,3] float32, faces [F,3] int32) of a [X,Y,Z] float32 volume, in the kernels' order."""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    X, Y, Z = vol.shape
    level = np.float32(level)
    inside = vol > level
    # crossing bits [X,Y,Z,3] and vertex ids in (point, axis) order
    bits = np.zeros((X, Y, Z, 3), dtype=bool)
    bits[:-1, :, :, 0] = inside[:-1] != inside[1:]
    bits[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    bits[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = bits.reshape(-1)
    vid = np.cumsum(flat) - 1
    p, a = np.divmod(np.nonzero(flat)[0], 3)
    idx = np.stack(np.unravel_index(p, (X, Y, Z)), -1)
    step = np.eye(3, dtype=np.int64)[a]
    vlo = vol.reshape(-1)[p].astype(np.float64)
    vhi = vol[tuple((idx + step).T)].astype(np.float64)
    with np.errstate(all="ignore"):
        t = (np.float64(level) - vlo) / (vhi - vlo)
    sp = np.asarray(spacing, dtype=np.float64)
    pos = idx.astype(np.float64) * sp
    rows = np.arange(len(p))
    pos[rows, a] = (idx[rows, a] + t) * sp[a]
    verts = pos.astype(np.float32)
    # cells: corner values [.., 8], masks, face decisions, then triangles per configuration
    c = np.stack([vol[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz] for dz, dy, dx in itertools.product((0, 1), repeat=3)],
                 -1).reshape(-1, 8)
    mask = ((c > level).astype(np.int64) << np.arange(8)).sum(-1)
    act = np.nonzero((mask != 0) & (mask != 255))[0]
    c, mask = c[act], mask[act]
    conn = np.zeros(len(act), dtype=np.int64)
    for f, (ax, side) in enumerate(FACES):
        u, w = _others(ax)
        q = [[0] * 3 for _ in range(4)]
        for k, (du, dw) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
            q[k][ax], q[k][u], q[k][w] = side, du, dw
        q00, q10, q01, q11 = (_corner_id(x) for x in q)
        ins = [(mask >> x) & 1 for x in (q00, q10, q01, q11)]
        amb = (ins[0] == ins[3]) & (ins[1] == ins[2]) & (ins[0] != ins[1])
        dec = _decider(c[:, q00], c[:, q10], c[:, q01], c[:, q11], level)
        conn |= (amb & dec).astype(np.int64) << f
    ci = np.stack(np.unravel_index(act, (X - 1, Y - 1, Z - 1)), -1)
    key = mask * 64 + conn
    tris_of = {k: cell_triangles(int(k) >> 6, int(k) & 63) for k in np.unique(key)}
    n_t = np.array([len(tris_of[k]) for k in key], dtype=np.int64)
    cell_of_tri = np.repeat(np.arange(len(act)), n_t)
    local = np.array([e for k in key for tri in tris_of[k] for e in tri], dtype=np.int64).reshape(-1, 3)
    if len(local) == 0:
        return verts, np.zeros((0, 3), dtype=np.int32)
    e_axis = local // 4
    lo_corner = np.zeros_like(local)
    for e in range(12):
        ax = e // 4
        u, w = _others(ax)
        off = [0, 0, 0]
        off[u], off[w] = e & 1, (e >> 1) & 1
        lo_corner[local == e] = _corner_id(off)
    off = np.stack([lo_corner & 1, lo_corner >> 1 & 1, lo_corner >> 2 & 1], -1)
    gp = ci[cell_of_tri][:, None, :] + off
    lin = (gp[..., 0] * Y + gp[..., 1]) * Z + gp[..., 2]
    faces = vid[lin * 3 + e_axis].astype(np.int32)
    return verts, faces


def crossed_edge_count(vol, level):
    """number of grid edges whose endpoints lie on different sides of level (= V)"""
    ins = np.asarray(vol) > np.float32(level)
    return int((ins[1:] != ins[:-1]).sum() + (ins[:, 1:] != ins[:, :-1]).sum() + (ins[:, :, 1:] != ins[:, :, :-1]).sum())
