"""Obstacle footprints (include/lmot.h, lmot_set_obstacles) restated once in NumPy: each cluster's cells, the convex hull of their corners by
the monotone chain over column extremes, the metres conversion, z range and box index, plus an independent brute-force hull and the
140-vertex lattice polygon of the vertex-count bound.  Shared by test_obstacles_cpu.py and test_obstacles_gpu.py."""
import math

import numpy as np

import layer_scenes as ls

f32 = np.float32
GRID = 250
MAX_HULL = 140                 # LMOT_OBSTACLE_MAX_HULL


# ------------------------------------------------------------------------------------------------ the hull of a cell set
def _cross(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def _chain(points):
    h = []
    for p in points:
        while len(h) >= 2 and _cross(h[-2], h[-1], p) <= 0:
            h.pop()
        h.append(p)
    return h


def hull(cells):
    """cells: iterable of (u, v) -> the footprint's vertices as an (m, 2) int array: the convex hull of every cell corner,
    counter-clockwise from the smallest (u, v), collinear corners dropped"""
    lo, hi = {}, {}
    for u, v in cells:
        u, v = int(u), int(v)
        for c in (u, u + 1):
            lo[c] = min(lo.get(c, v), v)
            hi[c] = max(hi.get(c, v + 1), v + 1)
    if not lo:
        return np.zeros((0, 2), np.int64)
    cols = sorted(lo)
    u0, u1 = cols[0], cols[-1]
    lower = _chain([(u, lo[u]) for u in cols] + [(u1, hi[u1])])
    upper = _chain([(u, hi[u]) for u in reversed(cols)] + [(u0, lo[u0])])
    return np.array(lower[:-1] + upper[:-1], np.int64)


def corners(cells):
    c = set()
    for u, v in cells:
        for du in (0, 1):
            for dv in (0, 1):
                c.add((int(u) + du, int(v) + dv))
    return np.array(sorted(c), np.int64).reshape(-1, 2)


def brute_vertices(cells):
    """the hull's vertex set by definition, in integer arithmetic: corner p is a vertex iff the vectors q - p to every other corner lie in an
    open half-plane, i.e. some w_a has every w_b strictly to its left or pointing its own way"""
    C = corners(cells)
    out = set()
    for i in range(len(C)):
        W = np.delete(C, i, axis=0) - C[i]
        if len(W) == 0:
            out.add(tuple(C[i]))
            continue
        cr = W[:, None, 0] * W[None, :, 1] - W[:, None, 1] * W[None, :, 0]          # cr[a, b] = w_a x w_b
        dt = W[:, None, 0] * W[None, :, 0] + W[:, None, 1] * W[None, :, 1]
        if np.any(np.all((cr > 0) | ((cr == 0) & (dt > 0)), axis=1)):
            out.add(tuple(C[i]))
    return out


def to_metres(verts, roi=50.0):
    """(float)((double)u * roi / 250.0 - roi / 2.0) with the unit's float roi_m"""
    r = float(f32(roi))
    return (np.asarray(verts, np.float64) * r / 250.0 - r / 2.0).astype(f32)


# ------------------------------------------------------------------------------------------------ the obstacles of a unit
def obstacles(elev, ids, k, roi=50.0, box_ok=None, max_boxes=1024):
    """one unit: its cloud E (N, >=3), each point's cluster id (0: none) and the cluster count k -> list of dicts (cluster, n_points,
    n_cells, z_min, z_max, box, hull (m, 2) lattice, xy (m, 2) float32 metres), cluster order.  box_ok[c - 1]: the rule filter's verdict on
    cluster c (None: every box -1)"""
    pts = np.asarray(elev, f32)
    xi, yi, ok = ls.columns(pts, roi)
    out, rank = [], 0
    for c in range(1, k + 1):
        sel = np.nonzero((ids == c) & ok)[0]
        cells = set(zip(xi[sel].tolist(), yi[sel].tolist()))
        h = hull(cells)
        z = pts[ids == c, 2]
        box = -1
        if box_ok is not None and box_ok[c - 1]:
            box = rank if rank < max_boxes else -1
            rank += 1
        out.append(dict(cluster=c, n_points=int((ids == c).sum()), n_cells=len(cells), z_min=f32(z.min()) if len(z) else f32(0),
                        z_max=f32(z.max()) if len(z) else f32(0), box=box, hull=h, xy=to_metres(h, roi)))
    return out


def label_ids(elev, grid, roi=50.0):
    """cluster id of every point of E from a 250 x 250 label grid (componentClustering's), 0 for points without a cell"""
    xi, yi, ok = ls.columns(np.asarray(elev, f32), roi)
    ids = np.zeros(len(xi), np.int32)
    ids[ok] = np.asarray(grid)[xi[ok], yi[ok]]
    return ids


def ref_box_flags(ref, elev, ids, k, roi=50.0):
    """the reference's verdict per cluster: boxFitting(E_c, grid_c, 1) returns a box or nothing (seeded per cluster, so exact)"""
    pts = np.ascontiguousarray(np.asarray(elev, f32)[:, :3])
    xi, yi, _ = ls.columns(pts, roi)
    flags, boxes = [], []
    for c in range(1, k + 1):
        sel = np.nonzero(ids == c)[0]
        if len(sel) == 0:
            flags.append(False)
            continue
        grid = np.zeros((GRID, GRID), np.int32)
        grid[xi[sel], yi[sel]] = 1
        b, _ = ref.box_fitting(pts[sel], grid, 1)
        flags.append(len(b) > 0)
        boxes.extend(list(b))
    return np.array(flags, bool), np.array(boxes, f32).reshape(-1, 8, 3)


def inside(poly_xy, pts):
    """points (N, 2) inside or on the convex counter-clockwise polygon (float64 test)"""
    P = np.asarray(poly_xy, np.float64)
    q = np.asarray(pts, np.float64)
    ok = np.ones(len(q), bool)
    for i in range(len(P)):
        a, b = P[i], P[(i + 1) % len(P)]
        ok &= (b[0] - a[0]) * (q[:, 1] - a[1]) - (b[1] - a[1]) * (q[:, 0] - a[0]) >= -1e-9
    return ok


# ------------------------------------------------------------------------------------------------ the vertex-count bound
def primitive_vectors(m_max):
    """every primitive integer vector (a, b) with 1 <= |a| + |b| <= m_max"""
    out = []
    for m in range(1, m_max + 1):
        for a in range(-m, m + 1):
            for b in sorted({m - abs(a), abs(a) - m}):
                if math.gcd(abs(a), abs(b)) == 1:
                    out.append((a, b))
    return out


def bound_from_l1(budget=4 * GRID):
    """the most distinct primitive vectors whose |a| + |b| sum to at most `budget` (cheapest first): the vertex-count bound"""
    n, spent, m = 0, 0, 1
    while True:
        cnt = len([v for v in primitive_vectors(m) if abs(v[0]) + abs(v[1]) == m])
        take = min(cnt, (budget - spent) // m)
        n += take
        spent += take * m
        if take < cnt:
            return n
        m += 1


def max_hull_polygon():
    """the 140-vertex convex lattice polygon in [0, 250]^2: every primitive vector with |a| + |b| <= 10 and six pairs with |a| + |b| = 11,
    in angle order, moved to the origin"""
    extra = [(1, 10), (10, 1), (2, 9), (9, 2), (3, 8), (8, 3)]
    vs = primitive_vectors(10) + extra + [(-a, -b) for a, b in extra]
    vs.sort(key=lambda v: math.atan2(v[1], v[0]))
    pts = [(0, 0)]
    for a, b in vs[:-1]:
        pts.append((pts[-1][0] + a, pts[-1][1] + b))
    P = np.array(pts, np.int64)
    return P - P.min(axis=0)


def max_hull_cells():
    """the cells whose squares lie inside max_hull_polygon()"""
    P = max_hull_polygon()
    u, v = np.meshgrid(np.arange(GRID), np.arange(GRID), indexing="ij")
    ok = np.ones(u.shape, bool)
    for i in range(len(P)):
        a, b = P[i], P[(i + 1) % len(P)]
        for du in (0, 1):
            for dv in (0, 1):
                ok &= (b[0] - a[0]) * (v + dv - a[1]) - (b[1] - a[1]) * (u + du - a[0]) >= 0
    return list(zip(u[ok].tolist(), v[ok].tolist()))
