"""Box search (include/lmot.h, lmot_set_box_search): steps 1-5 restated once, in NumPy; the reference's getClusteredPoints and
ruleBasedFilter around them (oracle/_ref/libref_box_search_<mode>.so, oracle/ref_box_search.cpp); and the yaw error of boxes against
synth.py's cars.  Shared by test_box_search_cpu.py and test_box_search_gpu.py."""
import ctypes as C
import math
import os

import numpy as np

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def angles(A):
    """step 1: (A, 2) float32 (c_a, s_a), theta_a = (pi / 2) * a / A in double with the host libm"""
    return np.array([[math.cos((math.pi / 2) * a / A), math.sin((math.pi / 2) * a / A)] for a in range(A)], np.float64).astype(f32)


def fit(xy, A, chunk=8):
    """steps 2-5 on one cluster's points (n, >= 2) -> (a*, corners (4, 2) float32, S (A,) uint64).  float32 NumPy ufuncs round every
    operation once and never contract."""
    x = np.ascontiguousarray(xy[:, 0], f32)
    y = np.ascontiguousarray(xy[:, 1], f32)
    tab = angles(A)
    S = np.zeros(A, np.uint64)
    ext = np.zeros((A, 4), f32)
    for a0 in range(0, A, chunk):
        c = tab[a0:a0 + chunk, 0][:, None]
        s = tab[a0:a0 + chunk, 1][:, None]
        u = x * c + y * s
        w = y * c - x * s
        umin, umax = u.min(1, keepdims=True), u.max(1, keepdims=True)
        wmin, wmax = w.min(1, keepdims=True), w.max(1, keepdims=True)
        d1 = np.minimum(umax - u, u - umin)
        d2 = np.minimum(wmax - w, w - wmin)
        d = np.maximum(np.minimum(d1, d2), f32(0.01))
        q = (f32(65536.0) / d).astype(np.uint32)
        S[a0:a0 + chunk] = q.sum(1, dtype=np.uint64)
        ext[a0:a0 + chunk] = np.concatenate([umin, umax, wmin, wmax], 1)
    a = int(np.argmax(S))                      # the first maximum: ties go to the smallest a
    c, s = tab[a]
    u0, u1, w0, w1 = ext[a]
    U = np.array([u0, u1, u1, u0], f32)
    W = np.array([w0, w0, w1, w1], f32)
    pc = np.stack([U * c - W * s, U * s + W * c], 1).astype(f32)
    return a, pc, S


class RefSearch:
    """the reference's getClusteredPoints / ruleBasedFilter of libref_<mode>.so (load RefOracle(mode) first: the helper binds to it)"""

    def __init__(self, mode="intended"):
        self.lib = C.CDLL(lib_path(mode))
        self.lib.ref_bs_clusters.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        self.lib.ref_bs_clusters.restype = C.c_int
        self.lib.ref_bs_rule.argtypes = [C.c_void_p, C.c_float, C.c_int]
        self.lib.ref_bs_rule.restype = C.c_int
        self.lib.ref_bs_sensor_height.restype = C.c_float
        self.sensor_height = f32(self.lib.ref_bs_sensor_height())

    def clusters(self, elev, grid, k):
        """cluster c's points (n_c, 3) in the reference's order, c = 1 .. k"""
        e = np.ascontiguousarray(elev, f32).reshape(-1, 3) if len(elev) else np.zeros((1, 3), f32)
        g = np.ascontiguousarray(grid, np.int32).reshape(-1)
        pts = np.zeros((max(len(elev), 1), 3), f32)
        off = np.zeros(k + 1, np.int32)
        self.lib.ref_bs_clusters(e.ctypes.data, len(elev), 3, g.ctypes.data, int(k), pts.ctypes.data, off.ctypes.data)
        return [pts[off[c]:off[c + 1]] for c in range(k)]

    def rule(self, pc, max_z, n):
        p = np.ascontiguousarray(pc, f32).reshape(8)
        return bool(self.lib.ref_bs_rule(p.ctypes.data, float(max_z), int(n)))

    def boxes(self, elev, grid, k, A, sensor_height=None, min_points=30):
        """the searched boxes of a unit in cluster order -> (m, 8, 3) float32"""
        h = self.sensor_height if sensor_height is None else f32(sensor_height)
        out = []
        for pts in self.clusters(elev, grid, k):
            n = len(pts)
            if n == 0 or n < min_points:
                continue
            max_z = max(f32(-99.0), pts[:, 2].max())
            _, pc, _ = fit(pts, A)
            if self.rule(pc, max_z, n):
                b = np.zeros((8, 3), f32)
                b[:4, :2] = pc
                b[4:, :2] = pc
                b[:4, 2] = -h
                b[4:, 2] = max_z
                out.append(b)
        return np.array(out, f32).reshape(-1, 8, 3)


def lib_path(mode):
    return os.path.join(ROOT, "oracle", "_ref", f"libref_box_search_{mode}.so")


def have_ref_search(mode="intended"):
    return os.path.exists(lib_path(mode))


def ref_search_detect(ref, rs, points, A):
    """the reference's groundRemove and componentClustering, then the search -> ((n_elev, n_ground, num_cluster, n_boxes), boxes)"""
    e, g = ref.ground_remove(points)
    grid, k = ref.component_clustering(e)
    b = rs.boxes(e, grid, k, A)
    return (len(e), len(g), k, len(b)), b


# ------------------------------------------------------------------------------------------------ yaw error against synth.py's cars
def box_yaw_errors(boxes, cars, radius=2.0):
    """cars: (m, 3) x, y, yaw of the true cars.  Each box whose centre (the mean of its four bottom corners: the intersection of the
    diagonals) lies within `radius` of a car's centre is matched to the nearest one; its yaw (edge P0 -> P1) against the car's, modulo
    90 degrees -> degrees, one per matched box"""
    out = []
    for b in np.asarray(boxes, np.float64).reshape(-1, 8, 3):
        cx, cy = b[:4, 0].mean(), b[:4, 1].mean()
        if len(cars) == 0:
            break
        d = np.hypot(cars[:, 0] - cx, cars[:, 1] - cy)
        j = int(np.argmin(d))
        if d[j] > radius:
            continue
        yb = math.atan2(b[1, 1] - b[0, 1], b[1, 0] - b[0, 0])
        e = math.degrees(yb - cars[j, 2]) % 90.0
        out.append(min(e, 90.0 - e))
    return out


def scene_cars(synth, cfg, n_frames):
    """(x, y, yaw) of the cars in each of the first n_frames frames of synth.frames(cfg)"""
    sc = synth.make_scene(cfg)
    out = []
    for _ in range(n_frames):
        car = sc.size[:, 0] > 4.0
        out.append(np.stack([sc.pos[car, 0], sc.pos[car, 1], sc.yaw[car]], 1))
        synth.advance(sc)
    return out
