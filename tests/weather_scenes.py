"""The dynamic radius outlier filter considered in DESIGN.md §6m, on the elevated cloud E in cloud order, all arithmetic in double on
coordinates widened from float:
  1. point i's range r_i = sqrt(x_i * x_i + y_i * y_i);
  2. its radius R_i = min(max(min_radius, beta * (alpha_rad * r_i)), max_radius);
  3. point j != i (duplicates included) is a neighbour of i iff ((dx * dx + dy * dy) + dz * dz) <= R_i * R_i, d = p_j - p_i;
  4. E_kept: the points with at least min_neighbors neighbours, in cloud order.
Here: a NumPy restatement of steps 1-4, a pairwise evaluation of the same definition, snowy frames of synth.py's scene, and the
reference's detection on E and on E_kept.  Shared by test_outlier_cpu.py and scripts/outlier_premise.py."""
import numpy as np
from scipy.spatial import cKDTree

f32 = np.float32
DEFAULTS = dict(alpha_rad=0.0035, beta=3.0, min_radius=0.04, max_radius=1.0, min_neighbors=3)
# snow levels: the share of rays a flake intercepts
SNOW = {"light": 0.005, "moderate": 0.015, "heavy": 0.03}
# 64 beams (synth.py's default sensor) and a 32-beam sensor with the HDL-32E's elevations, both at about 0.2 deg azimuth steps
SENSORS = {"64": dict(rings=64, azimuths=1875), "32": dict(rings=32, azimuths=1800, elev_top_deg=10.67, elev_bot_deg=-30.67)}


def radii(points, alpha_rad=0.0035, beta=3.0, min_radius=0.04, max_radius=1.0, **_):
    """steps 1-2: R_i in double, left to right"""
    p = np.asarray(points, f32)[:, :3].astype(np.float64)
    r = np.sqrt(p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1])
    return np.minimum(np.maximum(min_radius, beta * (alpha_rad * r)), max_radius)


def _d2(p, i, j):
    d = p[j] - p[i]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def neighbour_counts(points, **cfg):
    """step 3: each point's neighbour count.  A k-d tree proposes candidates a little beyond R_i; the exact test
    decides."""
    c = dict(DEFAULTS, **cfg)
    p = np.asarray(points, f32)[:, :3].astype(np.float64)
    n = len(p)
    if n == 0:
        return np.zeros(0, np.int64)
    R = radii(p, **c)
    lists = cKDTree(p).query_ball_point(p, R * (1 + 1e-9) + 1e-9)
    cnt = np.zeros(n, np.int64)
    for i, cand in enumerate(lists):
        j = np.asarray(cand, np.int64)
        j = j[j != i]
        if len(j):
            cnt[i] = int(np.count_nonzero(_d2(p, i, j) <= R[i] * R[i]))
    return cnt


def keep_flags(points, **cfg):
    """step 4: the keep flag of every point of E"""
    c = dict(DEFAULTS, **cfg)
    k = int(c["min_neighbors"])
    if k == 0:
        return np.ones(len(points), bool)
    return neighbour_counts(points, **c) >= k


def keep_brute(points, **cfg):
    """steps 1-4 by the letter: every pair"""
    c = dict(DEFAULTS, **cfg)
    p = np.asarray(points, f32)[:, :3].astype(np.float64)
    n = len(p)
    R = radii(p, **c)
    out = np.zeros(n, bool)
    for i in range(n):
        cnt = 0
        for j in range(n):
            if j != i:
                dx, dy, dz = p[j, 0] - p[i, 0], p[j, 1] - p[i, 1], p[j, 2] - p[i, 2]
                if (dx * dx + dy * dy) + dz * dz <= R[i] * R[i]:
                    cnt += 1
        out[i] = cnt >= int(c["min_neighbors"])
    return out


def kept(points, **cfg):
    """E_kept in cloud order"""
    p = np.asarray(points, f32)
    return np.ascontiguousarray(p[keep_flags(p, **cfg)])


def snow(points, p, seed, mean_m=8.0):
    """each ray's return is replaced, with probability p, by a flake's: at a range drawn from an exponential distribution of mean
    mean_m truncated to [0, true range), on the ray's own direction"""
    pts = np.array(points, f32, copy=True)
    rng = np.random.default_rng(seed)
    q = pts[:, :3].astype(np.float64)
    t = np.sqrt((q * q).sum(1))
    hit = (rng.random(len(q)) < p) & (t > 0)
    u = rng.random(len(q))
    d = -mean_m * np.log1p(-u * -np.expm1(-t / mean_m))
    s = np.where(hit, d / np.where(t > 0, t, 1.0), 1.0)
    pts[hit, :3] = (q[hit] * s[hit, None]).astype(f32)
    return pts


def scene_frames(synth, sensor="64", n_frames=3, seed=5, level=None):
    """(points, object centres (K, 2)) for n_frames frames of synth.py's scene rendered by `sensor`, with snow of `level` (None: clean)"""
    cfg = synth.SceneConfig(seed=seed, n_objects=60, **SENSORS[sensor])
    sc = synth.make_scene(cfg)
    out = []
    for f in range(n_frames):
        pts = synth.render(sc)
        if level is not None:
            pts = snow(pts, SNOW[level], seed=1000 * seed + 17 * f + int(1000 * SNOW[level]))
        out.append((pts, sc.pos.copy()))
        synth.advance(sc)
    return out


def centres(boxes):
    b = np.asarray(boxes, f32).reshape(-1, 8, 3)
    return b[:, :4, :2].astype(np.float64).mean(1)


def score(boxes, objects, tol=1.0):
    """(objects found: a box centre within tol of the object's centre, ghost boxes: boxes within tol of no object)"""
    c = centres(boxes)
    if len(c) == 0:
        return 0, 0
    d = np.hypot(c[:, None, 0] - objects[None, :, 0], c[:, None, 1] - objects[None, :, 1])
    return int((d <= tol).any(0).sum()), int((~(d <= tol).any(1)).sum())


def ref_detect(ref, pts, filt=None):
    """the reference's groundRemove, then (filt: a setting) the filter, componentClustering and boxFitting -> (counts, boxes, cloud)"""
    e, g = ref.ground_remove(pts)
    ek = e if filt is None else kept(e, **filt)
    grid, k = ref.component_clustering(ek)
    b, _ = ref.box_fitting(ek, grid, k)
    return (len(e), len(g), k, len(b)), b, ek
