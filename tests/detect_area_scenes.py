"""Detection areas (include/lmot.h, lmot_set_detect_area): a NumPy restatement of the cell mask and of the E_area filter, the reference's
detection on E_area, and a cluttered roadside scene.  Shared by test_detect_area_cpu.py and test_detect_area_gpu.py."""
import numpy as np

f32 = np.float32
GRID = 250


def mask_ref(rings, keep_outside=False, pose=None, roi=50.0):
    """the definition cell by cell, in float64 without contraction (NumPy evaluates one rounding per operation) -> (250, 8) uint32"""
    m = np.eye(3, 4, dtype=f32) if pose is None else np.asarray(pose, f32).reshape(3, 4)
    r00, r01, t0, r10, r11, t1 = (float(m[0, 0]), float(m[0, 1]), float(m[0, 3]), float(m[1, 0]), float(m[1, 1]), float(m[1, 3]))
    roi = float(f32(roi))
    edges = []
    for ring in rings:
        p = np.asarray(ring, np.float64).reshape(-1, 2)
        dx, dy = p[:, 0] - t0, p[:, 1] - t1
        u, w = r00 * dx + r10 * dy, r01 * dx + r11 * dy
        edges.append((u, w, np.roll(u, -1), np.roll(w, -1)))
    au, aw, bu, bw = (np.concatenate(x) for x in zip(*edges))
    centre = (np.arange(GRID, dtype=np.float64) + 0.5) * roi / 250.0 - roi / 2.0
    inside = np.zeros((GRID, GRID), bool)
    with np.errstate(all="ignore"):
        for xI in range(GRID):
            cx = centre[xI]
            s = (au > cx) != (bu > cx)
            yc = aw[s] + (cx - au[s]) * (bw[s] - aw[s]) / (bu[s] - au[s])
            inside[xI] = ((centre[:, None] < yc[None, :]).sum(1) & 1).astype(bool)
    bits = inside != bool(keep_outside)
    out = np.zeros((GRID, 8), np.uint32)
    for y in range(GRID):
        out[:, y >> 5] |= bits[:, y].astype(np.uint32) << np.uint32(y & 31)
    return out


def cells(points, roi=50.0):
    """componentClustering's float binning (component_clustering.cpp:43-48): (xI, yI, in-grid) per point, in float32"""
    p = np.asarray(points, f32)
    roi = f32(roi)
    half = roi / f32(2)
    xc, yc = p[:, 0] + half, p[:, 1] + half
    ok = (xc >= 0) & (xc < roi) & (yc >= 0) & (yc < roi)
    xi = np.floor((f32(GRID) * xc) / roi).astype(np.int64)
    yi = np.floor((f32(GRID) * yc) / roi).astype(np.int64)
    return np.where(ok, xi, 0), np.where(ok, yi, 0), ok


def area_filter(points, mask, roi=50.0):
    """E_area: the points whose clustering cell has its mask bit set, in cloud order"""
    xi, yi, ok = cells(points, roi)
    bit = (mask[xi, yi >> 5] >> (yi & 31).astype(np.uint32)) & 1
    return np.ascontiguousarray(np.asarray(points, f32)[ok & (bit == 1)])


def ref_detect_area(ref, pts, mask, roi=50.0):
    """the reference's groundRemove, the E_area filter, componentClustering and boxFitting -> (counts, boxes, E_area, grid)"""
    e, g = ref.ground_remove(pts)
    ea = area_filter(e, mask, roi)
    grid, k = ref.component_clustering(ea)
    b, _ = ref.box_fitting(ea, grid, k)
    return (len(e), len(g), k, len(b)), b, ea, grid


def rect(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], np.float64)


CORRIDOR = [rect(-25.0, -7.0, 25.0, 7.0)]
# roadside clutter outside the corridor: poles (0.3 x 0.3 x 3 m) and hedges (3 x 0.8 x 1.2 m), (x, y, length, width, height)
CLUTTER = ([(x, s * 12.0, 0.3, 0.3, 3.0) for x in (-18.0, -9.0, 0.0, 9.0, 18.0) for s in (-1, 1)]
           + [(x, s * 17.0, 3.0, 0.8, 1.2) for x in (-14.0, -4.0, 6.0, 16.0) for s in (-1, 1)])


def clutter_points(seed=0, z_ground=-1.73, per_m2=400.0):
    """dense samples of the clutter's four sides and top, XYZI float32"""
    rng = np.random.default_rng(seed)
    out = []
    for x, y, L, W, H in CLUTTER:
        n = int(per_m2 * (2 * (L + W) * H + L * W))
        face = rng.integers(0, 5, n)
        u, v = rng.random(n), rng.random(n)
        px = x + (u - 0.5) * L
        py = y + (v - 0.5) * W
        pz = z_ground + 0.3 + rng.random(n) * (H - 0.3)
        px = np.where(face == 0, x - L / 2, np.where(face == 1, x + L / 2, px))
        py = np.where(face == 2, y - W / 2, np.where(face == 3, y + W / 2, py))
        pz = np.where(face == 4, z_ground + H, pz)
        out.append(np.stack([px, py, pz, np.ones(n)], 1))
    return np.concatenate(out).astype(f32)


def cluttered_frames(synth, n_frames, seed=7):
    """(ts, synth frame + clutter) per frame"""
    extra = clutter_points(seed)
    for ts, p in synth.frames(synth.SceneConfig(seed=seed, rings=32, azimuths=900, n_objects=20), n_frames):
        yield ts, np.ascontiguousarray(np.concatenate([p, extra]).astype(f32))


def near_clutter(boxes, tol=1.0):
    """per box: its centre lies within tol of a clutter item's footprint"""
    b = np.asarray(boxes, f32).reshape(-1, 8, 3)
    c = b[:, :4, :2].mean(1)
    hit = np.zeros(len(b), bool)
    for x, y, L, W, _ in CLUTTER:
        hit |= (np.abs(c[:, 0] - x) <= L / 2 + tol) & (np.abs(c[:, 1] - y) <= W / 2 + tol)
    return hit
