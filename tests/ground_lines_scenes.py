"""Ground lines (include/lmot.h, lmot_set_ground_lines): steps 2-5 restated once in NumPy / Python doubles, scenes whose ground is not
the sensor frame's plane z = -1.73 (grades, a pitched and a rolled sensor), and the reference's own chain on the line-labelled cloud.
Shared by test_ground_lines_cpu.py and test_ground_lines_gpu.py."""
import importlib
import math

import numpy as np

f32 = np.float32
NCH, NBIN = 80, 120
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")


# ------------------------------------------------------------------------------------------------ steps 2-3: the lines of a grid
def _fit(S):
    n, sr, sz, srr, srz, szz = S
    den = n * srr - sr * sr
    m = (n * srz - sr * sz) / den
    c = (sz - m * sr) / n
    sse = szz - 2 * m * srz - 2 * c * sz + m * m * srr + 2 * m * c * sr + n * c * c
    return m, c, sse


def _add(S, r, z):
    n, sr, sz, srr, srz, szz = S
    return (n + 1, sr + r, sz + z, srr + r * r, srz + r * z, szz + z * z)


def channel_lines(minz_row, r_min, r_max, sensor_height, max_slope=0.3, max_rmse=0.08, max_step=0.3):
    """step 2 for one channel: [(first bin, m, c)] in bin order (Python floats are IEEE doubles, evaluated as written)"""
    r_min, r_max, sensor_height = float(r_min), float(r_max), float(sensor_height)
    lines = []
    S, first, r0, z0 = (0.0,) * 6, 0, 0.0, 0.0

    def close(S):
        if S[0] >= 2:
            m, c, _ = _fit(S)
            lines.append((first, m, c))
        return (0.0,) * 6

    for b in range(NBIN):
        if not float(minz_row[b]) < 1000.0:
            continue
        r = r_min + (b + 0.5) * (r_max - r_min) / 120
        z = float(minz_row[b])
        if S[0] >= 2:
            T = _add(S, r, z)
            m, c, sse = _fit(T)
            if abs(m) <= max_slope and sse <= T[0] * max_rmse * max_rmse:
                S = T
                continue
            S = close(S)
        while True:
            if lines:
                _, lm, lc = lines[-1]
                ok = abs(z - (lm * r + lc)) <= max_step
            else:
                ok = abs(z + sensor_height) <= max_slope * r + max_step
            if ok and S[0] == 1:
                ok = abs(z - z0) <= max_slope * (r - r0)
            if ok:
                if S[0] == 0:
                    first, r0, z0 = b, r, z
                S = _add(S, r, z)
                break
            if S[0] == 1:
                S = (0.0,) * 6
                continue
            break
    close(S)
    return lines


def lines_grid(minz, r_min, r_max, sensor_height, **kw):
    """steps 2-3: (80, 120) float32 ground heights of a (80, 120) min-z grid"""
    minz = np.asarray(minz, f32).reshape(NCH, NBIN)
    r_min, r_max = float(r_min), float(r_max)
    out = np.empty((NCH, NBIN), f32)
    for ch in range(NCH):
        L = channel_lines(minz[ch], r_min, r_max, sensor_height, **kw)
        for b in range(NBIN):
            if not L:
                out[ch, b] = f32(-float(sensor_height))
                continue
            k = 0
            for j, (fb, _, _) in enumerate(L):
                if fb <= b:
                    k = j
            _, m, c = L[k]
            r = r_min + (b + 0.5) * (r_max - r_min) / 120
            out[ch, b] = f32(m * r + c)
    return out


# ------------------------------------------------------------------------------------------------ step 4: labels, step 5: box heights
def window_cells(ref, points, r_min, r_max):
    """cell id (ch * 120 + b) of every point, -1 outside the window (groundRemove's filterCloud and index guard)"""
    p = np.ascontiguousarray(points[:, :3], f32)
    d = np.sqrt(p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1])
    ch, b = ref.cell_index(p)
    ok = (d > f32(r_min)) & (d < f32(r_max)) & (ch >= 0) & (ch < NCH) & (b >= 0) & (b < NBIN)
    return np.where(ok, ch * NBIN + b, -1)


def line_labels(points, cells, gz, tol=0.25):
    """step 4: (elevated mask, ground mask) of the in-window points"""
    z = np.asarray(points[:, 2], f32).astype(np.float64)
    inw = cells >= 0
    g = np.where(inw, gz.reshape(-1)[np.maximum(cells, 0)], f32(0)).astype(np.float64)
    ground = inw & (z < g + tol)
    return inw & ~ground, ground


def lowest_ground(pts, cells, gz, sensor_height):
    """step 5: g of a cluster's points (n, 3) with their cells: gz of its lowest point's cell (first in order), else -sensor_height"""
    j = int(np.argmin(np.asarray(pts[:, 2], f32)))
    c = int(cells[j])
    return f32(gz.reshape(-1)[c]) if c >= 0 else f32(-f32(sensor_height))


def cluster_members(elev, grid, k, roi=50.0, ng=250):
    """the point indices of clusters 1 .. k of elevated cloud `elev`, in cloud order, as boxFitting's getClusteredPoints reads them"""
    roi = f32(roi)
    xc = np.asarray(elev[:, 0], f32) + roi / f32(2)
    yc = np.asarray(elev[:, 1], f32) + roi / f32(2)
    ok = (xc >= 0) & (xc < roi) & (yc >= 0) & (yc < roi)
    xi = np.floor(f32(ng) * xc / roi).astype(np.int64)
    yi = np.floor(f32(ng) * yc / roi).astype(np.int64)
    lab = np.where(ok, grid.reshape(-1)[np.clip(xi, 0, ng - 1) * ng + np.clip(yi, 0, ng - 1)], 0)
    return [np.nonzero(lab == c)[0] for c in range(1, k + 1)]


def ref_lines_detect(rt, points, r_min=float(f32(3.4)), r_max=120.0, sensor_height=2.0, tol=0.25, fitter=None, search=None, **kw):
    """the reference's chain with ground lines (rt: oracle.ref_detect_tunable.RefDetectTunable): its polar grid's minZ -> host lines
    (restated) -> step 4 labels -> its componentClustering -> its boxFitting per cluster with sensorHeight = -g.  The unit values are
    lmot_params' floats, widened to double as the library does.  fitter: the oracle whose boxFitting and sensorHeight are used (default
    rt; oracle.ref.RefOracle("o2") for the other rule mode).  search: (box_search_scenes.RefSearch bound to fitter, A) -> box search's fit
    with the reference's ruleBasedFilter instead of boxFitting.
    -> dict(elev, ground, grid, k, boxes (m, 8, 3), gz)"""
    import ctypes as C
    fitter = fitter or rt
    sh = C.c_float.in_dll(fitter.lib, "sensorHeight")
    saved = sh.value
    minz = rt.polar_grid(points)["minz"]
    gz = lines_grid(minz, r_min, r_max, sensor_height, **kw)
    cells = window_cells(rt, points, r_min, r_max)
    e, g = line_labels(points, cells, gz, tol)
    elev = np.ascontiguousarray(points[e, :3], f32)
    grid, k = rt.component_clustering(elev)
    members = cluster_members(elev, grid, k)
    ecells = cells[e]
    boxes = []
    try:
        for c in range(1, k + 1):
            idx = members[c - 1]
            if len(idx) == 0:
                continue
            h = -lowest_ground(elev[idx], ecells[idx], gz, sensor_height)
            sh.value = float(h)
            if search is None:
                b, _ = fitter.box_fitting(elev, np.where(grid == c, 1, 0).astype(np.int32), 1)
            else:
                b = _searched(search, elev[idx], h)
            boxes.extend(list(b))
    finally:
        sh.value = saved
    return dict(elev=elev, ground=np.ascontiguousarray(points[g, :3], f32), grid=grid, k=k,
                boxes=np.array(boxes, f32).reshape(-1, 8, 3), gz=gz)


def _searched(search, pts, h, min_points=30):
    """box search's fit (box_search_scenes.fit) of one cluster's points with the reference's ruleBasedFilter at sensorHeight h"""
    from box_search_scenes import fit
    rs, A = search
    n = len(pts)
    if n < min_points:
        return []
    max_z = max(f32(-99.0), pts[:, 2].max())
    _, pc, _ = fit(pts, A)
    if not rs.rule(pc, max_z, n):
        return []
    b = np.zeros((8, 3), f32)
    b[:4, :2] = pc
    b[4:, :2] = pc
    b[:4, 2] = -f32(h)
    b[4:, 2] = max_z
    return [b]


# ------------------------------------------------------------------------------------------------ scenes
SCENES = {                     # name: (ground slope dz/dx, dz/dy), (sensor pitch, roll) in degrees
    "flat": ((0.0, 0.0), (0.0, 0.0)),
    "grade4": ((0.04, 0.0), (0.0, 0.0)),
    "grade8": ((0.08, 0.0), (0.0, 0.0)),
    "pitch3": ((0.0, 0.0), (3.0, 0.0)),
    "roll2": ((0.0, 0.0), (0.0, 2.0)),
}


def _rot(pitch_deg, roll_deg):
    """sensor -> world rotation of a sensor pitched about y, then rolled about x"""
    p, r = math.radians(pitch_deg), math.radians(roll_deg)
    ry = np.array([[math.cos(p), 0, math.sin(p)], [0, 1, 0], [-math.sin(p), 0, math.cos(p)]])
    rx = np.array([[1, 0, 0], [0, math.cos(r), -math.sin(r)], [0, math.sin(r), math.cos(r)]])
    return ry @ rx


def render(name, n_objects=40, seed=3, rings=64, azimuths=1875):
    """synth.py's ray caster with the ground plane z = -1.73 + gx*x + gy*y of the world and the sensor at the origin turned by
    (pitch, roll); objects stand on the ground.  -> (points (N, 4) float32 in the sensor frame, objects (K, 2): their centres' x, y in
    the sensor frame)"""
    (gx, gy), (pitch, roll) = SCENES[name]
    cfg = synth.SceneConfig(rings=rings, azimuths=azimuths, n_objects=n_objects, seed=seed)
    sc = synth.make_scene(cfg)
    R = _rot(pitch, roll)
    rng = np.random.default_rng((cfg.seed << 20) + 1)
    elev = np.deg2rad(np.linspace(cfg.elev_top_deg, cfg.elev_bot_deg, rings))
    az = (np.arange(azimuths) + 0.5) * (2 * math.pi / azimuths) - math.pi
    ce, se = np.cos(elev)[:, None], np.sin(elev)[:, None]
    ds = np.stack([ce * np.cos(az)[None, :], ce * np.sin(az)[None, :], np.broadcast_to(se, (rings, azimuths))], -1)
    dw = ds @ R.T                                   # each ray in the world frame
    dx, dy, dz = dw[..., 0], dw[..., 1], dw[..., 2]
    z0 = synth.SENSOR_Z_GROUND
    den = dz - gx * dx - gy * dy
    with np.errstate(divide="ignore"):
        t_ground = np.where(den < -1e-9, z0 / den, np.inf)
    t_wall = synth.WALL_R / np.maximum(np.hypot(dx, dy), 1e-9)
    t = np.minimum(t_ground, t_wall)
    for k in range(len(sc.pos)):
        cx, cy = sc.pos[k]
        L, W, H = sc.size[k]
        base = z0 + gx * cx + gy * cy
        c, s = math.cos(sc.yaw[k]), math.sin(sc.yaw[k])
        obx, oby = c * -cx + s * -cy, -s * -cx + c * -cy
        bdx, bdy = c * dx + s * dy, -s * dx + c * dy
        tmin = np.full(dx.shape, -np.inf)
        tmax = np.full(dx.shape, np.inf)
        for o, dd, lo, hi in ((obx, bdx, -L / 2, L / 2), (oby, bdy, -W / 2, W / 2), (0.0, dz, base, base + H)):
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / np.where(np.abs(dd) < 1e-12, 1e-12, dd)
            t1, t2 = (lo - o) * inv, (hi - o) * inv
            tmin = np.maximum(tmin, np.minimum(t1, t2))
            tmax = np.minimum(tmax, np.maximum(t1, t2))
        hit = (tmax >= np.maximum(tmin, 0.0)) & (tmin > 0.0) & (tmin < t)
        t = np.where(hit, tmin, t)
    t = t + rng.normal(0.0, cfg.range_noise, size=t.shape)
    pts = np.concatenate([(ds * t[..., None]).reshape(-1, 3), np.full((rings * azimuths, 1), 0.5)], 1).astype(f32)
    cz = z0 + gx * sc.pos[:, 0] + gy * sc.pos[:, 1] + sc.size[:, 2] / 2
    centres = np.stack([sc.pos[:, 0], sc.pos[:, 1], cz], 1) @ R          # world -> sensor frame
    return pts, centres[:, :2]


def objects_found(boxes, objects, radius=2.0):
    """objects with a box whose centre (mean of its four bottom corners) lies within `radius` of theirs"""
    b = np.asarray(boxes, np.float64).reshape(-1, 8, 3)
    if len(b) == 0:
        return 0
    c = b[:, :4, :2].mean(1)
    d = np.hypot(objects[:, None, 0] - c[None, :, 0], objects[:, None, 1] - c[None, :, 1])
    return int((d.min(1) <= radius).sum())
