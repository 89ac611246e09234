"""Background subtraction for stationary sensors, as considered in DESIGN.md §6n, restated in NumPy, and a stationary-sensor scene to
measure it on.  Shared by test_background_cpu.py and scripts/background_premise.py.

The definition, per sensor, with every step in float32 (IEEE round to nearest, no fused multiply-add):
  cell of a point (x, y, z) in the sensor's frame:
    rxy = sqrt(x * x + y * y), r = sqrt((x * x + y * y) + z * z), az = atan2f(y, x), el = atan2f(z, rxy);
    col = floor((az + PI) / TWO_PI * cols), clamped to cols - 1;
    row = floor((el - el_min) / (el_max - el_min) * rows); a point with row outside [0, rows) has no cell.
    PI, TWO_PI are pi and 2 pi rounded to float; el_min, el_max are the window's degrees times pi / 180 in double, rounded to float.
  learning, frames 1..L, over every point the ground removal keeps (ground and elevated):
    hits[c] += 1 for every cell c that at least one point of the frame falls in; B[c] = max(B[c], r), B starting at 0.
  freeze, at the end of frame L:
    B[c] = +inf where hits[c] < ceil(min_hit_frac * L) (min_hit_frac as float, the product in double);
    Bn[row, col] = min of B over rows row - nbr_rows .. row + nbr_rows (clipped at the window) and columns col - nbr_cols .. col +
    nbr_cols (wrapping around).
  filter: a point of the elevated cloud E is kept iff it has no cell or r < Bn[c] - margin_m (float subtraction); E_fg keeps E's order.
atan2f is numpy's float32 arctan2, which is the host libm's atan2f here (test_host_cpu.py::test_atan2f_restatement_equals_host_libm).
"""
import math

import numpy as np

import detect_area_scenes as das
import layer_scenes as ls
import weather_scenes as ws

f32 = np.float32
PI = f32(math.pi)
TWO_PI = f32(2.0 * math.pi)
DEFAULTS = dict(rows=64, elev_min_deg=-25.0, elev_max_deg=3.0, cols=1800, learn_frames=50, min_hit_frac=0.5, margin_m=0.3,
                nbr_cols=1, nbr_rows=0)
MAX_ROWS, MAX_COLS = 128, 4096


def validate(rows, elev_min_deg, elev_max_deg, cols, learn_frames, min_hit_frac, margin_m, nbr_cols, nbr_rows):
    """the setting's limits; raises ValueError"""
    ok = (1 <= rows <= MAX_ROWS and 1 <= cols <= MAX_COLS and learn_frames >= 1 and np.isfinite(elev_min_deg)
          and np.isfinite(elev_max_deg) and -90.0 <= elev_min_deg < elev_max_deg <= 90.0 and 0.0 <= min_hit_frac <= 1.0
          and np.isfinite(margin_m) and margin_m >= 0.0 and 0 <= nbr_cols < cols and 0 <= nbr_rows < rows)
    if not ok:
        raise ValueError("invalid background setting")


def window(elev_min_deg, elev_max_deg, **_):
    lo = f32(float(elev_min_deg) * (math.pi / 180.0))
    hi = f32(float(elev_max_deg) * (math.pi / 180.0))
    return lo, hi, f32(hi - lo)


def cells(points, rows=64, elev_min_deg=-25.0, elev_max_deg=3.0, cols=1800, **_):
    """-> (cell index row * cols + col, -1 for no cell (int64), r (float32)) of every point"""
    p = np.asarray(points, f32).reshape(len(points), -1)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(invalid="ignore", over="ignore"):
        s = x * x + y * y
        rxy = np.sqrt(s)
        r = np.sqrt(s + z * z)
        az = np.arctan2(y, x)
        el = np.arctan2(z, rxy)
        colf = np.floor((az + PI) / TWO_PI * f32(cols))
        col = np.minimum(np.where(colf == colf, colf, 0).astype(np.int64), cols - 1)
        lo, _, span = window(elev_min_deg, elev_max_deg)
        rowf = np.floor((el - lo) / span * f32(rows))
    has = (rowf >= 0) & (rowf < rows) & (colf == colf)
    row = np.where(has, rowf, 0).astype(np.int64)
    return np.where(has, row * cols + col, -1), r


class Learner:
    """hits and B of one sensor's table while it learns"""

    def __init__(self, **cfg):
        self.c = dict(DEFAULTS, **cfg)
        n = self.c["rows"] * self.c["cols"]
        self.hits = np.zeros(n, np.int64)
        self.B = np.zeros(n, f32)
        self.frames = 0

    def learn(self, kept_points):
        c, r = cells(kept_points, **self.c)
        m = c >= 0
        c, r = c[m], r[m]
        self.hits[np.unique(c)] += 1
        np.maximum.at(self.B, c, r)
        self.frames += 1

    def freeze(self, **cfg):
        """Bn (rows, cols) float32 from what was learned; cfg overrides min_hit_frac, nbr_cols, nbr_rows"""
        c = dict(self.c, **cfg)
        return freeze(self.hits, self.B, self.frames, **c)


def freeze(hits, B, frames, rows, cols, min_hit_frac, nbr_cols, nbr_rows, **_):
    need = math.ceil(float(f32(min_hit_frac)) * frames)
    t = np.where(np.asarray(hits).reshape(rows, cols) < need, f32(np.inf), np.asarray(B, f32).reshape(rows, cols))
    out = t.copy()
    for dc in range(-nbr_cols, nbr_cols + 1):
        out = np.minimum(out, np.roll(t, -dc, axis=1))
    t, out = out, out.copy()
    for dr in range(1, nbr_rows + 1):
        out[:-dr] = np.minimum(out[:-dr], t[dr:])
        out[dr:] = np.minimum(out[dr:], t[:-dr])
    return out


def freeze_brute(hits, B, frames, rows, cols, min_hit_frac, nbr_cols, nbr_rows, **_):
    """the freeze rule by the letter, one cell at a time"""
    need = math.ceil(float(f32(min_hit_frac)) * frames)
    hits = np.asarray(hits).reshape(rows, cols)
    B = np.asarray(B, f32).reshape(rows, cols)
    out = np.empty((rows, cols), f32)
    for i in range(rows):
        for j in range(cols):
            m = f32(np.inf)
            for a in range(max(0, i - nbr_rows), min(rows, i + nbr_rows + 1)):
                for d in range(-nbr_cols, nbr_cols + 1):
                    b = (j + d) % cols
                    v = B[a, b] if hits[a, b] >= need else f32(np.inf)
                    m = min(m, v)
            out[i, j] = m
    return out


def keep_flags(elevated, Bn, margin_m=0.3, **cfg):
    c, r = cells(elevated, **dict(DEFAULTS, **cfg))
    has = c >= 0
    bn = np.where(has, Bn.reshape(-1)[np.where(has, c, 0)], f32(np.inf))
    with np.errstate(invalid="ignore"):
        return ~has | (r < bn - f32(margin_m))


def foreground(elevated, Bn, margin_m=0.3, **cfg):
    e = np.asarray(elevated, f32)
    return np.ascontiguousarray(e[keep_flags(e, Bn, margin_m, **cfg)])


# ------------------------------------------------------------------------------------------------ a stationary-sensor scene
def static_solids(seed):
    """(cx, cy, yaw, L, W, z0, z1 above the ground) of the scene's static structure: detect_area_scenes' poles and hedges, the tree trunks
    and canopies, shelter roofs and posts and the sign gantry of layer_scenes, and layer_scenes' cars and truck, parked for good"""
    out = [(x, y, 0.0, L, W, 0.0, H) for x, y, L, W, H in das.CLUTTER]
    solids, _ = ls._boxes_of(np.random.default_rng(seed), "64")
    for s in solids:
        _, _, _, L, W, z0, z1 = s
        is_ped = L <= 0.6 and W <= 0.6 and z0 == 0.0 and z1 < 2.0
        if not is_ped:
            out.append(s)
    return out


def render(sensor, solids, movers, rng):
    """ray cast synth.py's ground and wall, the static solids and the movers (cx, cy, yaw, L, W, H) from a sensor 1.73 m above flat
    ground -> XYZI float32, ring-major, gaussian range noise of 0.03 m drawn from rng"""
    import importlib
    synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
    cfg = synth.SceneConfig(**ws.SENSORS[sensor])
    elev = np.deg2rad(np.linspace(cfg.elev_top_deg, cfg.elev_bot_deg, cfg.rings))
    az = (np.arange(cfg.azimuths) + 0.5) * (2 * math.pi / cfg.azimuths) - math.pi
    ce, se = np.cos(elev)[:, None], np.sin(elev)[:, None]
    dx, dy = ce * np.cos(az)[None, :], ce * np.sin(az)[None, :]
    dz = np.broadcast_to(se, dx.shape)
    z0 = synth.SENSOR_Z_GROUND
    with np.errstate(divide="ignore"):
        t = np.where(dz < -1e-9, z0 / dz, np.inf)
    t = np.minimum(t, synth.WALL_R / np.maximum(np.hypot(dx, dy), 1e-9))
    for cx, cy, yaw, L, W, h0, h1 in list(solids) + [(x, y, w, L, W_, 0.0, H) for x, y, w, L, W_, H in movers]:
        c, s = math.cos(yaw), math.sin(yaw)
        obx, oby = c * -cx + s * -cy, -s * -cx + c * -cy
        bdx, bdy = c * dx + s * dy, -s * dx + c * dy
        tmin = np.full(dx.shape, -np.inf)
        tmax = np.full(dx.shape, np.inf)
        for o, dd, lo, hi in ((obx, bdx, -L / 2, L / 2), (oby, bdy, -W / 2, W / 2), (0.0, dz, z0 + h0, z0 + h1)):
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / np.where(np.abs(dd) < 1e-12, 1e-12, dd)
            t1, t2 = (lo - o) * inv, (hi - o) * inv
            tmin = np.maximum(tmin, np.minimum(t1, t2))
            tmax = np.minimum(tmax, np.maximum(t1, t2))
        hit = (tmax >= np.maximum(tmin, 0.0)) & (tmin > 0.0) & (tmin < t)
        t = np.where(hit, tmin, t)
    t = t + rng.normal(0.0, 0.03, size=t.shape)
    ds = np.stack([dx, dy, dz], -1)
    return np.concatenate([(ds * t[..., None]).reshape(-1, 3), np.full((t.size, 1), 0.5)], 1).astype(f32)


MODES = ("moving", "leave", "arrive")


def _corners(cx, cy, yaw, L, W, grow=0.0):
    c, s = math.cos(yaw), math.sin(yaw)
    h = np.array([[1, 1], [1, -1], [-1, -1], [-1, 1]]) * [L / 2 + grow, W / 2 + grow]
    return np.stack([cx + c * h[:, 0] - s * h[:, 1], cy + s * h[:, 0] + c * h[:, 1]], 1)


def overlap(a, b, grow=0.0):
    """footprints a, b = (cx, cy, yaw, L, W) overlap once a grows by grow on every side (separating axes)"""
    pa, pb = _corners(*a[:5], grow), _corners(*b[:5])
    for yaw in (a[2], a[2] + math.pi / 2, b[2], b[2] + math.pi / 2):
        ax = np.array([math.cos(yaw), math.sin(yaw)])
        u, v = pa @ ax, pb @ ax
        if u.max() < v.min() or v.max() < u.min():
            return False
    return True


def stationary_frames(synth, sensor, mode, learn_frames, scored_frames, seed, n_objects=40, clear=0.5):
    """[(points, scored object centres (K, 2), learned (K,) bool, learning)] per frame from a sensor that does not move.  synth.py's
    objects that move are the movers, advanced by synth.advance; the ones synth.py leaves standing are parked, like static_solids.
      moving: every mover moves through learning and scoring.
      leave:  every second mover stands still through learning (parked), then drives off.
      arrive: every second mover is absent during learning, then appears and parks where synth.py's scene had it at that time.
    Scored objects: the movers, including those that park or leave.  synth.py does not keep its objects apart, so a parked object or a
    ground-standing static solid that a mover ever comes within `clear` of is left out of the scene: a car cannot drive through a hedge.
    learned: the object's footprint at this frame overlaps its own in every learning frame, so the object is in the background table
    where it now stands."""
    sc = synth.make_scene(synth.SceneConfig(seed=seed, n_objects=n_objects, **ws.SENSORS[sensor]))
    moving = sc.vel > 0
    special = np.zeros(len(sc.vel), bool)
    special[np.flatnonzero(moving)[::2]] = True
    vel = sc.vel.copy()
    path = []                                             # per frame: (footprints (K, 5) of the movers, shown (K,))
    for f in range(learn_frames + scored_frames):
        learning = f < learn_frames
        show = np.ones(len(vel), bool)
        if mode == "leave":
            sc.vel = np.where(special & learning, 0.0, vel)
        if mode == "arrive":
            show = ~special if learning else show
            sc.vel = vel if learning else np.where(special, 0.0, vel)
        path.append((np.concatenate([sc.pos, sc.yaw[:, None], sc.size[:, :2]], 1)[moving], show[moving]))
        synth.advance(sc)
    sc0 = synth.make_scene(synth.SceneConfig(seed=seed, n_objects=n_objects, **ws.SENSORS[sensor]))
    standing = [(*sc0.pos[k], sc0.yaw[k], *sc0.size[k][:2], 0.0, sc0.size[k][2]) for k in np.flatnonzero(~moving)]
    standing += list(static_solids(seed))
    heights = {k: sc0.size[k][2] for k in np.flatnonzero(moving)}

    def clear_of_movers(s):
        if s[5] > 0.0:                                    # overhead: canopies, roofs, the gantry beam
            return True
        return not any(overlap(fp, s, clear) for fps, shown in path for fp in fps[shown])

    solids = [s for s in standing if clear_of_movers(s)]
    rng = np.random.default_rng(seed)
    hz = np.array([heights[k] for k in np.flatnonzero(moving)])
    out = []
    for f, (fps, shown) in enumerate(path):
        learning = f < learn_frames
        pts = render(sensor, solids, [(*fp, h) for fp, h in zip(fps[shown], hz[shown])], rng)
        learned = np.array([all(overlap(fp, path[j][0][i]) for j in range(learn_frames) if path[j][1][i])
                            and any(path[j][1][i] for j in range(learn_frames)) for i, fp in enumerate(fps) if shown[i]], bool)
        out.append((pts, fps[shown, :2].copy(), learned, learning))
    return out


def matched(boxes, obj, tol=1.0):
    """(per object: a box centre lies within tol of its centre, ghost boxes: boxes within tol of no object)"""
    c = ws.centres(boxes)
    if len(c) == 0:
        return np.zeros(len(obj), bool), 0
    d = np.hypot(c[:, None, 0] - obj[None, :, 0], c[:, None, 1] - obj[None, :, 1]) <= tol
    return d.any(0), int((~d.any(1)).sum())


def ref_boxes(ref, e):
    """the reference's componentClustering and boxFitting on the elevated cloud e"""
    grid, k = ref.component_clustering(e)
    return ref.box_fitting(e, grid, k)[0]
