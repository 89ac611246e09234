"""Layered clustering (include/lmot.h, lmot_set_layers): steps 1-6 restated once in NumPy, the per-cluster reference oracle of step 7,
and ray-cast scenes where objects stand under canopies, shelter roofs and a sign gantry.  Shared by test_layers_cpu.py and
test_layers_gpu.py."""
import importlib
import math

import numpy as np
from scipy import ndimage

f32 = np.float32
GRID = 250
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")


# ------------------------------------------------------------------------------------------------ steps 1-6
def columns(points, roi=50.0):
    """step 1: componentClustering's float binning -> (xI, yI, has a column) per point, in float32"""
    p = np.asarray(points, f32)
    roi = f32(roi)
    half = roi / f32(2)
    xc, yc = p[:, 0] + half, p[:, 1] + half
    ok = (xc >= 0) & (xc < roi) & (yc >= 0) & (yc < roi)
    xi = np.clip(np.floor((f32(GRID) * xc) / roi).astype(np.int64), 0, GRID - 1)
    yi = np.clip(np.floor((f32(GRID) * yc) / roi).astype(np.int64), 0, GRID - 1)
    return xi, yi, ok


def slices(points, sensor_height, n_slices=32, slice_m=0.2, z_min=-0.5):
    """step 2: ((double)z + (double)sensor_height) - z_min, divided by slice_m, floored, clamped"""
    z = np.asarray(points, f32)[:, 2].astype(np.float64)
    h = (z + float(f32(sensor_height))) - float(z_min)
    return np.clip(np.floor(h / float(slice_m)), 0, n_slices - 1).astype(np.int64)


def point_clusters(points, sensor_height=2.0, n_slices=32, slice_m=0.2, z_min=-0.5, gap_slices=2, roi=50.0):
    """steps 1-6 of one unit's cloud E (N, >=3) -> (ids (N,) int32, num_cluster); sensor_height: lmot_params' default (the reference's
    sensorHeight), which the scenes' sensor 1.73 m above the ground does not change"""
    pts = np.asarray(points, f32)
    S, g = int(n_slices), int(gap_slices)
    ids = np.zeros(len(pts), np.int32)
    if len(pts) == 0:
        return ids, 0
    xi, yi, ok = columns(pts, roi)
    s = slices(pts, sensor_height, S, slice_m, z_min)
    count = np.zeros((GRID, GRID), np.int64)
    np.add.at(count, (xi[ok], yi[ok]), 1)
    seed = ok & (count[xi, yi] > 1)
    V = np.zeros((GRID, GRID, S), bool)
    V[xi[seed], yi[seed], s[seed]] = True
    O = ndimage.maximum_filter(V.astype(np.uint8), size=(3, 3, 2 * g + 1), mode="constant", cval=0).astype(bool)
    lab, k = ndimage.label(O, structure=np.ones((3, 3, 3), bool))
    if k == 0:
        return ids, 0
    # ids in the order of each component's smallest (x, y, s), x outermost (the C order of O)
    first = ndimage.minimum(np.arange(O.size).reshape(O.shape), lab, np.arange(1, k + 1))
    rank = np.empty(k + 1, np.int32)
    rank[0] = 0
    rank[1 + np.argsort(np.asarray(first))] = np.arange(1, k + 1, dtype=np.int32)
    ids[ok] = rank[lab[xi[ok], yi[ok], s[ok]]]
    return ids, k


# ------------------------------------------------------------------------------------------------ step 7: the per-cluster reference oracle
def oracle_boxes(ref, elev, ids, k, roi=50.0):
    """boxFitting(E_c, grid_c, 1) of the reference per cluster c = 1 .. k, accepted boxes in id order (ref: oracle.ref.RefOracle, whose
    sensorHeight is the unit's) -> (m, 8, 3) float32"""
    pts = np.ascontiguousarray(np.asarray(elev, f32)[:, :3])
    xi, yi, _ = columns(pts, roi)
    out = []
    for c in range(1, k + 1):
        sel = np.nonzero(ids == c)[0]
        if len(sel) == 0:
            continue
        grid = np.zeros((GRID, GRID), np.int32)
        grid[xi[sel], yi[sel]] = 1
        b, _ = ref.box_fitting(pts[sel], grid, 1)
        out.extend(list(b))
    return np.array(out, f32).reshape(-1, 8, 3)


def ref_layers_detect(ref, points, **layers):
    """the reference's groundRemove, then steps 1-7 on its elevated cloud -> dict(elev, ids, k, boxes)"""
    e, _ = ref.ground_remove(points)
    ids, k = point_clusters(e, **layers)
    return dict(elev=e, ids=ids, k=k, boxes=oracle_boxes(ref, e, ids, k))


# ------------------------------------------------------------------------------------------------ scenes
SENSORS = {                    # name: (rings, azimuths, top, bottom elevation in degrees)
    "64": (64, 1800, 15.0, -25.0),
    "32": (32, 1800, 10.67, -30.67),
}


def _boxes_of(rng, kind):
    """solids (cx, cy, yaw, L, W, z0, z1 above the ground) of the scene, and the objects a box should be found for: (cx, cy, kind)"""
    solids, objects = [], []
    occupied = []

    def place(r_lo, r_hi, clear):
        for _ in range(200):
            r, a = rng.uniform(r_lo, r_hi), rng.uniform(-math.pi, math.pi)
            x, y = r * math.cos(a), r * math.sin(a)
            if abs(x) < 22 and abs(y) < 22 and all(math.hypot(x - ox, y - oy) > clear + oc for ox, oy, oc in occupied):
                occupied.append((x, y, clear))
                return x, y
        raise RuntimeError("scene too full")

    for _ in range(5):                                     # cars under tree canopies: trunk 1.8 m from the car, canopy 3-7 m
        x, y = place(6, 22, 3.2)
        yaw = rng.uniform(0, math.pi)
        solids.append((x, y, yaw, 4.4, 1.8, 0.0, 1.5))
        objects.append((x, y, "car_canopy"))
        tx, ty = x + 1.8 * -math.sin(yaw) * 1.2, y + 1.8 * math.cos(yaw) * 1.2
        solids.append((tx, ty, 0.0, 0.35, 0.35, 0.0, 3.2))
        solids.append((x, y, yaw + 0.3, 6.0, 5.0, 3.0, 7.0))
    for _ in range(3):                                     # pedestrians under a 2.5 m shelter roof on two posts
        x, y = place(6, 20, 2.2)
        yaw = rng.uniform(0, math.pi)
        c, s = math.cos(yaw), math.sin(yaw)
        solids.append((x, y, yaw, 4.0, 2.0, 2.5, 2.7))
        for d in (-1.8, 1.8):
            solids.append((x + c * d - s * 0.9, y + s * d + c * 0.9, yaw, 0.15, 0.15, 0.0, 2.5))
        solids.append((x, y - 0.0, yaw, 0.5, 0.6, 0.0, 1.75))
        objects.append((x, y, "ped_shelter"))
    x, y = place(8, 22, 3.0)                              # a car under a 5.5 m sign gantry
    yaw = rng.uniform(0, math.pi)
    c, s = math.cos(yaw), math.sin(yaw)
    solids.append((x, y, yaw, 4.4, 1.8, 0.0, 1.5))
    solids.append((x, y, yaw + math.pi / 2, 12.0, 0.8, 5.5, 6.5))
    for d in (-6.0, 6.0):
        solids.append((x - s * d, y + c * d, 0.0, 0.4, 0.4, 0.0, 5.5))
    objects.append((x, y, "car_gantry"))
    x, y = place(8, 22, 4.0)                               # a 3.5 m truck (must not split)
    solids.append((x, y, rng.uniform(0, math.pi), 8.0, 2.5, 0.0, 3.5))
    objects.append((x, y, "truck"))
    for _ in range(5):                                     # open-field cars and pedestrians
        x, y = place(5, 22, 2.4)
        solids.append((x, y, rng.uniform(0, math.pi), 4.4, 1.8, 0.0, 1.5))
        objects.append((x, y, "car_open"))
    for _ in range(3):
        x, y = place(5, 18, 1.0)
        solids.append((x, y, 0.0, 0.5, 0.6, 0.0, 1.75))
        objects.append((x, y, "ped_open"))
    return solids, objects


def render(sensor="64", seed=7):
    """a flat-ground scene ray cast from a sensor 1.73 m above the ground -> (points (N, 4) float32, objects [(x, y, kind)])"""
    rings, azimuths, top, bot = SENSORS[sensor]
    rng = np.random.default_rng(seed)
    solids, objects = _boxes_of(rng, sensor)
    elev = np.deg2rad(np.linspace(top, bot, rings))
    az = (np.arange(azimuths) + 0.5) * (2 * math.pi / azimuths) - math.pi
    ce, se = np.cos(elev)[:, None], np.sin(elev)[:, None]
    dx, dy = ce * np.cos(az)[None, :], ce * np.sin(az)[None, :]
    dz = np.broadcast_to(se, (rings, azimuths))
    z0 = synth.SENSOR_Z_GROUND
    with np.errstate(divide="ignore"):
        t = np.where(dz < -1e-9, z0 / dz, np.inf)
    t = np.minimum(t, synth.WALL_R / np.maximum(np.hypot(dx, dy), 1e-9))
    for cx, cy, yaw, L, W, h0, h1 in solids:
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
    t = t + rng.normal(0.0, 0.02, size=t.shape)
    ds = np.stack([dx, dy, dz], -1)
    pts = np.concatenate([(ds * t[..., None]).reshape(-1, 3), np.full((rings * azimuths, 1), 0.5)], 1).astype(f32)
    return pts, objects


def found(boxes, objects, kind_prefix="", radius=1.5):
    """objects of the kinds starting with kind_prefix that have a box whose bottom centre lies within radius of theirs"""
    b = np.asarray(boxes, np.float64).reshape(-1, 8, 3)
    sel = [(x, y) for x, y, k in objects if k.startswith(kind_prefix)]
    if len(b) == 0 or not sel:
        return 0
    c = b[:, :4, :2].mean(1)
    o = np.array(sel)
    d = np.hypot(o[:, None, 0] - c[None, :, 0], o[:, None, 1] - c[None, :, 1])
    return int((d.min(1) <= radius).sum())
