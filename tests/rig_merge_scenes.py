"""Scenes and oracles of merging rigs (lmot_set_rig_merge): numpy and the compiled reference only, no device.

Overlapping scene: one synth frame per tick is the vehicle's view.  Sensor k of a rig is yawed by a quarter turn q_k and sees the rows whose
vehicle-frame azimuth lies in its half-open 180 degree field of view; its cloud is those rows rotated into its own frame (a quarter-turn
rotation: exact) with z shifted by its mounting height as rig_ticks does.  Its pose maps every point back onto the same vehicle-frame
scene, so where fields of view overlap the same object arrives from two sensors.

The vehicle frame's origin sits h_vehicle above the ground (lmot_params.sensor_height in merged mode): a sensor at height h has pose
translation z = h - h_vehicle.

Merged oracle: reference ground removal per sensor (its mount), every elevated cloud through the rig arithmetic (rig_apply), the clouds
concatenated in table order (cut at max_points), then reference clustering and box fitting with sensorHeight = h_vehicle.
"""
import contextlib
import ctypes as C
import math

import numpy as np

from test_sensor_rig_gpu import H_DEFAULT, mount, ref_mount, rig_apply, yaw_pose

f32 = np.float32
QUARTER = [(1, 0), (0, 1), (-1, 0), (0, -1)]          # (cos, sin) of yaw 0, pi/2, pi, -pi/2


def overlap_rig(n, heights=None, h_vehicle=H_DEFAULT):
    """n sensors, sensor k yawed by quarter turn k % 4 (n = 2: yaws 0 and pi, fields of view that only touch), mounted at heights[k].
    -> [(pose 3x4, h, quarter)]"""
    heights = heights if heights is not None else [H_DEFAULT] * n
    qs = [0, 2] if n == 2 else [k % 4 for k in range(n)]
    return [(yaw_pose(*QUARTER[q], 0.0, 0.0, f32(h) - f32(h_vehicle)), h, q) for q, h in zip(qs, heights)]


def _in_fov(pts, q, full):
    if full:
        return np.ones(len(pts), bool)
    a = np.arctan2(pts[:, 1].astype(np.float64), pts[:, 0].astype(np.float64))
    d = (a - q * math.pi / 2 + math.pi) % (2 * math.pi) - math.pi
    return (d >= -math.pi / 2) & (d < math.pi / 2)


def sensor_cloud(view, q, h, full=False):
    """the rows of the vehicle's view (synth frame) sensor (q, h) sees, in its own frame"""
    p = view[_in_fov(view, q, full)].copy()
    c, s = QUARTER[q]
    x, y = p[:, 0].copy(), p[:, 1].copy()
    p[:, 0] = c * x + s * y                            # R^T (x, y) for a quarter turn: exact
    p[:, 1] = -s * x + c * y
    p[:, 2] += f32(H_DEFAULT - h)
    return np.ascontiguousarray(p)


def overlap_ticks(synth, rig, n_ticks, seed=5, n_objects=30, rings=32, azimuths=900):
    """(ts, [sensor clouds], scene positions (K, 2) in the vehicle frame, sizes (K, 3)) per tick"""
    cfg = synth.SceneConfig(seed=seed, n_objects=n_objects, rings=rings, azimuths=azimuths)
    sc = synth.make_scene(cfg)
    full = len(rig) == 1
    for f in range(n_ticks):
        view = synth.render(sc)
        yield (f + 1) * synth.DT_US, [sensor_cloud(view, q, h, full) for _, h, q in rig], sc.pos.copy(), sc.size.copy()
        synth.advance(sc)


@contextlib.contextmanager
def ref_vehicle(ref, h_vehicle):
    """the reference's sensorHeight (box_fitting.cpp:26) = the vehicle frame origin's height while the block runs"""
    g = C.c_float.in_dll(ref.lib, "sensorHeight")
    saved = g.value
    assert saved == float(f32(H_DEFAULT)), saved
    g.value = h_vehicle
    try:
        yield
    finally:
        g.value = saved


def merged_detection(ref, rig, frames, h_vehicle=H_DEFAULT, max_points=1 << 20):
    """-> (rows [(n_elev, n_ground, num_cluster, n_boxes)] per sensor as lmot_batch_out reports them, the box list, merged cloud, cut)"""
    rows, E = [], []
    for pts, (pose, h, _) in zip(frames, rig):
        with ref_mount(ref, h):
            e, g = ref.ground_remove(pts)
        rows.append([len(e), len(g), 0, 0])
        E.append(rig_apply(pose, e))
    E = np.concatenate(E).astype(f32)
    cut = len(E) > max_points
    E = E[:max_points]
    with ref_vehicle(ref, h_vehicle):
        grid, k = ref.component_clustering(E)
        b, _ = ref.box_fitting(E, grid, k)
    rows[0][2], rows[0][3] = k, len(b)
    return [tuple(r) for r in rows], b, E, cut


def separate_detection(ref, rig, frames):
    """the rig without merge: each sensor's boxes under its own mount, moved into the vehicle frame, concatenated"""
    lists = []
    for pts, (pose, h, _) in zip(frames, rig):
        with ref_mount(ref, h):
            e, _ = ref.ground_remove(pts)
            grid, k = ref.component_clustering(e)
            b, _ = ref.box_fitting(e, grid, k)
        lists.append(rig_apply(pose, b))
    return np.concatenate(lists) if lists else np.zeros((0, 8, 3), f32)


def doubled_view_detection(ref, view):
    """the reference on the vehicle's whole view as one 360 degree sensor at the origin would see it, its elevated cloud taken TWICE:
    what the merged cloud of a rig whose fields of view cover every direction exactly twice amounts to (same points, each twice)"""
    e, _ = ref.ground_remove(view)
    E = np.concatenate([e, e])
    grid, k = ref.component_clustering(E)
    b, _ = ref.box_fitting(E, grid, k)
    return b


def boxes_per_object(boxes, pos, size):
    """number of boxes whose centre lies nearest to each ground-truth object and inside its footprint circle (+0.5 m)"""
    counts = np.zeros(len(pos), int)
    if len(boxes) == 0:
        return counts
    ctr = boxes.reshape(-1, 8, 3)[:, :, :2].astype(np.float64).mean(1)
    d = np.hypot(ctr[:, None, 0] - pos[None, :, 0], ctr[:, None, 1] - pos[None, :, 1])
    near = d.argmin(1)
    reach = 0.5 * np.hypot(size[:, 0], size[:, 1]) + 0.5
    for i, j in enumerate(near):
        if d[i, j] <= reach[j]:
            counts[j] += 1
    return counts


def table_kw(rig):
    """set_sensors / seq_set_sensors keyword arguments of a rig (each sensor's mount)"""
    ms = [mount(h) for _, h, _ in rig]
    return dict(poses=[p for p, _, _ in rig], **{k: [m[k] for m in ms] for k in ms[0]})
