"""Python-side mirror of the C ABI in include/lmot.h (ctypes; used by tests/, bench.py and __graft_entry__).

The product is liblmot.so (CUDA kernels for sm_90a behind `extern "C"`).  This module only loads it and
marshals numpy arrays / raw device pointers; it contains NO implementation of any pipeline stage and there is
no CPU fallback: if the library is missing or no CUDA device is usable, construction raises.

Entry points mirror the reference's four free functions (SURVEY.md §8b):
    Lmot.ground_remove(points)            <- groundRemove           ground_removal.cpp:177
    Lmot.component_cluster(elevated)      <- componentClustering    component_clustering.cpp:260
    Lmot.box_fit(elevated, grid, k)       <- boxFitting             box_fitting.cpp:422
    Lmot.track_step(boxes, ts, v, yaw)    <- getOriginPoints + immUkfJpdaf   imm_ukf_jpda.cpp:74,704
    Lmot.frame(points, ts, v, yaw)        <- all four, device resident between stages

The directory name is not a Python identifier; import it with
    importlib.import_module("3d-lidar-multi-object-tracking_b200")
"""
from __future__ import annotations

import ctypes as C
import os

# The frame pipeline uses up to 8 detection streams + 1 tracker stream per context; with the default of 8 hardware
# work queues streams alias and serialise each other.  Must be set before the CUDA context exists.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "liblmot.so")
TRACK_DUMP_DOUBLES = 236

OK, ERR_INVALID, ERR_CUDA, ERR_CAPACITY, ERR_STATE = 0, -1, -2, -3, -4
WARN_TRACK_TABLE_FULL = 1
RULE_INTENDED, RULE_GCC13_O2_COMPAT = 0, 1


class LmotError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"lmot status {status}: {msg}")
        self.status = status


class Params(C.Structure):
    _fields_ = [
        ("r_min", C.c_float), ("r_max", C.c_float), ("t_hmin", C.c_float), ("t_hmax", C.c_float),
        ("t_hdiff", C.c_float), ("h_sensor", C.c_float), ("ground_tolerance", C.c_double),
        ("roi_m", C.c_float),
        ("ram_points", C.c_int), ("l_slope_dist", C.c_int), ("l_num_points", C.c_int), ("sensor_height", C.c_float),
        ("t_height_min", C.c_float), ("t_height_max", C.c_float), ("t_width_min", C.c_float), ("t_width_max", C.c_float),
        ("t_len_min", C.c_float), ("t_len_max", C.c_float), ("t_area_max", C.c_float),
        ("t_ratio_min", C.c_float), ("t_ratio_max", C.c_float), ("min_len_ratio", C.c_float), ("t_pt_per_m3", C.c_float),
        ("min_cluster_points", C.c_int), ("rule_filter", C.c_int),
        ("oracle_compat_first_frame", C.c_int),
        ("max_points", C.c_int), ("max_clusters", C.c_int), ("max_boxes", C.c_int), ("max_tracks", C.c_int),
        ("node_prefilter", C.c_int), ("filter_z_min", C.c_float), ("filter_z_max", C.c_float),
        ("filter_x_min", C.c_float), ("filter_x_max", C.c_float), ("filter_y_min", C.c_float), ("filter_y_max", C.c_float),
        ("global_frame", C.c_int),
        ("pipeline_depth", C.c_int), ("result_ring", C.c_int),
    ]


class TrackOut(C.Structure):
    _fields_ = [
        ("cap", C.c_int), ("n_tracks", C.c_int), ("n_vis", C.c_int),
        ("targets", C.POINTER(C.c_float)), ("vandyaw", C.POINTER(C.c_double)), ("track_manage", C.POINTER(C.c_int32)),
        ("is_static", C.POINTER(C.c_uint8)), ("is_vis", C.POINTER(C.c_uint8)), ("vis_bb", C.POINTER(C.c_float)),
    ]


MAX_BATCH = 8


class BatchOut(C.Structure):
    _fields_ = [
        ("n_frames", C.c_int),
        ("n_elevated", C.c_int * MAX_BATCH), ("n_ground", C.c_int * MAX_BATCH), ("num_cluster", C.c_int * MAX_BATCH), ("n_boxes", C.c_int * MAX_BATCH),
        ("n_boxes_total", C.c_int), ("boxes", C.POINTER(C.c_float)), ("max_boxes", C.c_int), ("tracks", TrackOut),
    ]


class Sensor(C.Structure):
    """lmot_sensor: where one sensor of a rig is mounted (pose = sensor -> vehicle frame, row-major 3x4 [R | t])."""
    _fields_ = [("pose", C.c_float * 12), ("h_sensor", C.c_float), ("t_hmin", C.c_float), ("t_hmax", C.c_float), ("sensor_height", C.c_float)]


class TrackerParams(C.Structure):
    """lmot_tracker_params: the IMM-UKF-PDA noise, gating and track-management constants of one track table."""
    _fields_ = [
        ("gamma_g", C.c_double), ("p_g", C.c_double), ("p_d", C.c_double), ("distance_thres", C.c_double), ("lifetime_thres", C.c_int),
        ("bb_yaw_change_thres", C.c_double), ("second_init_v", C.c_double), ("static_lifetime", C.c_int), ("static_dist", C.c_double),
        ("std_a", C.c_double * 3), ("std_yawdd", C.c_double * 3), ("std_las_x", C.c_double), ("std_las_y", C.c_double),
        ("trans", (C.c_double * 3) * 3), ("mode_prob0", C.c_double * 3), ("p0_diag", C.c_double * 5),
    ]


def _tracker_params_dict(p: TrackerParams) -> dict:
    out = {}
    for name, _ in TrackerParams._fields_:
        v = getattr(p, name)
        if name == "trans":
            out[name] = [list(row) for row in v]
        elif isinstance(v, C.Array):
            out[name] = list(v)
        else:
            out[name] = v
    return out


def default_tracker_params() -> dict:
    """lmot_default_tracker_params as a dict of field -> value (lists for the array fields)"""
    p = TrackerParams()
    load_library().lmot_default_tracker_params(C.byref(p))
    return _tracker_params_dict(p)


def _tracker_params(fields: dict) -> TrackerParams:
    """the defaults with `fields` replaced (unknown names raise)"""
    p = TrackerParams()
    load_library().lmot_default_tracker_params(C.byref(p))
    names = dict(TrackerParams._fields_)
    for name, val in fields.items():
        if name not in names:
            raise ValueError(f"unknown tracker parameter {name!r}")
        if name == "trans":
            a = np.asarray(val, np.float64).reshape(3, 3)
            for i in range(3):
                p.trans[i][:] = [float(x) for x in a[i]]
        elif name in ("std_a", "std_yawdd", "mode_prob0", "p0_diag"):
            getattr(p, name)[:] = [float(x) for x in np.asarray(val, np.float64).reshape(-1)]
        elif names[name] is C.c_int:
            setattr(p, name, int(val))
        else:
            setattr(p, name, float(val))
    return p


class DetectParams(C.Structure):
    """lmot_detect_params: ground removal, clustering ROI and box-fitting values of one sequence."""
    _fields_ = [
        ("r_min", C.c_float), ("r_max", C.c_float), ("t_hmin", C.c_float), ("t_hmax", C.c_float),
        ("t_hdiff", C.c_float), ("h_sensor", C.c_float), ("ground_tolerance", C.c_double),
        ("node_prefilter", C.c_int), ("filter_z_min", C.c_float), ("filter_z_max", C.c_float),
        ("filter_x_min", C.c_float), ("filter_x_max", C.c_float), ("filter_y_min", C.c_float), ("filter_y_max", C.c_float),
        ("roi_m", C.c_float),
        ("ram_points", C.c_int), ("l_slope_dist", C.c_int), ("l_num_points", C.c_int), ("sensor_height", C.c_float),
        ("t_height_min", C.c_float), ("t_height_max", C.c_float), ("t_width_min", C.c_float), ("t_width_max", C.c_float),
        ("t_len_min", C.c_float), ("t_len_max", C.c_float), ("t_area_max", C.c_float),
        ("t_ratio_min", C.c_float), ("t_ratio_max", C.c_float), ("min_len_ratio", C.c_float), ("t_pt_per_m3", C.c_float),
        ("min_cluster_points", C.c_int), ("rule_filter", C.c_int),
    ]


MAX_RAM_POINTS = 1024


def default_detect_params(params: Params | None = None) -> dict:
    """lmot_default_detect_params: `params`' detection fields (None: the defaults) as a dict of field -> value"""
    d = DetectParams()
    load_library().lmot_default_detect_params(C.byref(params) if params is not None else None, C.byref(d))
    return {name: getattr(d, name) for name, _ in DetectParams._fields_}


def _detect_params(base: dict, fields: dict) -> DetectParams:
    """`base` (a default_detect_params dict) with `fields` replaced (unknown names raise)"""
    d = DetectParams()
    names = dict(DetectParams._fields_)
    for name, val in {**base, **fields}.items():
        if name not in names:
            raise ValueError(f"unknown detection parameter {name!r}")
        setattr(d, name, int(val) if names[name] is C.c_int else float(val))
    return d


class Deskew(C.Structure):
    """lmot_deskew: sweep deskew of a stream's frames (include/lmot.h)."""
    _fields_ = [("on", C.c_int), ("time_field", C.c_int), ("time_scale", C.c_double), ("time_offset", C.c_double),
                ("t_min", C.c_double), ("t_max", C.c_double)]


DESKEW_SLICES = 256                     # LMOT_DESKEW_SLICES


def default_deskew() -> dict:
    """lmot_default_deskew as a dict of field -> value"""
    d = Deskew()
    load_library().lmot_default_deskew(C.byref(d))
    return {name: getattr(d, name) for name, _ in Deskew._fields_}


def _deskew(fields: dict) -> Deskew:
    """the defaults with `fields` replaced (unknown names raise)"""
    d = Deskew()
    load_library().lmot_default_deskew(C.byref(d))
    names = dict(Deskew._fields_)
    for name, val in fields.items():
        if name not in names:
            raise ValueError(f"unknown deskew setting {name!r}")
        setattr(d, name, int(val) if names[name] is C.c_int else float(val))
    return d


def deskew_table(v: float, omega: float, mount=None, **fields) -> np.ndarray:
    """lmot_deskew_table: the (DESKEW_SLICES, 3, 4) float32 pose table of one frame moving at v (m/s) and turning at omega (rad/s),
    for the settings `fields` (the defaults replaced) and a sensor mounted at `mount` ((3, 4) or (12,) [R | t]; None: identity)."""
    lib = load_library()
    out = np.zeros((DESKEW_SLICES, 12), np.float32)
    m = None
    if mount is not None:
        m = Sensor()
        lib.lmot_default_sensor(None, C.byref(m))
        m.pose[:] = [float(x) for x in np.asarray(mount, np.float32).reshape(12)]
    fn = lib.lmot_deskew_table
    fn.argtypes = [C.POINTER(Deskew), C.c_double, C.c_double, C.c_void_p, C.c_void_p]
    st = fn(C.byref(_deskew(fields)), float(v), float(omega), C.cast(C.byref(m), C.c_void_p) if m is not None else None,
            out.ctypes.data_as(C.c_void_p))
    if st != OK:
        raise LmotError(st, lib.lmot_strerror(st).decode())
    return out.reshape(DESKEW_SLICES, 3, 4)


class Area(C.Structure):
    """lmot_area: a detection area, polygon rings of (x, y) vertices in the vehicle frame (include/lmot.h)."""
    _fields_ = [("n_rings", C.c_int), ("ring_len", C.c_void_p), ("xy", C.c_void_p), ("keep_outside", C.c_int)]


AREA_MAX_RINGS, AREA_MAX_VERTICES = 64, 1024     # LMOT_AREA_MAX_RINGS / LMOT_AREA_MAX_VERTICES


def _area(rings, keep_outside=False):
    """(Area or None, keep-alive arrays) of `rings`: a sequence of (m, 2) vertex arrays (None or empty: no area).  Ring lengths and
    vertices are passed as given; the library validates them."""
    if rings is None or len(rings) == 0:
        return None, ()
    arrs = [np.asarray(r, np.float64).reshape(-1, 2) for r in rings]
    lens = np.array([len(a) for a in arrs], np.int32)
    xy = np.ascontiguousarray(np.concatenate(arrs) if len(arrs) else np.zeros((0, 2)), np.float64)
    a = Area(len(arrs), lens.ctypes.data, xy.ctypes.data, int(keep_outside))
    return a, (lens, xy)


def detect_area_mask(rings, keep_outside=False, mount=None, roi_m=50.0) -> np.ndarray:
    """lmot_detect_area_mask: the (250, 8) uint32 cell mask of the area `rings` for a unit mounted at `mount` ((3, 4) or (12,) [R | t];
    None: identity) with clustering extent roi_m.  Row x = the grid's x cell, bit y & 31 of word y >> 5 = cell (x, y)."""
    lib = load_library()
    a, keep = _area(rings, keep_outside)
    m = None
    if mount is not None:
        m = Sensor()
        lib.lmot_default_sensor(None, C.byref(m))
        m.pose[:] = [float(x) for x in np.asarray(mount, np.float32).reshape(12)]
    out = np.zeros((250, 8), np.uint32)
    fn = lib.lmot_detect_area_mask
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    st = fn(C.cast(C.byref(a), C.c_void_p) if a is not None else None, C.cast(C.byref(m), C.c_void_p) if m is not None else None,
            float(roi_m), out.ctypes.data_as(C.c_void_p))
    if st != OK:
        raise LmotError(st, lib.lmot_strerror(st).decode())
    return out


class Accumulate(C.Structure):
    """lmot_accumulate: sweep accumulation of the context's frames (include/lmot.h)."""
    _fields_ = [("sweeps", C.c_int), ("max_age_s", C.c_double)]


MAX_SWEEPS = 8                          # LMOT_MAX_SWEEPS


class AccumInfo(C.Structure):
    """lmot_accum_info: what the most recently returned frame result accumulated, per unit."""
    _fields_ = [("n_units", C.c_int), ("sweeps_used", C.c_int * 8), ("n_points", C.c_int * 8),
                ("stamp_us", (C.c_double * (MAX_SWEEPS - 1)) * 8), ("pose", ((C.c_float * 12) * (MAX_SWEEPS - 1)) * 8)]


def default_accumulate() -> dict:
    lib = load_library()
    a = Accumulate()
    lib.lmot_default_accumulate(C.byref(a))
    return {name: getattr(a, name) for name, _ in Accumulate._fields_}


def _accumulate(fields: dict) -> Accumulate:
    base = default_accumulate()
    unknown = set(fields) - set(base)
    if unknown:
        raise KeyError(f"unknown accumulate fields {sorted(unknown)}")
    base.update(fields)
    return Accumulate(int(base["sweeps"]), float(base["max_age_s"]))


def accumulate_pose(fold_s, fold_t, mount=None) -> np.ndarray:
    """lmot_accumulate_pose: the (3, 4) float32 pose D moving a sweep recorded at fold_s = (x, y, yaw) (ego8[5..7] after that step) into
    the frame of fold_t, for a unit mounted at `mount` ((3, 4) or (12,) [R | t]; None: identity)."""
    lib = load_library()
    fs = np.ascontiguousarray(fold_s, np.float64).reshape(3)
    ft = np.ascontiguousarray(fold_t, np.float64).reshape(3)
    m = None
    if mount is not None:
        m = Sensor()
        lib.lmot_default_sensor(None, C.byref(m))
        m.pose[:] = [float(x) for x in np.asarray(mount, np.float32).reshape(12)]
    out = np.zeros(12, np.float32)
    st = lib.lmot_accumulate_pose(fs.ctypes.data, ft.ctypes.data, C.cast(C.byref(m), C.c_void_p) if m is not None else None, out.ctypes.data)
    if st != OK:
        raise LmotError(st, lib.lmot_strerror(st).decode())
    return out.reshape(3, 4)


class BoxSearch(C.Structure):
    """lmot_box_search: each cluster's rectangle by a search over yaw with the closeness criterion (include/lmot.h)."""
    _fields_ = [("on", C.c_int), ("n_angles", C.c_int)]


BOX_SEARCH_MAX_ANGLES = 360             # LMOT_BOX_SEARCH_MAX_ANGLES


def default_box_search() -> dict:
    lib = load_library()
    b = BoxSearch()
    lib.lmot_default_box_search(C.byref(b))
    return {name: getattr(b, name) for name, _ in BoxSearch._fields_}


def _box_search(fields: dict) -> BoxSearch:
    base = default_box_search()
    unknown = set(fields) - set(base)
    if unknown:
        raise KeyError(f"unknown box search fields {sorted(unknown)}")
    base.update(fields)
    return BoxSearch(int(base["on"]), int(base["n_angles"]))


def box_search_angles(n_angles: int) -> np.ndarray:
    """lmot_box_search_angles: the (n_angles, 2) float32 table (cos, sin) of theta_a = (pi / 2) * a / n_angles; no device needed."""
    lib = load_library()
    out = np.zeros((max(int(n_angles), 1), 2), np.float32)
    st = lib.lmot_box_search_angles(int(n_angles), out.ctypes.data_as(C.c_void_p))
    if st != OK:
        raise LmotError(st, lib.lmot_strerror(st).decode())
    return out


class GroundLines(C.Structure):
    """lmot_ground_lines: slope-following ground removal and box heights from the local ground (include/lmot.h)."""
    _fields_ = [("on", C.c_int), ("max_slope", C.c_double), ("max_rmse", C.c_double), ("max_step", C.c_double)]


def default_ground_lines() -> dict:
    lib = load_library()
    g = GroundLines()
    lib.lmot_default_ground_lines(C.byref(g))
    return {name: getattr(g, name) for name, _ in GroundLines._fields_}


def _ground_lines(fields: dict) -> GroundLines:
    base = default_ground_lines()
    unknown = set(fields) - set(base)
    if unknown:
        raise KeyError(f"unknown ground lines fields {sorted(unknown)}")
    base.update(fields)
    return GroundLines(int(base["on"]), float(base["max_slope"]), float(base["max_rmse"]), float(base["max_step"]))


def ground_lines_grid(minz, r_min: float, r_max: float, sensor_height: float, **fields) -> np.ndarray:
    """lmot_ground_lines_grid: the (80, 120) float32 ground heights of the lines through a (80, 120) float32 min-z grid (1000: empty
    cell); `fields` replace the default setting's values.  A frame's grid is reproduced with its float32 r_min / r_max / sensor_height
    widened to double.  No device needed."""
    lib = load_library()
    mz = np.ascontiguousarray(np.asarray(minz, np.float32).reshape(80, 120))
    out = np.zeros((80, 120), np.float32)
    g = _ground_lines(fields)
    st = lib.lmot_ground_lines_grid(C.byref(g), mz.ctypes.data_as(C.c_void_p), float(r_min), float(r_max), float(sensor_height),
                                    out.ctypes.data_as(C.c_void_p))
    if st != OK:
        raise LmotError(st, lib.lmot_strerror(st).decode())
    return out


class Layers(C.Structure):
    """lmot_layers: layered clustering, connected components over (x, y, height slice) (include/lmot.h)."""
    _fields_ = [("on", C.c_int), ("n_slices", C.c_int), ("slice_m", C.c_double), ("z_min", C.c_double), ("gap_slices", C.c_int)]


def default_layers() -> dict:
    lib = load_library()
    l = Layers()
    lib.lmot_default_layers(C.byref(l))
    return {name: getattr(l, name) for name, _ in Layers._fields_}


def _layers(fields: dict) -> Layers:
    base = default_layers()
    unknown = set(fields) - set(base)
    if unknown:
        raise KeyError(f"unknown layers fields {sorted(unknown)}")
    base.update(fields)
    return Layers(int(base["on"]), int(base["n_slices"]), float(base["slice_m"]), float(base["z_min"]), int(base["gap_slices"]))


class Obstacles(C.Structure):
    """lmot_obstacles: obstacle footprints of every cluster (include/lmot.h)."""
    _fields_ = [("on", C.c_int), ("max_vertices", C.c_int)]


OBSTACLE_MAX_HULL = 140                # LMOT_OBSTACLE_MAX_HULL
OBSTACLE_DTYPE = np.dtype([("cluster", np.int32), ("n_points", np.int32), ("n_cells", np.int32), ("box", np.int32),
                           ("vertex_offset", np.int32), ("vertex_count", np.int32), ("z_min", np.float32), ("z_max", np.float32)])


class ObstaclesOut(C.Structure):
    _fields_ = [("obstacles", C.c_void_p), ("cap_obstacles", C.c_int), ("vertices", C.c_void_p), ("cap_vertices", C.c_int),
                ("n_units", C.c_int), ("n_obstacles", C.c_int), ("n_vertices", C.c_int)]


def default_obstacles() -> dict:
    lib = load_library()
    o = Obstacles()
    lib.lmot_default_obstacles(C.byref(o))
    return {name: getattr(o, name) for name, _ in Obstacles._fields_}


def _obstacles(fields: dict) -> Obstacles:
    base = default_obstacles()
    unknown = set(fields) - set(base)
    if unknown:
        raise KeyError(f"unknown obstacles fields {sorted(unknown)}")
    base.update(fields)
    return Obstacles(int(base["on"]), int(base["max_vertices"]))


def obstacle_polygons(res: dict) -> list:
    """The footprint of every obstacle of an obstacles_result as a float32 [count, 2] array (empty where the pool overflowed)."""
    v = res["vertices"]
    return [v[o: o + c] for o, c in zip(res["obstacles"]["vertex_offset"], res["obstacles"]["vertex_count"])]


class EgoMatch(C.Structure):
    """lmot_ego_match: scan-matched ego motion settings (include/lmot.h)."""
    _fields_ = [("grid", C.c_int), ("cell_m", C.c_double), ("z_min", C.c_double), ("z_max", C.c_double), ("r_min", C.c_double),
                ("r_max", C.c_double), ("sub_m", C.c_double), ("max_points", C.c_int), ("yaw_step", C.c_double), ("yaw_half", C.c_int),
                ("shift_half", C.c_int), ("refine", C.c_int), ("min_points", C.c_int), ("min_score_frac", C.c_double), ("sensor", C.c_int)]


class EgoOut(C.Structure):
    _fields_ = [("ok", C.c_int), ("n_used", C.c_int), ("n_ref", C.c_int), ("score", C.c_int), ("score_max", C.c_int),
                ("dx", C.c_double), ("dy", C.c_double), ("dtheta", C.c_double), ("v", C.c_double), ("yaw", C.c_double)]


def default_ego_match() -> dict:
    lib = load_library()
    m = EgoMatch()
    lib.lmot_default_ego_match(C.byref(m))
    return {name: getattr(m, name) for name, _ in EgoMatch._fields_}


def _ego_match(fields: dict) -> EgoMatch:
    base = default_ego_match()
    unknown = set(fields) - set(base)
    if unknown:
        raise KeyError(f"unknown ego match fields {sorted(unknown)}")
    base.update(fields)
    return EgoMatch(*[t(base[name]) for name, t in ((n, int if c is C.c_int else float) for n, c in EgoMatch._fields_)])


def _ego_dict(o: EgoOut) -> dict:
    return {name: getattr(o, name) for name, _ in EgoOut._fields_}


class FrameOut(C.Structure):
    _fields_ = [
        ("n_elevated", C.c_int), ("n_ground", C.c_int), ("num_cluster", C.c_int), ("n_boxes", C.c_int),
        ("boxes", C.POINTER(C.c_float)), ("max_boxes", C.c_int), ("tracks", TrackOut),
    ]


MAX_PRED_TIMES = 32                    # LMOT_MAX_PRED_TIMES
PRED_VALID, PRED_DEAD, PRED_GUARD_P, PRED_GUARD_S = 1, 2, 4, 8
PRED_FIELDS = (("x", 5), ("P", 25), ("mode_prob", 3), ("gate_z", 2), ("gate_S", 4))   # per (time, row), float64


class PredOut(C.Structure):
    _fields_ = [("cap", C.c_int), ("n_rows", C.c_int), ("ids", C.c_void_p), ("track_manage", C.c_void_p), ("flags", C.c_void_p),
                ("x", C.c_void_p), ("P", C.c_void_p), ("mode_prob", C.c_void_p), ("gate_z", C.c_void_p), ("gate_S", C.c_void_p)]


def pred_out(cap: int, ptrs: dict) -> PredOut:
    """lmot_pred_out of `cap` rows over the given array addresses (keys ids, track_manage, flags, x, P, mode_prob, optional gate_z /
    gate_S; device addresses for the _dev forms).  Layout: ids / track_manage [cap], flags [n_t][cap], x [n_t][cap][5], P [n_t][cap][25],
    mode_prob [n_t][cap][3], gate_z [n_t][cap][2], gate_S [n_t][cap][4]."""
    o = PredOut()
    o.cap = int(cap)
    for name, _ in PredOut._fields_[2:]:
        setattr(o, name, int(ptrs[name]) if ptrs.get(name) else None)
    return o


class SeqOut(C.Structure):
    _fields_ = [("n_seq", C.c_int), ("seq", FrameOut * MAX_BATCH)]


SEQ_SKIP, SEQ_FRAMES, SEQ_LISTS = 0, 1, 2          # lmot_seq_entry.kind
SEQ_RESTART = 1                                     # lmot_seq_entry.flags


class SeqEntry(C.Structure):
    _fields_ = [("kind", C.c_int), ("flags", C.c_int), ("timestamp_us", C.c_double), ("v_gps", C.c_double), ("yaw_gps", C.c_double),
                ("data", C.POINTER(C.c_void_p)), ("n", C.POINTER(C.c_int)), ("d_counts", C.c_void_p), ("cap_per_list", C.c_int)]


# every symbol include/lmot.h declares (tests assert the library exports all of them)
ABI_SYMBOLS = [
    "lmot_default_params", "lmot_create", "lmot_destroy", "lmot_get_params", "lmot_strerror", "lmot_last_error", "lmot_build_info",
    "lmot_set_stream", "lmot_pinned_alloc", "lmot_pinned_free", "lmot_ground_remove", "lmot_component_cluster", "lmot_cluster_outputs", "lmot_box_fit", "lmot_track_step", "lmot_frame",
    "lmot_frame_dev", "lmot_frame_fetch", "lmot_frame_submit", "lmot_frame_collect", "lmot_frames_in_flight", "lmot_frame_ready", "lmot_flush",
    "lmot_ground_remove_dev", "lmot_detect_dev", "lmot_sync",
    "lmot_batch_submit", "lmot_batch_dev", "lmot_batch_detect_dev", "lmot_batch_collect", "lmot_batch_fetch", "lmot_batch", "lmot_batch_ground_ccl_dev",
    "lmot_default_sensor", "lmot_set_sensors", "lmot_get_sensors",
    "lmot_set_rig_merge", "lmot_get_rig_merge", "lmot_seq_set_rig_merge", "lmot_seq_get_rig_merge",
    "lmot_seq_open", "lmot_seq_submit", "lmot_seq_dev", "lmot_seq_collect", "lmot_seq_fetch", "lmot_seq", "lmot_seq_tracker_reset",
    "lmot_seq_tracker_dump", "lmot_seq_tracker_get_ego", "lmot_seq_set_sensors", "lmot_seq_get_sensors", "lmot_seq_frame_counts",
    "lmot_seq_track_submit", "lmot_seq_track_dev", "lmot_seq_track", "lmot_seq_tracker_load", "lmot_seq_tracker_set_ego",
    "lmot_seq_tick_submit", "lmot_seq_tick_dev", "lmot_seq_tick", "lmot_seq_stepped",
    "lmot_default_deskew", "lmot_set_deskew", "lmot_get_deskew", "lmot_seq_set_deskew", "lmot_seq_get_deskew", "lmot_deskew_table",
    "lmot_set_detect_area", "lmot_get_detect_area", "lmot_seq_set_detect_area", "lmot_seq_get_detect_area", "lmot_detect_area_mask",
    "lmot_debug_area_masks",
    "lmot_default_accumulate", "lmot_set_accumulate", "lmot_get_accumulate", "lmot_accumulate_info", "lmot_accumulate_pose",
    "lmot_seq_set_accumulate", "lmot_seq_get_accumulate", "lmot_seq_accumulate_info",
    "lmot_default_box_search", "lmot_set_box_search", "lmot_get_box_search", "lmot_seq_set_box_search", "lmot_seq_get_box_search",
    "lmot_box_search_angles",
    "lmot_default_ground_lines", "lmot_set_ground_lines", "lmot_get_ground_lines", "lmot_seq_set_ground_lines", "lmot_seq_get_ground_lines",
    "lmot_ground_lines_grid", "lmot_debug_ground_lines",
    "lmot_default_layers", "lmot_set_layers", "lmot_get_layers", "lmot_seq_set_layers", "lmot_seq_get_layers", "lmot_debug_point_clusters",
    "lmot_default_obstacles", "lmot_set_obstacles", "lmot_get_obstacles", "lmot_seq_set_obstacles", "lmot_seq_get_obstacles",
    "lmot_obstacles_result", "lmot_seq_obstacles_result",
    "lmot_default_ego_match", "lmot_set_ego_match", "lmot_get_ego_match", "lmot_seq_set_ego_match", "lmot_seq_get_ego_match",
    "lmot_ego_reset", "lmot_seq_ego_reset", "lmot_ego_estimate", "lmot_ego_estimate_dev", "lmot_seq_ego_estimate", "lmot_seq_ego_estimate_dev",
    "lmot_default_tracker_params", "lmot_set_tracker_params", "lmot_get_tracker_params", "lmot_seq_set_tracker_params",
    "lmot_seq_get_tracker_params", "lmot_default_detect_params", "lmot_seq_set_detect_params", "lmot_seq_get_detect_params",
    "lmot_set_track_retirement", "lmot_get_track_retirement", "lmot_seq_set_track_retirement", "lmot_seq_get_track_retirement",
    "lmot_track_ids", "lmot_seq_track_ids",
    "lmot_predict_tracks", "lmot_predict_tracks_dev", "lmot_seq_predict_tracks", "lmot_seq_predict_tracks_dev",
    "lmot_detect_boxes_dev", "lmot_track_step_lists_dev", "lmot_tracker_counters_dev", "lmot_tracker_table_received",
    "lmot_origin_points", "lmot_tracker_table", "lmot_tracker_set_num_tracks", "lmot_tracker_reset", "lmot_tracker_num_tracks", "lmot_tracker_dump", "lmot_tracker_load", "lmot_tracker_get_ego", "lmot_tracker_set_ego",
    "lmot_debug_polar_grid", "lmot_debug_cell_index", "lmot_debug_label_grid", "lmot_selftest_atan2f",
    "lmot_enable_timing", "lmot_last_stage_ms", "lmot_last_kernel_ms", "lmot_debug_host_ns",
]

_lib = None


def load_library() -> C.CDLL:
    """Load liblmot.so (raises OSError when it has not been built: there is nothing to fall back to)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OSError(f"{LIB_PATH} not built -- run `python -c 'import __graft_entry__ as g; g.build()'`")
        lib = C.CDLL(LIB_PATH)
        lib.lmot_strerror.restype = C.c_char_p
        lib.lmot_last_error.restype = C.c_char_p
        lib.lmot_build_info.restype = C.c_char_p
        lib.lmot_last_error.argtypes = [C.c_void_p]
        lib.lmot_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(Params), C.c_int]
        lib.lmot_destroy.argtypes = [C.c_void_p]
        lib.lmot_accumulate_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.lmot_box_search_angles.argtypes = [C.c_int, C.c_void_p]
        lib.lmot_ground_lines_grid.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_void_p]
        lib.lmot_ego_estimate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p]
        lib.lmot_ego_estimate_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p]
        lib.lmot_seq_ego_estimate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        lib.lmot_seq_ego_estimate_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def default_params() -> Params:
    p = Params()
    load_library().lmot_default_params(C.byref(p))
    return p


_EMPTY = np.zeros(4, np.float32)        # the data pointer of an empty host frame (never read)


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _pts(points):
    p = np.ascontiguousarray(points, dtype=np.float32)
    if p.ndim != 2 or p.shape[1] < 3:
        raise ValueError("points must be (N, >=3) float32")
    return p, int(p.shape[0]), int(p.shape[1])


class Lmot:
    """One context = one sensor stream on one GPU (not thread-safe, like the reference's globals)."""

    def __init__(self, params: Params | None = None, device: int = 0):
        self.lib = load_library()
        self.params = params if params is not None else default_params()
        h = C.c_void_p()
        st = self.lib.lmot_create(C.byref(h), C.byref(self.params), device)
        if st != OK:
            raise LmotError(st, self.lib.lmot_strerror(st).decode())
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.lmot_destroy(self.h)
            self.h = None
            self.lib.lmot_pinned_free.argtypes = [C.c_void_p]
            for ptr in getattr(self, "_pinned", []):
                self.lib.lmot_pinned_free(ptr)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, st: int):
        if st < 0:
            raise LmotError(st, self.lib.lmot_strerror(st).decode() + " | " + self.lib.lmot_last_error(self.h).decode())
        self.last_warning = st          # > 0: LMOT_WARN_* (the call's outputs are valid)

    def set_stream(self, cuda_stream_handle: int | None):
        self._chk(self.lib.lmot_set_stream(self.h, C.c_void_p(cuda_stream_handle or 0)))

    def sync(self):
        self._chk(self.lib.lmot_sync(self.h))

    # ---- groundRemove ------------------------------------------------------------------------------------
    def ground_remove(self, points):
        """-> dict(labels (N,) u8, elevated (Ne,4) f32, ground (Ng,4) f32); clouds keep input order."""
        p, n, s = _pts(points)
        labels = np.zeros(max(n, 1), np.uint8)
        elev = np.zeros((max(n, 1), 4), np.float32)
        grnd = np.zeros((max(n, 1), 4), np.float32)
        ne, ng = C.c_int(0), C.c_int(0)
        self._chk(self.lib.lmot_ground_remove(self.h, _fp(p), n, s, labels.ctypes.data_as(C.POINTER(C.c_uint8)), _fp(elev),
                                              C.byref(ne), _fp(grnd), C.byref(ng)))
        return dict(labels=labels[:n], elevated=elev[: ne.value], ground=grnd[: ng.value])

    def ground_remove_dev(self, d_ptr: int, n: int):
        self._chk(self.lib.lmot_ground_remove_dev(self.h, C.c_void_p(d_ptr), n))

    def cluster_outputs(self, cap: int | None = None):
        """Side outputs of the cluster node for the last clustering: (clustered (n,4), obstacles (m,4) [x,y,z,cluster], cost_map (50,50))"""
        cap = cap or int(self.params.max_points)
        cl = np.zeros((cap, 4), np.float32); ob = np.zeros((62500, 4), np.float32); cm = np.zeros(2500, np.int32)
        ncl = C.c_int(0); nob = C.c_int(0)
        self._chk(self.lib.lmot_cluster_outputs(self.h, _fp(cl), cap, C.byref(ncl), _fp(ob), 62500, C.byref(nob),
                                                cm.ctypes.data_as(C.POINTER(C.c_int32))))
        return cl[: ncl.value].copy(), ob[: nob.value].copy(), cm.reshape(50, 50)

    # ---- componentClustering ------------------------------------------------------------------------------
    def component_cluster(self, elevated):
        """-> (grid (250,250) int32 x-major, num_cluster)"""
        if len(elevated) == 0:
            p, n, s = np.zeros((1, 4), np.float32), 0, 4
        else:
            p, n, s = _pts(elevated)
        grid = np.zeros(250 * 250, np.int32)
        nc = C.c_int(0)
        self._chk(self.lib.lmot_component_cluster(self.h, _fp(p), n, s, grid.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nc)))
        return grid.reshape(250, 250), nc.value

    # ---- boxFitting ---------------------------------------------------------------------------------------
    def box_fit(self, elevated, grid, num_cluster, max_boxes: int = 1024):
        """-> (boxes (B,8,3) f32, markers (B,6) f32) in cluster-id order"""
        if len(elevated) == 0:
            p, n, s = np.zeros((1, 4), np.float32), 0, 4
        else:
            p, n, s = _pts(elevated)
        g = np.ascontiguousarray(grid, np.int32).reshape(-1)
        boxes = np.zeros((max_boxes, 8, 3), np.float32)
        markers = np.zeros((max_boxes, 6), np.float32)
        nb = C.c_int(0)
        self._chk(self.lib.lmot_box_fit(self.h, _fp(p), n, s, g.ctypes.data_as(C.POINTER(C.c_int32)), int(num_cluster), _fp(boxes),
                                        max_boxes, C.byref(nb), _fp(markers)))
        return boxes[: nb.value].copy(), markers[: nb.value].copy()

    # ---- getOriginPoints + immUkfJpdaf -------------------------------------------------------------------
    def _new_track_bufs(self, cap):
        bufs = dict(targets=np.zeros((cap, 3), np.float32), vandyaw=np.zeros((cap, 2), np.float64),
                    track_manage=np.zeros(cap, np.int32), is_static=np.zeros(cap, np.uint8), is_vis=np.zeros(cap, np.uint8),
                    vis_bb=np.zeros((cap, 8, 3), np.float32), boxes=np.zeros((self.params.max_boxes, 8, 3), np.float32))
        to = TrackOut()
        to.cap = cap
        to.targets = _fp(bufs["targets"]); to.vandyaw = bufs["vandyaw"].ctypes.data_as(C.POINTER(C.c_double))
        to.track_manage = bufs["track_manage"].ctypes.data_as(C.POINTER(C.c_int32))
        to.is_static = bufs["is_static"].ctypes.data_as(C.POINTER(C.c_uint8))
        to.is_vis = bufs["is_vis"].ctypes.data_as(C.POINTER(C.c_uint8)); to.vis_bb = _fp(bufs["vis_bb"])
        return to, bufs

    def _track_out(self, cap):
        """Output buffers are allocated once per (context, cap) and reused: the hot loop must not allocate megabytes."""
        cache = self.__dict__.setdefault("_out_cache", {})
        if cap not in cache:
            to, bufs = self._new_track_bufs(cap)
            fo = FrameOut()
            fo.boxes = _fp(bufs["boxes"]); fo.max_boxes = self.params.max_boxes
            fo_nb = FrameOut()
            fo_nb.max_boxes = self.params.max_boxes
            cache[cap] = (to, bufs, fo, fo_nb)
        to, bufs, _, _ = cache[cap]
        return to, bufs

    def _frame_out(self, cap, want_boxes=True):
        to, bufs = self._track_out(cap)
        _, _, fo, fo_nb = self._out_cache[cap]
        f = fo if want_boxes else fo_nb
        f.tracks = to
        return f, bufs

    @staticmethod
    def _track_result(to, bufs):
        t, v = to.n_tracks, to.n_vis
        return dict(targets=bufs["targets"][:t].copy(), vandyaw=bufs["vandyaw"][:t].copy(),
                    track_manage=bufs["track_manage"][:t].copy(), is_static=bufs["is_static"][:t].copy(),
                    is_vis=bufs["is_vis"][:t].copy(), vis_bb=bufs["vis_bb"][:v].copy())

    @staticmethod
    def _frame_result(fo, bufs, want_boxes=True):
        r = Lmot._track_result(fo.tracks, bufs)
        r.update(n_elevated=fo.n_elevated, n_ground=fo.n_ground, num_cluster=fo.num_cluster,
                 boxes=bufs["boxes"][: fo.n_boxes].copy() if want_boxes else bufs["boxes"][:0])
        return r

    def track_step(self, boxes, timestamp_us, v_gps=0.0, yaw_gps=0.0, cap: int | None = None):
        b = np.ascontiguousarray(boxes, np.float32).reshape(-1, 8, 3)
        m = b.shape[0]
        if m == 0:
            b = np.zeros((1, 8, 3), np.float32)
        cap = cap or self.params.max_tracks
        to, bufs = self._track_out(cap)
        self._chk(self.lib.lmot_track_step(self.h, _fp(b), m, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps), C.byref(to)))
        return self._track_result(to, bufs)

    def frame(self, points, timestamp_us, v_gps=0.0, yaw_gps=0.0, cap: int | None = None):
        """The whole hot path on one host frame -> dict(n_elevated, n_ground, num_cluster, boxes, tracks...)."""
        p, n, s = _pts(points)
        fo, bufs = self._frame_out(cap or self.params.max_tracks)
        self._chk(self.lib.lmot_frame(self.h, _fp(p), n, s, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps), C.byref(fo)))
        return self._frame_result(fo, bufs)

    def frame_dev(self, d_ptr: int, n: int, timestamp_us, v_gps=0.0, yaw_gps=0.0):
        """Asynchronous: device-resident XYZI frame (stride 4) through all four stages on the context's stream."""
        self._chk(self.lib.lmot_frame_dev(self.h, C.c_void_p(d_ptr), n, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps)))

    def flush(self):
        """Device-side join: the caller stream waits for everything submitted so far."""
        self._chk(self.lib.lmot_flush(self.h))

    def pinned_array(self, shape, dtype=np.float32) -> np.ndarray:
        """numpy array in page-locked host memory (lmot_pinned_alloc); freed when the context closes."""
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.lib.lmot_pinned_alloc.restype = C.c_void_p
        self.lib.lmot_pinned_alloc.argtypes = [C.c_size_t]
        ptr = self.lib.lmot_pinned_alloc(nbytes)
        if not ptr:
            raise LmotError(-1, "lmot_pinned_alloc failed")
        self._pinned = getattr(self, "_pinned", [])
        self._pinned.append(ptr)
        buf = (C.c_char * nbytes).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def frame_submit(self, points, timestamp_us, v_gps=0.0, yaw_gps=0.0):
        """Asynchronous host frame (pinned memory recommended); collect results later with frame_collect()."""
        p, n, s = _pts(points)
        self._chk(self.lib.lmot_frame_submit(self.h, _fp(p), n, s, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps)))

    def frame_collect(self, cap: int | None = None, want_boxes: bool = True):
        """Results of the oldest submitted frame (blocks until it is done)."""
        fo, bufs = self._frame_out(cap or self.params.max_tracks, want_boxes)
        self._chk(self.lib.lmot_frame_collect(self.h, C.byref(fo)))
        return self._frame_result(fo, bufs, want_boxes)

    def frame_ready(self) -> bool:
        return self.lib.lmot_frame_ready(self.h) == 1

    def frames_in_flight(self) -> int:
        n = C.c_int(0)
        self._chk(self.lib.lmot_frames_in_flight(self.h, C.byref(n)))
        return n.value

    def detect_dev(self, d_ptr: int, n: int):
        self._chk(self.lib.lmot_detect_dev(self.h, C.c_void_p(d_ptr), n))

    def frame_fetch(self, cap: int | None = None, want_boxes: bool = True):
        fo, bufs = self._frame_out(cap or self.params.max_tracks, want_boxes)
        self._chk(self.lib.lmot_frame_fetch(self.h, C.byref(fo)))
        return self._frame_result(fo, bufs, want_boxes)

    def track_step_lists_dev(self, d_lists: int, d_counts: int, n_lists: int, cap_per_list: int, timestamp_us, v_gps=0.0, yaw_gps=0.0):
        """Asynchronous: n_lists padded device box lists (cap_per_list boxes each, lengths in the device ints at d_counts) as one
        tracker step; results with frame_fetch()."""
        self._chk(self.lib.lmot_track_step_lists_dev(self.h, C.c_void_p(d_lists), C.c_void_p(d_counts), int(n_lists), int(cap_per_list),
                                                     C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps)))

    # ---- batched ticks: F sensor streams, one frame each, one shared track table (BASELINE.json configs[3]) --------
    def batch_prepare(self, dev_frames):
        """Marshal a tick's (device pointer, n) list ONCE: the returned handle can be passed to batch_dev / batch_detect_dev /
        batch_ground_ccl_dev in place of the list (a timing loop must not build ctypes arrays on every call)."""
        return ("prepared",) + tuple(self._batch_args(dev_frames, True))

    def _batch_args(self, frames, device: bool):
        if isinstance(frames, tuple) and frames and frames[0] == "prepared":
            return frames[1:]
        F = len(frames)
        ptrs = (C.c_void_p * F)()
        ns = (C.c_int * F)()
        keep = []
        stride = 4
        for i, f in enumerate(frames):
            if device:
                ptrs[i], ns[i] = int(f[0]), int(f[1])
            else:
                p, n, stride = _pts(f)
                keep.append(p)
                ptrs[i], ns[i] = p.ctypes.data, n
        return ptrs, ns, F, stride, keep

    def _batch_result(self, bo, bufs, want_boxes=True):
        r = Lmot._track_result(bo.tracks, bufs)
        F = bo.n_frames
        r.update(n_frames=F, n_elevated=list(bo.n_elevated[:F]), n_ground=list(bo.n_ground[:F]), num_cluster=list(bo.num_cluster[:F]),
                 n_boxes=list(bo.n_boxes[:F]), boxes=bufs["boxes"][: bo.n_boxes_total].copy() if want_boxes else bufs["boxes"][:0])
        return r

    def _batch_out(self, cap, want_boxes=True):
        to, bufs = self._track_out(cap)
        bo = BatchOut()
        if want_boxes:
            bo.boxes = _fp(bufs["boxes"])
        bo.max_boxes = self.params.max_boxes
        bo.tracks = to
        return bo, bufs

    def batch(self, frames, timestamp_us, v_gps=0.0, yaw_gps=0.0, cap: int | None = None):
        """One tick, synchronous: `frames` = list of (N_i, >=3) host arrays (one per sensor stream)."""
        ptrs, ns, F, stride, keep = self._batch_args(frames, False)
        bo, bufs = self._batch_out(cap or self.params.max_tracks)
        self._chk(self.lib.lmot_batch(self.h, ptrs, ns, F, stride, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps), C.byref(bo)))
        return self._batch_result(bo, bufs)

    def batch_submit(self, frames, timestamp_us, v_gps=0.0, yaw_gps=0.0):
        ptrs, ns, F, stride, keep = self._batch_args(frames, False)
        self._keep = keep          # the copies are asynchronous: the host arrays must outlive the call
        self._chk(self.lib.lmot_batch_submit(self.h, ptrs, ns, F, stride, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps)))

    def batch_dev(self, dev_frames, timestamp_us, v_gps=0.0, yaw_gps=0.0):
        """dev_frames = list of (device pointer, n) of stride-4 float frames."""
        ptrs, ns, F, _, _ = self._batch_args(dev_frames, True)
        self._chk(self.lib.lmot_batch_dev(self.h, ptrs, ns, F, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps)))

    def batch_detect_dev(self, dev_frames):
        ptrs, ns, F, _, _ = self._batch_args(dev_frames, True)
        self._chk(self.lib.lmot_batch_detect_dev(self.h, ptrs, ns, F))

    def batch_ground_ccl_dev(self, dev_frames):
        ptrs, ns, F, _, _ = self._batch_args(dev_frames, True)
        self._chk(self.lib.lmot_batch_ground_ccl_dev(self.h, ptrs, ns, F))

    def batch_collect(self, cap: int | None = None, want_boxes: bool = True):
        bo, bufs = self._batch_out(cap or self.params.max_tracks, want_boxes)
        self._chk(self.lib.lmot_batch_collect(self.h, C.byref(bo)))
        return self._batch_result(bo, bufs, want_boxes)

    def batch_fetch(self, cap: int | None = None, want_boxes: bool = True):
        bo, bufs = self._batch_out(cap or self.params.max_tracks, want_boxes)
        self._chk(self.lib.lmot_batch_fetch(self.h, C.byref(bo)))
        return self._batch_result(bo, bufs, want_boxes)

    # ---- sensor rig: sensor k = frame k of a batched tick / list k of track_step_lists_dev (lmot_set_sensors) ----------------
    def set_sensors(self, poses, h_sensor=None, t_hmin=None, t_hmax=None, sensor_height=None):
        """poses: (n, 3, 4) or (n, 12) sensor -> vehicle transforms [R | t] (n = 0 or None: no sensors).  The four thresholds are
        per-sensor sequences (or one value for all); None keeps this context's lmot_params value."""
        arr, n = self._sensor_table(poses, h_sensor, t_hmin, t_hmax, sensor_height)
        self._chk(self.lib.lmot_set_sensors(self.h, arr, n))

    def _sensor_table(self, poses, h_sensor, t_hmin, t_hmax, sensor_height):
        """(lmot_sensor array or None, n) for set_sensors / seq_set_sensors"""
        if poses is None or len(poses) == 0:
            return None, 0
        P = np.asarray(poses, np.float32).reshape(len(poses), 12)
        n = P.shape[0]
        arr = (Sensor * n)()
        for k in range(n):
            self.lib.lmot_default_sensor(C.byref(self.params), C.byref(arr[k]))
            arr[k].pose[:] = [float(v) for v in P[k]]
            for name, val in (("h_sensor", h_sensor), ("t_hmin", t_hmin), ("t_hmax", t_hmax), ("sensor_height", sensor_height)):
                if val is not None:
                    setattr(arr[k], name, float(np.broadcast_to(np.asarray(val, np.float32), (n,))[k]))
        return arr, n

    @staticmethod
    def _sensor_dict(s):
        return dict(poses=np.array([list(e.pose) for e in s], np.float32).reshape(-1, 3, 4),
                    **{k: np.array([getattr(e, k) for e in s], np.float32) for k in ("h_sensor", "t_hmin", "t_hmax", "sensor_height")})

    def _get_sensors(self, fn, *k):
        arr = (Sensor * MAX_BATCH)()
        n = C.c_int(0)
        self._chk(fn(self.h, *k, arr, MAX_BATCH, C.byref(n)))
        return self._sensor_dict(arr[: n.value])

    def get_sensors(self):
        """-> dict(poses (n, 3, 4) f32, h_sensor, t_hmin, t_hmax, sensor_height: (n,) f32 each)"""
        return self._get_sensors(self.lib.lmot_get_sensors)

    # ---- merging rigs (lmot_set_rig_merge): the sensors' elevated clouds clustered and boxed as one vehicle-frame cloud ----------
    def set_rig_merge(self, on):
        """Batched ticks of this context's rig: with a sensor table set, ground removal per sensor, then ONE clustering and box fitting
        of the sensors' elevated clouds moved into the vehicle frame (an object seen by two sensors is one box).  lmot_params'
        sensor_height is then the vehicle frame origin's height above the ground.  Applies from the next submitted tick on."""
        self._chk(self.lib.lmot_set_rig_merge(self.h, int(on)))

    def _get_switch(self, fn, *k) -> bool:
        v = C.c_int(0)
        self._chk(fn(self.h, *k, C.byref(v)))
        return bool(v.value)

    def get_rig_merge(self) -> bool:
        return self._get_switch(self.lib.lmot_get_rig_merge)

    def seq_set_rig_merge(self, k: int, on):
        """Sequence k's FRAMES steps, as set_rig_merge (with sequence k's sensor table and detection values)."""
        self._chk(self.lib.lmot_seq_set_rig_merge(self.h, int(k), int(on)))

    def seq_get_rig_merge(self, k: int) -> bool:
        return self._get_switch(self.lib.lmot_seq_get_rig_merge, int(k))

    # ---- independent sequences: one frame of each sequence per tick, one track table per sequence (lmot_seq_*) ---------------
    def seq_open(self, n_seq: int, ring: int = 8):
        """n_seq (1..8) empty sequences and a ring of `ring` ticks (n_seq = 0 frees the set); drains the context."""
        self._chk(self.lib.lmot_seq_open(self.h, int(n_seq), int(ring)))
        self.n_seq = int(n_seq)

    def seq_prepare(self, dev_frames):
        """Marshal a tick's per-sequence (device pointer, n) entries ONCE for seq_dev (a timing loop must not build ctypes arrays on
        every call).  Entries as seq_dev takes them."""
        return ("seq_prepared",) + tuple(self._seq_args(dev_frames, True))

    @staticmethod
    def _frame_list(entry, device: bool) -> bool:
        """True if a sequence's entry is a Python list of frames (a sequence with a sensor table) rather than one frame"""
        if not isinstance(entry, list) or not entry:
            return False
        return all(isinstance(x, tuple) for x in entry) if device else all(np.ndim(x) == 2 for x in entry)

    def _seq_args(self, frames, device: bool):
        """per-sequence entries -> (ptrs, ns, n_seq, stride, keep) over the tick's frames in sequence order"""
        if isinstance(frames, tuple) and frames and frames[0] == "seq_prepared":
            return frames[1:]
        if isinstance(frames, tuple) and frames and frames[0] == "prepared":      # a batch_prepare handle: one frame per sequence
            return frames[1:]
        flat = []
        for e in frames:
            flat.extend(e if self._frame_list(e, device) else [e])
        ptrs, ns, _, stride, keep = self._batch_args(flat, device)
        return ptrs, ns, len(frames), stride, keep

    # ---- sensor tables of sequences (lmot_seq_set_sensors): sequence k sends one frame per sensor each tick ------------------
    def seq_set_sensors(self, k: int, poses, h_sensor=None, t_hmin=None, t_hmax=None, sensor_height=None):
        """Sequence k's sensor table, arguments as set_sensors (poses None or empty: no table, one frame per tick)."""
        arr, n = self._sensor_table(poses, h_sensor, t_hmin, t_hmax, sensor_height)
        self._chk(self.lib.lmot_seq_set_sensors(self.h, int(k), arr, n))

    def seq_get_sensors(self, k: int):
        """-> dict as get_sensors, for sequence k"""
        return self._get_sensors(self.lib.lmot_seq_get_sensors, int(k))

    # ---- tracker parameters (lmot_set_tracker_params / lmot_seq_set_tracker_params) --------------------------------------------
    def set_tracker_params(self, **fields):
        """The context's own track table: the given fields, every other one at its default (no fields: the defaults).
        Array fields take sequences (std_a (3,), trans (3, 3), ...).  Applies from the next submitted step on."""
        self._chk(self.lib.lmot_set_tracker_params(self.h, C.byref(_tracker_params(fields)) if fields else None))

    def _get_record(self, fn, cls, *k, as_dict=None) -> dict:
        """a stream's setting record (cls) read by fn, as a dict of field -> value (as_dict: the conversion, default getattr per field)"""
        r = cls()
        self._chk(fn(self.h, *k, C.byref(r)))
        return as_dict(r) if as_dict else {name: getattr(r, name) for name, _ in cls._fields_}

    def get_tracker_params(self) -> dict:
        return self._get_record(self.lib.lmot_get_tracker_params, TrackerParams, as_dict=_tracker_params_dict)

    def seq_set_tracker_params(self, k: int, **fields):
        """Sequence k's parameters, arguments as set_tracker_params."""
        self._chk(self.lib.lmot_seq_set_tracker_params(self.h, int(k), C.byref(_tracker_params(fields)) if fields else None))

    def seq_get_tracker_params(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_tracker_params, TrackerParams, int(k), as_dict=_tracker_params_dict)

    # ---- track retirement and track IDs (lmot_set_track_retirement / lmot_track_ids) -------------------------------------------
    def set_track_retirement(self, on: bool):
        """The context's own table: end every step by removing the tracks with trackManage 0.  Applies from the next submitted step on."""
        self._chk(self.lib.lmot_set_track_retirement(self.h, 1 if on else 0))

    def get_track_retirement(self) -> bool:
        return self._get_switch(self.lib.lmot_get_track_retirement)

    def seq_set_track_retirement(self, k: int, on: bool):
        self._chk(self.lib.lmot_seq_set_track_retirement(self.h, int(k), 1 if on else 0))

    def seq_get_track_retirement(self, k: int) -> bool:
        return self._get_switch(self.lib.lmot_seq_get_track_retirement, int(k))

    def _ids(self, fn, *k) -> np.ndarray:
        n = C.c_int(0)
        fn.argtypes = [C.c_void_p] + [C.c_int] * len(k) + [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        self._chk(fn(self.h, *k, None, 0, C.byref(n)))
        ids = np.zeros(n.value, np.int64)
        self._chk(fn(self.h, *k, ids.ctypes.data_as(C.c_void_p), n.value, C.byref(n)))
        return ids

    def track_ids(self) -> np.ndarray:
        """int64 IDs of the rows of the result most recently returned for the context's own table, in the order of its outputs."""
        return self._ids(self.lib.lmot_track_ids)

    def seq_track_ids(self, k: int) -> np.ndarray:
        """As track_ids, for sequence k of the tick most recently returned."""
        return self._ids(self.lib.lmot_seq_track_ids, int(k))

    # ---- track prediction (lmot_predict_tracks*) ----------------------------------------------------------------------------------
    def _predict(self, fn, k, t_us, cap):
        t = np.ascontiguousarray(np.atleast_1d(np.asarray(t_us, np.float64)))
        n_t = int(t.shape[0])
        fn.argtypes = [C.c_void_p] + [C.c_int] * len(k) + [C.c_void_p, C.c_int, C.POINTER(PredOut)]
        while True:
            cap = max(int(cap), 0)
            r = {"ids": np.zeros(cap, np.int64), "track_manage": np.zeros(cap, np.int32), "flags": np.zeros((n_t, cap), np.uint8)}
            for name, w in PRED_FIELDS:
                r[name] = np.zeros((n_t, cap, w), np.float64)
            r["P"] = r["P"].reshape(n_t, cap, 5, 5)
            o = pred_out(cap, {name: a.ctypes.data for name, a in r.items()})
            st = fn(self.h, *k, t.ctypes.data_as(C.c_void_p), n_t, C.byref(o))
            if st == ERR_CAPACITY and o.n_rows > cap:
                cap = o.n_rows
                continue
            self._chk(st)
            n = o.n_rows
            return {name: a[:n] if name in ("ids", "track_manage") else a[:, :n] for name, a in r.items()}

    def predict_tracks(self, t_us, cap: int = 1024) -> dict:
        """Every row of the context's own table predicted at the times t_us (us, 1..32 of them): ids [n], track_manage [n],
        flags [n_t, n] (PRED_*), x [n_t, n, 5], P [n_t, n, 5, 5], mode_prob [n_t, n, 3], gate_z [n_t, n, 2], gate_S [n_t, n, 4]
        (include/lmot.h, track prediction).  cap: first guess of the row count."""
        return self._predict(self.lib.lmot_predict_tracks, (), t_us, cap)

    def seq_predict_tracks(self, k: int, t_us, cap: int = 1024) -> dict:
        """As predict_tracks, for sequence k of the open set."""
        return self._predict(self.lib.lmot_seq_predict_tracks, (int(k),), t_us, cap)

    def predict_tracks_dev(self, t_us, out: PredOut, d_n_rows: int | None = None):
        """lmot_predict_tracks_dev: the own table into the device arrays of `out` (pred_out), the row count into the device int at
        d_n_rows; ordered on the context's caller stream."""
        t = np.ascontiguousarray(np.atleast_1d(np.asarray(t_us, np.float64)))
        fn = self.lib.lmot_predict_tracks_dev
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(PredOut), C.c_void_p]
        self._chk(fn(self.h, t.ctypes.data_as(C.c_void_p), int(t.shape[0]), C.byref(out), C.c_void_p(d_n_rows or 0)))

    def seq_predict_tracks_dev(self, t_us, outs, d_n_rows: int | None = None):
        """lmot_seq_predict_tracks_dev: every sequence in one launch; t_us [n_seq, n_t], outs = one PredOut per sequence, d_n_rows = device
        int[n_seq] (or None)."""
        t = np.ascontiguousarray(np.asarray(t_us, np.float64))
        if t.ndim != 2:
            raise ValueError("t_us must be [n_seq, n_t]")
        arr = (PredOut * len(outs))(*outs)
        fn = self.lib.lmot_seq_predict_tracks_dev
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(PredOut), C.c_void_p]
        self._chk(fn(self.h, t.ctypes.data_as(C.c_void_p), int(t.shape[1]), arr, C.c_void_p(d_n_rows or 0)))

    # ---- detection parameters of a sequence (lmot_seq_set_detect_params) --------------------------------------------------------
    def seq_set_detect_params(self, k: int, **fields):
        """Sequence k detects with this context's lmot_params values, `fields` replaced; no fields: it follows lmot_params again."""
        arg = C.byref(_detect_params(default_detect_params(self.params), fields)) if fields else None
        self._chk(self.lib.lmot_seq_set_detect_params(self.h, int(k), arg))

    def seq_get_detect_params(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_detect_params, DetectParams, int(k))

    # ---- sweep deskew (lmot_set_deskew / lmot_seq_set_deskew) --------------------------------------------------------------------
    def set_deskew(self, **fields):
        """The context's frames: deskew settings with `fields` replaced (on=1 turns it on; no fields: the defaults, off).  Applies from
        the next submitted frame on."""
        self._chk(self.lib.lmot_set_deskew(self.h, C.byref(_deskew(fields)) if fields else None))

    def get_deskew(self) -> dict:
        return self._get_record(self.lib.lmot_get_deskew, Deskew)

    def seq_set_deskew(self, k: int, **fields):
        """Sequence k's FRAMES steps, arguments as set_deskew."""
        self._chk(self.lib.lmot_seq_set_deskew(self.h, int(k), C.byref(_deskew(fields)) if fields else None))

    def seq_get_deskew(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_deskew, Deskew, int(k))

    # ---- detection areas (lmot_set_detect_area / lmot_seq_set_detect_area) ----------------------------------------------------------
    def _set_area(self, fn, rings, keep_outside, *k):
        a, keep = _area(rings, keep_outside)
        fn.argtypes = [C.c_void_p] + [C.c_int] * len(k) + [C.c_void_p]
        self._chk(fn(self.h, *k, C.cast(C.byref(a), C.c_void_p) if a is not None else None))

    def set_detect_area(self, rings, keep_outside=False):
        """The context's frames and batched ticks: cluster and box only the elevated points in cells inside `rings` (a sequence of (m, 2)
        vertex arrays in the vehicle frame; None or empty: off), or outside them with keep_outside.  Applies from the next submission."""
        self._set_area(self.lib.lmot_set_detect_area, rings, keep_outside)

    def seq_set_detect_area(self, k: int, rings, keep_outside=False):
        """Sequence k's FRAMES steps, arguments as set_detect_area."""
        self._set_area(self.lib.lmot_seq_set_detect_area, rings, keep_outside, int(k))

    def _get_area(self, fn, *k):
        lens = np.zeros(AREA_MAX_RINGS, np.int32)
        xy = np.zeros((AREA_MAX_VERTICES, 2), np.float64)
        nr, nv, ko = C.c_int(0), C.c_int(0), C.c_int(0)
        fn.argtypes = [C.c_void_p] + [C.c_int] * len(k) + [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        self._chk(fn(self.h, *k, C.byref(nr), lens.ctypes.data, AREA_MAX_RINGS, C.byref(nv), xy.ctypes.data, AREA_MAX_VERTICES, C.byref(ko)))
        rings, v0 = [], 0
        for L in lens[: nr.value]:
            rings.append(xy[v0 : v0 + L].copy())
            v0 += int(L)
        return dict(rings=rings, keep_outside=bool(ko.value))

    def get_detect_area(self) -> dict:
        """-> dict(rings: list of (m, 2) float64, keep_outside: bool); no rings: off"""
        return self._get_area(self.lib.lmot_get_detect_area)

    def seq_get_detect_area(self, k: int) -> dict:
        return self._get_area(self.lib.lmot_seq_get_detect_area, int(k))

    def debug_area_masks(self) -> np.ndarray:
        """lmot_debug_area_masks: (n_units, 250, 8) uint32 device masks of the most recent own-stream submission (0 units: unmasked)"""
        out = np.zeros((MAX_BATCH, 250, 8), np.uint32)
        n = C.c_int(0)
        fn = self.lib.lmot_debug_area_masks
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        self._chk(fn(self.h, out.ctypes.data, MAX_BATCH, C.byref(n)))
        return out[: n.value]

    # ---- sweep accumulation (lmot_set_accumulate) ----------------------------------------------------------------------------------
    def set_accumulate(self, **fields):
        """The context's frames: accumulation settings with `fields` replaced (sweeps=K > 1 turns it on; no fields: the defaults, off).
        Applies from the next submitted frame on; the history starts empty again."""
        self._chk(self.lib.lmot_set_accumulate(self.h, C.byref(_accumulate(fields)) if fields else None))

    def get_accumulate(self) -> dict:
        return self._get_record(self.lib.lmot_get_accumulate, Accumulate)

    def seq_set_accumulate(self, k: int, **fields):
        """Sequence k's FRAMES steps, arguments as set_accumulate."""
        self._chk(self.lib.lmot_seq_set_accumulate(self.h, int(k), C.byref(_accumulate(fields)) if fields else None))

    def seq_get_accumulate(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_accumulate, Accumulate, int(k))

    # ---- box search (lmot_set_box_search) -----------------------------------------------------------------------------------------
    def set_box_search(self, **fields):
        """The context's frames: box search settings with `fields` replaced (on=1 turns it on, n_angles=A; no fields: the defaults, off).
        Applies from the next submission on; frames in flight keep theirs."""
        self._chk(self.lib.lmot_set_box_search(self.h, C.byref(_box_search(fields)) if fields else None))

    def get_box_search(self) -> dict:
        return self._get_record(self.lib.lmot_get_box_search, BoxSearch)

    def seq_set_box_search(self, k: int, **fields):
        """Sequence k's FRAMES steps, arguments as set_box_search."""
        self._chk(self.lib.lmot_seq_set_box_search(self.h, int(k), C.byref(_box_search(fields)) if fields else None))

    def seq_get_box_search(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_box_search, BoxSearch, int(k))

    # ---- scan-matched ego motion (lmot_ego_estimate) -----------------------------------------------------------------------------
    def set_ego_match(self, **fields):
        """The context's own stream: scan matcher settings with `fields` replaced (no fields: the defaults).  Resets the matcher."""
        self._ego_set(None, fields)

    def get_ego_match(self) -> dict:
        return self._get_record(self.lib.lmot_get_ego_match, EgoMatch)

    def seq_set_ego_match(self, k: int, **fields):
        """Sequence k's matcher, arguments as set_ego_match."""
        self._ego_set(int(k), fields)

    def seq_get_ego_match(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_ego_match, EgoMatch, int(k))

    def _ego_set(self, k, fields):
        m = C.byref(_ego_match(fields)) if fields else None
        self._chk(self.lib.lmot_set_ego_match(self.h, m) if k is None else self.lib.lmot_seq_set_ego_match(self.h, k, m))

    def ego_reset(self):
        """The next ego_estimate is the stream's first: no reference, yaw back to 0."""
        self._chk(self.lib.lmot_ego_reset(self.h))

    def seq_ego_reset(self, k: int):
        self._chk(self.lib.lmot_seq_ego_reset(self.h, int(k)))

    def ego_estimate(self, points, timestamp_us) -> dict:
        """Synchronous: one host frame through the matcher -> dict of lmot_ego_out (pass its v / yaw as v_gps / yaw_gps)."""
        p, n, s = _pts(points)
        o = EgoOut()
        self._chk(self.lib.lmot_ego_estimate(self.h, p.ctypes.data if n else None, n, s, float(timestamp_us), C.byref(o)))
        return _ego_dict(o)

    def ego_estimate_dev(self, d_ptr: int, n: int, timestamp_us) -> dict:
        """Synchronous: a device XYZI frame (stride 4), ordered after the context's stream."""
        o = EgoOut()
        self._chk(self.lib.lmot_ego_estimate_dev(self.h, C.c_void_p(d_ptr or None), int(n), float(timestamp_us), C.byref(o)))
        return _ego_dict(o)

    def seq_ego_estimate(self, frames, timestamps) -> list:
        """One host frame per sequence (None: skipped, its state untouched) -> [dict or None]; frames share one stride."""
        arrs = [None if f is None else _pts(f) for f in frames]
        strides = {a[2] for a in arrs if a is not None}
        if len(strides) > 1:
            raise ValueError("every frame of one call has the same stride")
        ptrs = [None if a is None else (a[0].ctypes.data if a[1] else _EMPTY.ctypes.data) for a in arrs]
        return self._seq_ego(ptrs, [0 if a is None else a[1] for a in arrs], strides.pop() if strides else 4, timestamps, True)

    def seq_ego_estimate_dev(self, d_ptrs, ns, timestamps) -> list:
        """One device frame (stride 4) per sequence (0 / None: skipped), ordered after the context's stream."""
        return self._seq_ego([p or None for p in d_ptrs], list(ns), 4, timestamps, False)

    def _seq_ego(self, ptrs, ns, stride, timestamps, host):
        S = len(ptrs)
        P = (C.c_void_p * S)(*ptrs)
        N = (C.c_int * S)(*[int(v) for v in ns])
        T = (C.c_double * S)(*[float(t) for t in timestamps])
        O = (EgoOut * S)()
        if host:
            st = self.lib.lmot_seq_ego_estimate(self.h, P, N, S, stride, T, O)
        else:
            st = self.lib.lmot_seq_ego_estimate_dev(self.h, P, N, S, T, O)
        self._chk(st)
        return [None if ptrs[k] is None else _ego_dict(O[k]) for k in range(S)]

    # ---- ground lines (lmot_set_ground_lines) ------------------------------------------------------------------------------------
    def set_ground_lines(self, **fields):
        """The context's frames: ground lines settings with `fields` replaced (on=1 turns them on; no fields: the defaults, off).
        Applies from the next submission on; frames in flight keep theirs."""
        self._chk(self.lib.lmot_set_ground_lines(self.h, C.byref(_ground_lines(fields)) if fields else None))

    def get_ground_lines(self) -> dict:
        return self._get_record(self.lib.lmot_get_ground_lines, GroundLines)

    def seq_set_ground_lines(self, k: int, **fields):
        """Sequence k's FRAMES steps, arguments as set_ground_lines."""
        self._chk(self.lib.lmot_seq_set_ground_lines(self.h, int(k), C.byref(_ground_lines(fields)) if fields else None))

    def seq_get_ground_lines(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_ground_lines, GroundLines, int(k))

    def debug_ground_lines(self) -> np.ndarray:
        """lmot_debug_ground_lines: (n_frames, 80, 120) float32 ground grids of the most recent own-stream submission (0: lines off)"""
        out = np.zeros((MAX_BATCH, 80, 120), np.float32)
        n = C.c_int(0)
        fn = self.lib.lmot_debug_ground_lines
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        self._chk(fn(self.h, out.ctypes.data, MAX_BATCH, C.byref(n)))
        return out[: n.value]

    # ---- layered clustering (lmot_set_layers) -----------------------------------------------------------------------------------
    def set_layers(self, **fields):
        """The context's frames: layered clustering settings with `fields` replaced (on=1 turns it on; no fields: the defaults, off).
        Applies from the next submission on; frames in flight keep theirs."""
        self._chk(self.lib.lmot_set_layers(self.h, C.byref(_layers(fields)) if fields else None))

    def get_layers(self) -> dict:
        return self._get_record(self.lib.lmot_get_layers, Layers)

    def seq_set_layers(self, k: int, **fields):
        """Sequence k's FRAMES steps, arguments as set_layers."""
        self._chk(self.lib.lmot_seq_set_layers(self.h, int(k), C.byref(_layers(fields)) if fields else None))

    def seq_get_layers(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_layers, Layers, int(k))

    # ---- obstacle footprints (lmot_set_obstacles) --------------------------------------------------------------------------------
    def set_obstacles(self, **fields):
        """The context's frames: obstacle footprint settings with `fields` replaced (on=1 turns them on; no fields: the defaults, off).
        Applies from the next submission on; frames in flight keep theirs."""
        self._chk(self.lib.lmot_set_obstacles(self.h, C.byref(_obstacles(fields)) if fields else None))

    def get_obstacles(self) -> dict:
        return self._get_record(self.lib.lmot_get_obstacles, Obstacles)

    def seq_set_obstacles(self, k: int, **fields):
        """Sequence k's FRAMES steps, arguments as set_obstacles."""
        self._chk(self.lib.lmot_seq_set_obstacles(self.h, int(k), C.byref(_obstacles(fields)) if fields else None))

    def seq_get_obstacles(self, k: int) -> dict:
        return self._get_record(self.lib.lmot_seq_get_obstacles, Obstacles, int(k))

    def _obstacles_result(self, call) -> dict:
        probe = ObstaclesOut()
        st = call(C.byref(probe))
        if st not in (OK, ERR_CAPACITY):
            self._chk(st)
        rows = np.zeros(max(probe.n_obstacles, 1), OBSTACLE_DTYPE)
        nv = probe.n_vertices
        xy = np.zeros((max(nv, 1), 2), np.float32)
        out = ObstaclesOut(rows.ctypes.data, probe.n_obstacles, xy.ctypes.data, nv, 0, 0, 0)
        st = call(C.byref(out))
        if st not in (OK, ERR_CAPACITY):
            self._chk(st)
        r = rows[: out.n_obstacles]
        fit = r["vertex_count"] > 0
        stored = int((r["vertex_offset"][fit] + r["vertex_count"][fit]).max()) if fit.any() else 0     # the pool's filled part
        return {"status": st, "n_units": out.n_units, "obstacles": r.copy(), "n_vertices": out.n_vertices,
                "vertices": xy[:stored].copy()}

    def obstacles_result(self, unit: int = 0) -> dict:
        """lmot_obstacles_result: unit `unit` of the own-stream result most recently returned.  dict: status (OK, or ERR_CAPACITY when
        the vertex pool overflowed), n_units, obstacles (OBSTACLE_DTYPE rows in cluster order), n_vertices (needed in all) and
        vertices (float32 [stored, 2]); obstacle_polygons() cuts them per obstacle."""
        return self._obstacles_result(lambda o: self.lib.lmot_obstacles_result(self.h, int(unit), o))

    def seq_obstacles_result(self, k: int, unit: int = 0) -> dict:
        """lmot_seq_obstacles_result: sequence k's step of the tick most recently returned, as obstacles_result."""
        return self._obstacles_result(lambda o: self.lib.lmot_seq_obstacles_result(self.h, int(k), int(unit), o))

    def debug_point_clusters(self) -> list:
        """lmot_debug_point_clusters: one int32 array of per-point cluster ids per unit of the most recent own-stream submission, in
        each unit's cloud order ([]: it was not layered)"""
        fn = self.lib.lmot_debug_point_clusters
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_void_p]
        nu = C.c_int(0)
        npt = np.zeros(MAX_BATCH, np.int32)
        st = fn(self.h, None, 0, C.byref(nu), npt.ctypes.data)
        if st not in (OK, ERR_CAPACITY):
            self._chk(st)
        tot = int(npt[: nu.value].sum())
        ids = np.zeros(max(tot, 1), np.int32)
        self._chk(fn(self.h, ids.ctypes.data, tot, C.byref(nu), npt.ctypes.data))
        out, off = [], 0
        for u in range(nu.value):
            out.append(ids[off: off + npt[u]].copy())
            off += int(npt[u])
        return out

    def _accum_info(self, fn, *k) -> list:
        a = AccumInfo()
        self._chk(fn(self.h, *k, C.byref(a)))
        out = []
        for u in range(a.n_units):
            k = a.sweeps_used[u]
            out.append(dict(sweeps_used=k, n_points=a.n_points[u],
                            stamp_us=np.array([a.stamp_us[u][j] for j in range(k)], np.float64),
                            pose=np.array([list(a.pose[u][j]) for j in range(k)], np.float32).reshape(k, 3, 4)))
        return out

    def accumulate_info(self) -> list:
        """lmot_accumulate_info: one dict per unit of the most recently returned own-stream result (empty: it did not accumulate):
        sweeps_used, n_points (|E_acc|), stamp_us (sweeps_used,) and pose (sweeps_used, 3, 4) of the used sweeps, newest first."""
        return self._accum_info(self.lib.lmot_accumulate_info)

    def seq_accumulate_info(self, k: int) -> list:
        """lmot_seq_accumulate_info: as accumulate_info, for sequence k's most recently returned step"""
        return self._accum_info(self.lib.lmot_seq_accumulate_info, int(k))

    def seq_frame_counts(self, k: int) -> np.ndarray:
        """(n_frames, 4) int32: n_elevated, n_ground, num_cluster, n_boxes of each of sequence k's frames in the tick collected last"""
        out = np.zeros((MAX_BATCH, 4), np.int32)
        n = C.c_int(0)
        self._chk(self.lib.lmot_seq_frame_counts(self.h, int(k), out.ctypes.data_as(C.POINTER(C.c_int)), C.byref(n)))
        return out[: n.value].copy()

    @staticmethod
    def seq_scalars(n_seq, values, default=0.0):
        """Per-sequence doubles (timestamps / ego speeds / ego yaws) as the C array the seq_* calls take; one value is broadcast."""
        if isinstance(values, C.Array):
            return values
        v = np.broadcast_to(np.asarray(default if values is None else values, np.float64), (n_seq,))
        return (C.c_double * n_seq)(*[float(x) for x in v])

    def _seq_call_args(self, ptrs_ns_n, timestamps, v_gps, yaw_gps):
        ptrs, ns, S = ptrs_ns_n
        return ptrs, ns, S, self.seq_scalars(S, timestamps), self.seq_scalars(S, v_gps), self.seq_scalars(S, yaw_gps)

    def _seq_out(self, cap, want_boxes=True):
        cache = self.__dict__.setdefault("_seq_cache", {})
        if cap not in cache:
            so = SeqOut()
            sets = [self._new_track_bufs(cap) for _ in range(MAX_BATCH)]
            for k, (to, bufs) in enumerate(sets):
                so.seq[k].tracks = to
                so.seq[k].max_boxes = self.params.max_boxes
            cache[cap] = (so, sets)
        so, sets = cache[cap]
        for k, (_, bufs) in enumerate(sets):
            so.seq[k].boxes = _fp(bufs["boxes"]) if want_boxes else None
        return so, sets

    def _seq_result(self, so, sets, want_boxes=True):
        return self._seq_tick_result(so, sets, want_boxes)

    def seq(self, frames, timestamps, v_gps=None, yaw_gps=None, cap: int | None = None):
        """One tick, synchronous: `frames` = per sequence one (N, >=3) host array, or a list of them (one per sensor of a sequence with
        a sensor table); timestamps / v_gps / yaw_gps per sequence.  -> list of per-sequence dicts as frame() returns."""
        ptrs, ns, S, stride, keep = self._seq_args(frames, False)
        so, sets = self._seq_out(cap or self.params.max_tracks)
        ptrs, ns, S, ts, v, yaw = self._seq_call_args((ptrs, ns, S), timestamps, v_gps, yaw_gps)
        self._chk(self.lib.lmot_seq(self.h, ptrs, ns, S, stride, ts, v, yaw, C.byref(so)))
        return self._seq_result(so, sets)

    def seq_submit(self, frames, timestamps, v_gps=None, yaw_gps=None):
        ptrs, ns, S, stride, keep = self._seq_args(frames, False)
        self._keep = keep          # the copies are asynchronous: the host arrays must outlive the call
        ptrs, ns, S, ts, v, yaw = self._seq_call_args((ptrs, ns, S), timestamps, v_gps, yaw_gps)
        self._chk(self.lib.lmot_seq_submit(self.h, ptrs, ns, S, stride, ts, v, yaw))

    def seq_dev(self, dev_frames, timestamps, v_gps=None, yaw_gps=None):
        """dev_frames = per sequence one (device pointer, n) tuple of a stride-4 float frame, or a list of them (a sequence with a
        sensor table); or a seq_prepare handle."""
        ptrs, ns, S, _, _ = self._seq_args(dev_frames, True)
        ptrs, ns, S, ts, v, yaw = self._seq_call_args((ptrs, ns, S), timestamps, v_gps, yaw_gps)
        self._chk(self.lib.lmot_seq_dev(self.h, ptrs, ns, S, ts, v, yaw))

    def seq_collect(self, cap: int | None = None, want_boxes: bool = True):
        so, sets = self._seq_out(cap or self.params.max_tracks, want_boxes)
        self._chk(self.lib.lmot_seq_collect(self.h, C.byref(so)))
        return self._seq_result(so, sets, want_boxes)

    def seq_fetch(self, cap: int | None = None, want_boxes: bool = True):
        so, sets = self._seq_out(cap or self.params.max_tracks, want_boxes)
        self._chk(self.lib.lmot_seq_fetch(self.h, C.byref(so)))
        return self._seq_result(so, sets, want_boxes)

    # ---- tracking-only sequence ticks: caller box lists instead of frames (lmot_seq_track*) -----------------------------------------
    @staticmethod
    def _seq_lists(lists):
        """per-sequence entries -- one (m, 8, 3) box array, or a list of them for a sequence with a sensor table -- -> (ptrs, ms, n_seq,
        keep) over the tick's lists in sequence order"""
        flat = []
        for e in lists:
            flat.extend(e if isinstance(e, list) and e and all(np.ndim(x) == 3 for x in e) else [e])
        ptrs = (C.c_void_p * len(flat))()
        ms = (C.c_int * len(flat))()
        keep = []
        for i, b in enumerate(flat):
            a = np.ascontiguousarray(b, np.float32).reshape(-1, 8, 3)
            keep.append(a)
            ptrs[i], ms[i] = (a.ctypes.data if len(a) else None), len(a)
        return ptrs, ms, len(lists), keep

    def seq_track(self, lists, timestamps, v_gps=None, yaw_gps=None, cap: int | None = None):
        """One tracking-only tick, synchronous: `lists` = per sequence one (m, 8, 3) box array, or a list of them (one per sensor of a
        sequence with a sensor table).  -> list of per-sequence dicts as seq() returns (counts 0, boxes = the list that was tracked)."""
        ptrs, ms, S, keep = self._seq_lists(lists)
        so, sets = self._seq_out(cap or self.params.max_tracks)
        ptrs, ms, S, ts, v, yaw = self._seq_call_args((ptrs, ms, S), timestamps, v_gps, yaw_gps)
        self._chk(self.lib.lmot_seq_track(self.h, ptrs, ms, S, ts, v, yaw, C.byref(so)))
        return self._seq_result(so, sets)

    def seq_track_submit(self, lists, timestamps, v_gps=None, yaw_gps=None):
        """Asynchronous seq_track; results with seq_collect() / seq_fetch()."""
        ptrs, ms, S, keep = self._seq_lists(lists)
        self._keep = keep
        ptrs, ms, S, ts, v, yaw = self._seq_call_args((ptrs, ms, S), timestamps, v_gps, yaw_gps)
        self._chk(self.lib.lmot_seq_track_submit(self.h, ptrs, ms, S, ts, v, yaw))

    def seq_track_dev(self, d_lists: int, d_counts: int, cap_per_list: int, timestamps, v_gps=None, yaw_gps=None):
        """Asynchronous tracking-only tick from padded device lists (list i at d_lists + i * cap_per_list * 96 bytes, its length in the
        device int d_counts[i]), one list per frame of the tick in sequence order; ordered after the context's stream."""
        S = getattr(self, "n_seq", 0)
        ts, v, yaw = (self.seq_scalars(max(S, 1), x) for x in (timestamps, v_gps, yaw_gps))
        self._chk(self.lib.lmot_seq_track_dev(self.h, C.c_void_p(d_lists), C.c_void_p(d_counts), S, int(cap_per_list), ts, v, yaw))

    # ---- sequence ticks on each stream's own clock (lmot_seq_tick*): any subset of the sequences, each from frames or box lists -----
    def _seq_entries(self, entries, device: bool):
        """per-sequence entries -> (SeqEntry array, stride, keep).  An entry is None (the sequence skips the tick) or a dict with
        `frames=` (as one sequence's entry of seq() / seq_dev()) or `lists=` (host: as one sequence's entry of seq_track(); device: one
        device address per list, with `d_counts=` the device address of their int lengths and `cap=` boxes per list), `timestamp=`,
        `v_gps=`, `yaw_gps=` (default 0) and `restart=` (the sequence starts over with this step)."""
        arr = (SeqEntry * len(entries))()
        keep, stride = [], 4
        for k, d in enumerate(entries):
            if d is None:
                continue
            q = arr[k]
            q.flags = SEQ_RESTART if d.get("restart") else 0
            q.timestamp_us, q.v_gps, q.yaw_gps = (float(d.get(x) or 0.0) for x in ("timestamp", "v_gps", "yaw_gps"))
            if "frames" in d:
                q.kind = SEQ_FRAMES
                fr = d["frames"]
                ptrs, ns, _, st, kp = self._batch_args(fr if self._frame_list(fr, device) else [fr], device)
                stride = st
            elif device:
                q.kind = SEQ_LISTS
                ls = d["lists"] if isinstance(d["lists"], (list, tuple)) else [d["lists"]]
                ptrs, ns, kp = (C.c_void_p * len(ls))(*[int(x) for x in ls]), None, None
                q.d_counts, q.cap_per_list = int(d["d_counts"]), int(d["cap"])
            else:
                q.kind = SEQ_LISTS
                ptrs, ns, _, kp = self._seq_lists([d["lists"]])
            q.data = C.cast(ptrs, C.POINTER(C.c_void_p))
            if ns is not None:
                q.n = C.cast(ns, C.POINTER(C.c_int))
            keep += [ptrs, ns, kp]
        return arr, stride, keep

    def seq_tick(self, entries, cap: int | None = None):
        """One tick, synchronous, over host data: `entries` = one per sequence (see _seq_entries).  -> list of per-sequence dicts as
        seq() returns, None for a sequence that skipped the tick."""
        arr, stride, keep = self._seq_entries(entries, False)
        so, sets = self._seq_out(cap or self.params.max_tracks)
        self._chk(self.lib.lmot_seq_tick(self.h, arr, len(entries), stride, C.byref(so)))
        return self._seq_tick_result(so, sets)

    def seq_tick_submit(self, entries):
        """Asynchronous seq_tick; results with seq_collect() / seq_fetch()."""
        arr, stride, keep = self._seq_entries(entries, False)
        self._keep = keep          # the copies are asynchronous: the host arrays must outlive the call
        self._chk(self.lib.lmot_seq_tick_submit(self.h, arr, len(entries), stride))

    def seq_tick_dev(self, entries):
        """Asynchronous tick over device data (frames as seq_dev's entries; lists see _seq_entries), ordered after the context's stream."""
        arr, _, keep = self._seq_entries(entries, True)
        self._chk(self.lib.lmot_seq_tick_dev(self.h, arr, len(entries)))

    def seq_stepped(self) -> int:
        """Bit k: sequence k stepped in the tick most recently returned."""
        m = C.c_uint32(0)
        self._chk(self.lib.lmot_seq_stepped(self.h, C.byref(m)))
        return int(m.value)

    def _seq_tick_result(self, so, sets, want_boxes=True):
        mask = self.seq_stepped()
        return [self._frame_result(so.seq[k], sets[k][1], want_boxes) if mask >> k & 1 else None for k in range(so.n_seq)]

    def seq_tracker_load(self, k: int, dumps, init, timestamp_us, ego_velo=0.0, ego_yaw=0.0, ego_pre_yaw=0.0, ego_point_yaw=-np.pi / 2):
        """tracker_load for sequence k"""
        self._tracker_load(self.lib.lmot_seq_tracker_load, (int(k),), dumps, init, timestamp_us, ego_velo, ego_yaw, ego_pre_yaw, ego_point_yaw)

    def seq_tracker_set_ego(self, k: int, ego8):
        """tracker_set_ego for sequence k"""
        self._tracker_set_ego(self.lib.lmot_seq_tracker_set_ego, ego8, int(k))

    def seq_tracker_reset(self, k: int):
        self._chk(self.lib.lmot_seq_tracker_reset(self.h, int(k)))

    def seq_tracker_dump(self, k: int) -> np.ndarray:
        return self._tracker_dump(self.lib.lmot_seq_tracker_dump, int(k))

    def seq_tracker_get_ego(self, k: int) -> np.ndarray:
        return self._tracker_get_ego(self.lib.lmot_seq_tracker_get_ego, int(k))

    def _tracker_dump(self, fn, *k) -> np.ndarray:
        n = C.c_int(0)
        self._chk(fn(self.h, *k, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), TRACK_DUMP_DOUBLES), np.float64)
        self._chk(fn(self.h, *k, out.ctypes.data_as(C.POINTER(C.c_double)), max(n.value, 1), C.byref(n)))
        return out[: n.value]

    def _tracker_load(self, fn, k, dumps, init, timestamp_us, ego_velo, ego_yaw, ego_pre_yaw, ego_point_yaw):
        d = np.ascontiguousarray(dumps, np.float64).reshape(-1, TRACK_DUMP_DOUBLES)
        n = d.shape[0]
        if n == 0:
            d = np.zeros((1, TRACK_DUMP_DOUBLES), np.float64)
        self._chk(fn(self.h, *k, d.ctypes.data_as(C.POINTER(C.c_double)), n, int(init), C.c_double(timestamp_us), C.c_double(ego_velo),
                     C.c_double(ego_yaw), C.c_double(ego_pre_yaw), C.c_double(ego_point_yaw)))

    def _tracker_get_ego(self, fn, *k) -> np.ndarray:
        e = np.zeros(8, np.float64)
        self._chk(fn(self.h, *k, e.ctypes.data_as(C.POINTER(C.c_double))))
        return e

    def _tracker_set_ego(self, fn, ego8, *k):
        e = np.ascontiguousarray(ego8, np.float64)
        assert e.shape == (8,)
        self._chk(fn(self.h, *k, e.ctypes.data_as(C.POINTER(C.c_double))))

    def tracker_reset(self):
        self._chk(self.lib.lmot_tracker_reset(self.h))

    def tracker_num_tracks(self) -> int:
        n = C.c_int(0)
        self._chk(self.lib.lmot_tracker_num_tracks(self.h, C.byref(n)))
        return n.value

    def tracker_dump(self) -> np.ndarray:
        return self._tracker_dump(self.lib.lmot_tracker_dump)

    def tracker_load(self, dumps, init, timestamp_us, ego_velo=0.0, ego_yaw=0.0, ego_pre_yaw=0.0, ego_point_yaw=-np.pi / 2):
        self._tracker_load(self.lib.lmot_tracker_load, (), dumps, init, timestamp_us, ego_velo, ego_yaw, ego_pre_yaw, ego_point_yaw)

    def origin_points(self, timestamp_us, v_gps=0.0, yaw_gps=0.0) -> np.ndarray:
        """getOriginPoints for this frame WITHOUT advancing the tracker: (x, y, yaw, x, y, yaw + pi/2)."""
        o = np.zeros(6, np.float64)
        self._chk(self.lib.lmot_origin_points(self.h, C.c_double(timestamp_us), C.c_double(v_gps), C.c_double(yaw_gps), o.ctypes.data_as(C.POINTER(C.c_double))))
        return o

    def tracker_get_ego(self) -> np.ndarray:
        return self._tracker_get_ego(self.lib.lmot_tracker_get_ego)

    def tracker_set_ego(self, ego8):
        self._tracker_set_ego(self.lib.lmot_tracker_set_ego, ego8)

    def tracker_table(self):
        """-> (device pointer, bytes per track, capacity) of the track table (for NCCL broadcast, see shared_tracker.py)"""
        ptr = C.c_void_p(); bpt = C.c_int(0); cap = C.c_int(0)
        self._chk(self.lib.lmot_tracker_table(self.h, C.byref(ptr), C.byref(bpt), C.byref(cap)))
        return int(ptr.value), bpt.value, cap.value

    def tracker_set_num_tracks(self, n: int):
        self._chk(self.lib.lmot_tracker_set_num_tracks(self.h, int(n)))

    def enable_timing(self, on: bool = True):
        self._chk(self.lib.lmot_enable_timing(self.h, int(on)))

    def last_stage_ms(self):
        ms = (C.c_float * 4)()
        self._chk(self.lib.lmot_last_stage_ms(self.h, ms))
        return [float(x) for x in ms]

    def debug_host_ns(self, reset=True):
        ns = (C.c_double * 4)()
        self._chk(self.lib.lmot_debug_host_ns(self.h, ns, int(reset)))
        return [float(x) for x in ns]

    def last_kernel_ms(self):
        ms = (C.c_float * 32)(); n = C.c_int(0)
        self._chk(self.lib.lmot_last_kernel_ms(self.h, ms, 32, C.byref(n)))
        return [float(ms[i]) for i in range(min(n.value, 32))]

    def debug_label_grid(self):
        grid = np.zeros(250 * 250, np.int32)
        nc = C.c_int(0)
        self._chk(self.lib.lmot_debug_label_grid(self.h, grid.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nc)))
        return grid.reshape(250, 250), nc.value

    def debug_polar_grid(self):
        names = ["minz", "height", "smoothed", "hdiff", "hground"]
        arrs = [np.zeros(80 * 120, np.float32) for _ in names]
        isg = np.zeros(80 * 120, np.uint8)
        self._chk(self.lib.lmot_debug_polar_grid(self.h, *[_fp(a) for a in arrs], isg.ctypes.data_as(C.POINTER(C.c_uint8))))
        d = {k: v.reshape(80, 120) for k, v in zip(names, arrs)}
        d["isground"] = isg.reshape(80, 120)
        return d

    def debug_cell_index(self, n: int):
        ch = np.zeros(max(n, 1), np.int32); b = np.zeros(max(n, 1), np.int32)
        self._chk(self.lib.lmot_debug_cell_index(self.h, ch.ctypes.data_as(C.POINTER(C.c_int32)),
                                                 b.ctypes.data_as(C.POINTER(C.c_int32)), n))
        return ch[:n], b[:n]


def selftest_atan2f(y, x) -> np.ndarray:
    """Host-side evaluation of the library's bit-exact atan2f restatement (no GPU needed)."""
    lib = load_library()
    y = np.ascontiguousarray(y, np.float32); x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(y)
    st = lib.lmot_selftest_atan2f(_fp(y), _fp(x), int(y.size), _fp(out))
    if st != OK:
        raise LmotError(st, "selftest")
    return out


# ---- several GPUs, one track table: ctypes mirror of include/lmot_shared.h (liblmot_shared.so = host/shared_tracker.cpp + NCCL) ----
SHARED_LIB_PATH = os.path.join(HERE, "liblmot_shared.so")
SHARED_STREAMS, SHARED_FRAMES = 0, 1
SHARED_ABI_SYMBOLS = ["lmot_shared_unique_id", "lmot_shared_create", "lmot_shared_destroy", "lmot_shared_tick_dev", "lmot_shared_last_us", "lmot_shared_last_error"]
_shared_lib = None


def load_shared_library() -> C.CDLL:
    global _shared_lib
    if _shared_lib is None:
        load_library()
        if not os.path.exists(SHARED_LIB_PATH):
            raise OSError(f"{SHARED_LIB_PATH} not built")
        lib = C.CDLL(SHARED_LIB_PATH)
        lib.lmot_shared_last_error.restype = C.c_char_p
        lib.lmot_shared_last_error.argtypes = [C.c_void_p]
        lib.lmot_shared_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p]
        lib.lmot_shared_destroy.argtypes = [C.c_void_p]
        lib.lmot_shared_tick_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double, C.POINTER(TrackOut)]
        lib.lmot_shared_last_us.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        _shared_lib = lib
    return _shared_lib


def shared_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    st = load_shared_library().lmot_shared_unique_id(buf)
    if st != OK:
        raise LmotError(st, "lmot_shared_unique_id")
    return buf.raw


class SharedTracker:
    """One rank of `world` GPUs feeding ONE track table (owner rank runs the tracker; NCCL all-gather of boxes, broadcast of the table)."""

    def __init__(self, ctx: Lmot, rank: int, world: int, owner: int, unique_id: bytes):
        self.lib = load_shared_library()
        self.ctx, self.rank, self.world, self.owner = ctx, rank, world, owner
        h = C.c_void_p()
        st = self.lib.lmot_shared_create(C.byref(h), ctx.h, rank, world, owner, unique_id)
        if st != OK:
            raise LmotError(st, "lmot_shared_create")
        self.h = h

    def tick_dev(self, d_ptr: int, n: int, timestamp_us, v_gps=0.0, yaw_gps=0.0, mode=SHARED_STREAMS, frame_dt_us=0.0, cap: int | None = None):
        to, bufs = self.ctx._track_out(cap or self.ctx.params.max_tracks)
        st = self.lib.lmot_shared_tick_dev(self.h, C.c_void_p(d_ptr), int(n), float(timestamp_us), float(v_gps), float(yaw_gps), int(mode), float(frame_dt_us), C.byref(to))
        if st < 0:
            raise LmotError(st, self.lib.lmot_shared_last_error(self.h).decode())
        if self.rank == self.owner:
            return Lmot._track_result(to, bufs)
        return dict(n_tracks=to.n_tracks)

    def last_us(self):
        us = (C.c_float * 4)()
        self.lib.lmot_shared_last_us(self.h, us)
        return dict(zip(("detect", "allgather", "tracker", "broadcast"), (float(x) for x in us)))

    def close(self):
        if getattr(self, "h", None):
            self.lib.lmot_shared_destroy(self.h)
            self.h = None
