"""Every per-stream setting and tracker-state call in its two forms: the context's own stream (lmot_X) and sequence k (lmot_seq_X).

Both forms are driven through the same calls on one context: the defaults (NULL), valid values read back, one invalid value per
validated field (refused, the setting unchanged), NULL outputs, and for the sequence forms k = -1, k = n_seq and a context with no set
open.  The differences between the two forms that callers can observe are pinned where they are documented: which calls forget the
sweep-accumulation history (seen in accumulate_info after the next step), which drop uncollected sequence ticks (seen in lmot_seq_collect),
the timing-mode refusal of lmot_seq_predict_tracks and the frame total of lmot_seq_set_sensors.
"""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_SEQ = 2
K = 1                               # the sequence the sequence forms address


def _params(pkg):
    p = pkg.default_params()
    p.max_points = 1 << 16
    p.pipeline_depth = 2
    p.result_ring = 4
    return p


@pytest.fixture
def ctx(pkg):
    c = pkg.Lmot(_params(pkg))
    c.seq_open(N_SEQ, 4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def frames(synth):
    cfg = synth.SceneConfig(rings=32, azimuths=900, n_objects=20, seed=5)
    return [(ts, np.ascontiguousarray(p, np.float32)) for ts, p in synth.frames(cfg, 4)]


def _forms(ctx, name):
    """(label, call) of both forms of lmot_[seq_]<name>: call(*args) passes the context (and k) in front"""
    lib = ctx.lib
    own, seq = getattr(lib, "lmot_" + name), getattr(lib, "lmot_seq_" + name)
    return [("own", lambda *a: own(ctx.h, *a)), ("seq", lambda *a: seq(ctx.h, K, *a))]


def _bad_k(pkg, ctx, name, *args):
    """the sequence form refuses every k that names no open sequence, before it looks at anything else"""
    fn = getattr(ctx.lib, "lmot_seq_" + name)
    for k in (-1, N_SEQ, 1 << 20):
        assert fn(ctx.h, k, *args) == pkg.ERR_INVALID, (name, k)
    closed = pkg.Lmot(_params(pkg))
    try:
        assert fn(closed.h, 0, *args) == pkg.ERR_INVALID, (name, "no set open")
    finally:
        closed.close()


def _vals(s):
    """a ctypes structure's fields as nested lists"""
    def v(x):
        return [v(e) for e in x] if isinstance(x, C.Array) else x
    return {name: v(getattr(s, name)) for name, _ in s._fields_}


def _step_own(ctx, frames, i):
    ts, pts = frames[i]
    return ctx.frame(pts, ts)


def _step_seq(ctx, frames, i):
    ts, pts = frames[i]
    return ctx.seq([pts] * N_SEQ, [ts] * N_SEQ)


# ---- settings records: set NULL / valid / invalid, get, get NULL ---------------------------------------------------------------------

def _defaults(pkg, name, cls):
    s = cls()
    assert getattr(pkg.load_library(), "lmot_default_" + name)(C.byref(s)) == pkg.OK
    return _vals(s)


def _struct_cases(pkg):
    tp_valid = pkg._tracker_params(dict(gamma_g=7.5, p_g=0.97, lifetime_thres=2, static_lifetime=6, std_a=[1.5, 2.5, 3.5],
                                        trans=[[0.85, 0.1, 0.05], [0.07, 0.88, 0.05], [0.1, 0.05, 0.85]], p0_diag=[0.4, 0.6, 2.5, 8.0, 1.2]))
    zero_col = [[0.0, 0.5, 0.5], [0.0, 0.5, 0.5], [0.0, 0.0, 0.0]]
    return {
        "tracker_params": (pkg.TrackerParams, pkg._tracker_params, tp_valid,
                           [dict(gamma_g=0.0), dict(std_las_x=math.nan), dict(p_g=1.5), dict(p_d=0.0), dict(mode_prob0=[0.0, 0.5, 0.5]),
                            dict(distance_thres=math.inf), dict(static_dist=math.nan), dict(trans=zero_col), dict(trans=[[1.5, 0, 0], [0, 1, 0], [0, 0, 1]]),
                            dict(lifetime_thres=-1), dict(static_lifetime=-1)]),
        "deskew": (pkg.Deskew, pkg._deskew, pkg._deskew(dict(on=1, time_field=4, time_scale=1e-6, time_offset=0.5, t_min=-0.05, t_max=0.05)),
                   [dict(time_scale=math.nan), dict(time_offset=math.inf), dict(t_min=math.nan), dict(t_max=math.inf), dict(t_min=0.0, t_max=0.0),
                    dict(t_min=-1.5, t_max=0.0), dict(time_field=2)]),
        "accumulate": (pkg.Accumulate, pkg._accumulate, pkg._accumulate(dict(sweeps=3, max_age_s=0.3)),
                       [dict(sweeps=0), dict(sweeps=pkg.MAX_SWEEPS + 1), dict(max_age_s=math.nan), dict(max_age_s=0.0)]),
        "box_search": (pkg.BoxSearch, pkg._box_search, pkg._box_search(dict(on=1, n_angles=45)),
                       [dict(on=2), dict(n_angles=0), dict(n_angles=361)]),
        "ground_lines": (pkg.GroundLines, pkg._ground_lines, pkg._ground_lines(dict(on=1, max_slope=0.2, max_rmse=0.1, max_step=0.25)),
                         [dict(on=2), dict(max_slope=0.0), dict(max_rmse=math.nan), dict(max_step=-1.0), dict(max_step=math.inf)]),
        "layers": (pkg.Layers, pkg._layers, pkg._layers(dict(on=1, n_slices=16, slice_m=0.25, z_min=-0.3, gap_slices=3)),
                   [dict(on=2), dict(n_slices=0), dict(n_slices=33), dict(slice_m=0.0), dict(z_min=math.nan), dict(gap_slices=-1),
                    dict(n_slices=4, gap_slices=4)]),
        "obstacles": (pkg.Obstacles, pkg._obstacles, pkg._obstacles(dict(on=1, max_vertices=1000)),
                      [dict(on=2), dict(max_vertices=139), dict(max_vertices=(1 << 24) + 1)]),
    }


@pytest.mark.parametrize("name", ["tracker_params", "deskew", "accumulate", "box_search", "ground_lines", "layers", "obstacles"])
def test_setting_records(pkg, ctx, name):
    cls, make, valid, invalid = _struct_cases(pkg)[name]
    defaults = _defaults(pkg, name, cls)
    want_valid = _vals(valid)
    for label, set_ in _forms(ctx, "set_" + name):
        get_ = dict(_forms(ctx, "get_" + name))[label]

        def got():
            s = cls()
            assert get_(C.byref(s)) == pkg.OK, (name, label)
            return _vals(s)

        assert got() == defaults, (name, label, "fresh")
        assert set_(C.byref(valid)) == pkg.OK, (name, label)
        assert got() == want_valid, (name, label)
        for bad in invalid:
            assert set_(C.byref(make(bad))) == pkg.ERR_INVALID, (name, label, bad)
            assert got() == want_valid, (name, label, bad, "unchanged")
        assert set_(None) == pkg.OK, (name, label, "NULL: the defaults")
        assert got() == defaults, (name, label)
        assert get_(None) == pkg.ERR_INVALID, (name, label)
    # the two streams are separate records: the own stream back on the valid values leaves sequence K on the defaults
    assert getattr(ctx.lib, "lmot_set_" + name)(ctx.h, C.byref(valid)) == pkg.OK
    seq_get = getattr(ctx.lib, "lmot_seq_get_" + name)
    for k in range(N_SEQ):
        s = cls()
        assert seq_get(ctx.h, k, C.byref(s)) == pkg.OK and _vals(s) == defaults, k
    _bad_k(pkg, ctx, "set_" + name, C.byref(valid))
    _bad_k(pkg, ctx, "set_" + name, None)
    _bad_k(pkg, ctx, "get_" + name, C.byref(cls()))


def test_deskew_on_is_normalised(pkg, ctx):
    for label, set_ in _forms(ctx, "set_deskew"):
        assert set_(C.byref(pkg._deskew(dict(on=5)))) == pkg.OK
        d = pkg.Deskew()
        assert dict(_forms(ctx, "get_deskew"))[label](C.byref(d)) == pkg.OK and d.on == 1, label


# ---- sensors, rig merge, retirement --------------------------------------------------------------------------------------------------

def _table(pkg, n, yaw0=0.1):
    arr = (pkg.Sensor * max(n, 1))()
    for j in range(n):
        pkg.load_library().lmot_default_sensor(None, C.byref(arr[j]))
        c, s = math.cos(yaw0 * (j + 1)), math.sin(yaw0 * (j + 1))
        arr[j].pose[:] = [c, -s, 0.0, 0.5 * j, s, c, 0.0, -0.25 * j, 0.0, 0.0, 1.0, 1.5]
        arr[j].h_sensor = 1.5 + 0.1 * j
        arr[j].sensor_height = 1.6 + 0.1 * j
    return arr


def test_sensors(pkg, ctx):
    for label, set_ in _forms(ctx, "set_sensors"):
        get_ = dict(_forms(ctx, "get_sensors"))[label]
        out, n = (pkg.Sensor * 8)(), C.c_int(-1)

        def got():
            assert get_(out, 8, C.byref(n)) == pkg.OK, label
            return [_vals(out[j]) for j in range(n.value)]

        assert got() == [], label
        t = _table(pkg, 2)
        assert set_(t, 2) == pkg.OK, label
        want = [_vals(t[j]) for j in range(2)]
        assert got() == want, label
        bad_pose = _table(pkg, 1)
        bad_pose[0].pose[0] = 2.0                                          # not a rotation
        nan_pose = _table(pkg, 1)
        nan_pose[0].pose[3] = math.nan
        nan_h = _table(pkg, 1)
        nan_h[0].t_hmax = math.inf
        for args in ((_table(pkg, 1), -1), (_table(pkg, 8), 9), (None, 1), (bad_pose, 1), (nan_pose, 1), (nan_h, 1)):
            assert set_(*args) == pkg.ERR_INVALID, (label, args[1])
            assert got() == want, label
        # outputs: NULL count is fine, a short table is cut, negative or NULL-with-capacity is refused
        assert get_(out, 1, None) == pkg.OK and _vals(out[0]) == want[0], label
        assert get_(None, 0, C.byref(n)) == pkg.OK and n.value == 2, label
        assert get_(out, -1, C.byref(n)) == pkg.ERR_INVALID, label
        assert get_(None, 1, C.byref(n)) == pkg.ERR_INVALID, label
        assert set_(None, 0) == pkg.OK and got() == [], label
    _bad_k(pkg, ctx, "set_sensors", _table(pkg, 1), 1)
    _bad_k(pkg, ctx, "get_sensors", (pkg.Sensor * 8)(), 8, None)


def test_sensor_frame_total(pkg, ctx):
    """a tick's frames stay within LMOT_MAX_BATCH across the sequences (one frame for a sequence without a table); the own stream has
    no such total"""
    lib, h = ctx.lib, ctx.h
    assert lib.lmot_set_sensors(h, _table(pkg, 8), 8) == pkg.OK
    assert lib.lmot_seq_set_sensors(h, 0, _table(pkg, 7), 7) == pkg.OK                 # 7 + 1
    assert lib.lmot_seq_set_sensors(h, 1, _table(pkg, 2), 2) == pkg.ERR_INVALID        # 7 + 2
    assert lib.lmot_seq_set_sensors(h, 1, _table(pkg, 1), 1) == pkg.OK                 # 7 + 1
    assert lib.lmot_seq_set_sensors(h, 0, _table(pkg, 8), 8) == pkg.ERR_INVALID        # 8 + 1
    n = C.c_int(-1)
    assert lib.lmot_seq_get_sensors(h, 0, None, 0, C.byref(n)) == pkg.OK and n.value == 7
    assert lib.lmot_seq_set_sensors(h, 0, None, 0) == pkg.OK                           # 1 + 1
    assert lib.lmot_seq_set_sensors(h, 1, _table(pkg, 7), 7) == pkg.OK                 # 1 + 7


@pytest.mark.parametrize("name", ["rig_merge", "track_retirement"])
def test_switches(pkg, ctx, name):
    for label, set_ in _forms(ctx, "set_" + name):
        get_ = dict(_forms(ctx, "get_" + name))[label]
        v = C.c_int(-1)
        assert get_(C.byref(v)) == pkg.OK and v.value == 0, (name, label)
        assert set_(1) == pkg.OK and get_(C.byref(v)) == pkg.OK and v.value == 1, (name, label)
        if name == "rig_merge":
            assert set_(2) == pkg.ERR_INVALID and get_(C.byref(v)) == pkg.OK and v.value == 1, label
        else:                                                              # any non-zero value turns it on
            assert set_(0) == pkg.OK and set_(7) == pkg.OK and get_(C.byref(v)) == pkg.OK and v.value == 1, label
        assert set_(0) == pkg.OK and get_(C.byref(v)) == pkg.OK and v.value == 0, (name, label)
        assert get_(None) == pkg.ERR_INVALID, (name, label)
    _bad_k(pkg, ctx, "set_" + name, 1)
    _bad_k(pkg, ctx, "get_" + name, C.byref(C.c_int()))


# ---- detection areas ---------------------------------------------------------------------------------------------------------------

def _area_struct(pkg, rings, keep=0, lens=None):
    arrs = [np.asarray(r, np.float64).reshape(-1, 2) for r in rings]
    L = np.array(lens if lens is not None else [len(a) for a in arrs], np.int32)
    xy = np.ascontiguousarray(np.concatenate(arrs), np.float64)
    return pkg.Area(len(L), L.ctypes.data, xy.ctypes.data, keep), (L, xy)


def test_detect_area(pkg, ctx):
    sq = [[5, -5], [30, -5], [30, 5], [5, 5]]
    tri = [[-10, 0], [-20, 5], [-20, -5]]
    for label, set_ in _forms(ctx, "set_detect_area"):
        get_ = dict(_forms(ctx, "get_detect_area"))[label]
        lens, xy = np.zeros(64, np.int32), np.zeros((1024, 2), np.float64)
        nr, nv, ko = C.c_int(-1), C.c_int(-1), C.c_int(-1)

        def got():
            assert get_(C.byref(nr), lens.ctypes.data, 64, C.byref(nv), xy.ctypes.data, 1024, C.byref(ko)) == pkg.OK, label
            return nr.value, lens[: nr.value].tolist(), xy[: nv.value].tolist(), ko.value

        assert got() == (0, [], [], 0), label
        a, keep = _area_struct(pkg, [sq, tri], 1)
        assert set_(C.byref(a)) == pkg.OK, label
        want = (2, [4, 3], [list(map(float, v)) for v in sq + tri], 1)
        assert got() == want, label
        # (each struct with the arrays it points into, kept alive until the call)
        bads = [_area_struct(pkg, [sq], 2), _area_struct(pkg, [sq[:2]]), _area_struct(pkg, [[[math.nan, 0], [1, 0], [1, 1]]]),
                _area_struct(pkg, [np.zeros((1025, 2))]), _area_struct(pkg, [tri] * 65), (pkg.Area(-1, None, None, 0), ())]
        for b, _keep in bads:
            assert set_(C.byref(b)) == pkg.ERR_INVALID, label
            assert got() == want, label
        # outputs: every one may be NULL with no capacity; negative capacities and NULL arrays with capacity are refused
        assert get_(None, None, 0, None, None, 0, None) == pkg.OK, label
        assert get_(C.byref(nr), None, -1, None, None, 0, None) == pkg.ERR_INVALID, label
        assert get_(None, None, 0, C.byref(nv), None, -1, None) == pkg.ERR_INVALID, label
        assert get_(None, None, 1, None, None, 0, None) == pkg.ERR_INVALID, label
        assert get_(None, None, 0, None, None, 1, None) == pkg.ERR_INVALID, label
        assert set_(None) == pkg.OK and got() == (0, [], [], 0), label
    a, keep = _area_struct(pkg, [sq])
    _bad_k(pkg, ctx, "set_detect_area", C.byref(a))
    _bad_k(pkg, ctx, "get_detect_area", None, None, 0, None, None, 0, None)


def test_seq_detect_params(pkg, ctx):
    """sequence-only: NULL follows lmot_params, a valid record reads back, an invalid one is refused"""
    lib, h = ctx.lib, ctx.h
    d = pkg.DetectParams()
    assert lib.lmot_seq_get_detect_params(h, K, C.byref(d)) == pkg.OK
    base = _vals(d)
    mine = pkg._detect_params(pkg.default_detect_params(ctx.params), dict(roi_m=40.0, t_hmax=-0.5))
    assert lib.lmot_seq_set_detect_params(h, K, C.byref(mine)) == pkg.OK
    assert lib.lmot_seq_get_detect_params(h, K, C.byref(d)) == pkg.OK and _vals(d) == _vals(mine)
    bad = pkg._detect_params(pkg.default_detect_params(ctx.params), dict(roi_m=0.0))
    assert lib.lmot_seq_set_detect_params(h, K, C.byref(bad)) == pkg.ERR_INVALID
    assert lib.lmot_seq_get_detect_params(h, K, C.byref(d)) == pkg.OK and _vals(d) == _vals(mine)
    assert lib.lmot_seq_get_detect_params(h, K, None) == pkg.ERR_INVALID
    assert lib.lmot_seq_set_detect_params(h, K, None) == pkg.OK
    assert lib.lmot_seq_get_detect_params(h, K, C.byref(d)) == pkg.OK and _vals(d) == base
    _bad_k(pkg, ctx, "set_detect_params", None)
    _bad_k(pkg, ctx, "get_detect_params", C.byref(d))


# ---- results of the step most recently returned: accumulation info, obstacles, track IDs ---------------------------------------------

def test_step_results(pkg, ctx, frames):
    lib, h = ctx.lib, ctx.h
    forms_info = _forms(ctx, "accumulate_info")
    forms_obs = _forms(ctx, "obstacles_result")
    forms_ids = _forms(ctx, "track_ids")
    n = C.c_int(-1)
    for (label, info), (_, obs), (_, ids) in zip(forms_info, forms_obs, forms_ids):
        a = pkg.AccumInfo()
        assert info(C.byref(a)) == pkg.OK and a.n_units == 0, label
        assert info(None) == pkg.ERR_INVALID, label
        o = pkg.ObstaclesOut()
        assert obs(0, C.byref(o)) == pkg.ERR_STATE, label                     # no step returned yet
        assert obs(0, None) == pkg.ERR_INVALID, label
        assert ids(None, 0, C.byref(n)) == pkg.ERR_STATE, label
        assert ids(None, 0, None) == pkg.ERR_INVALID, label
        assert ids(None, -1, C.byref(n)) == pkg.ERR_INVALID, label
        assert ids(None, 1, C.byref(n)) == pkg.ERR_INVALID, label
    ctx.set_obstacles(on=1)
    ctx.seq_set_obstacles(K, on=1)
    for i in range(3):
        _step_own(ctx, frames, i)
        _step_seq(ctx, frames, i)
    for (label, info), (_, obs), (_, ids) in zip(forms_info, forms_obs, forms_ids):
        o = pkg.ObstaclesOut()
        assert obs(0, C.byref(o)) == pkg.OK and o.n_units == 1 and o.n_obstacles > 0, label
        assert obs(1, C.byref(o)) == pkg.ERR_INVALID and obs(-1, C.byref(o)) == pkg.ERR_INVALID, label
        assert ids(None, 0, C.byref(n)) == pkg.OK and n.value > 0, label
        v = np.full(n.value, -1, np.int64)
        assert ids(v.ctypes.data, n.value, C.byref(n)) == pkg.OK, label
        assert np.array_equal(v, np.arange(n.value)), label                # no retirement: the IDs are the rows
    o = pkg.ObstaclesOut()
    assert lib.lmot_seq_obstacles_result(h, 0, 0, C.byref(o)) == pkg.ERR_STATE       # sequence 0 has obstacles off
    _bad_k(pkg, ctx, "accumulate_info", C.byref(pkg.AccumInfo()))
    _bad_k(pkg, ctx, "obstacles_result", 0, C.byref(pkg.ObstaclesOut()))
    _bad_k(pkg, ctx, "track_ids", None, 0, C.byref(n))


# ---- track prediction ----------------------------------------------------------------------------------------------------------------

def test_predict(pkg, ctx, frames):
    lib, h = ctx.lib, ctx.h
    t = np.array([frames[0][0]], np.float64)
    empty = pkg.pred_out(0, {})
    for label, fn in _forms(ctx, "predict_tracks"):
        assert fn(t.ctypes.data, 1, None) == pkg.ERR_INVALID, label
        assert fn(t.ctypes.data, 1, C.byref(empty)) == pkg.ERR_STATE, label     # the table has no stamp yet
    for i in range(2):
        _step_own(ctx, frames, i)
        _step_seq(ctx, frames, i)
    ts = frames[1][0]
    for label, fn in _forms(ctx, "predict_tracks"):
        ok, many, nan, early = np.array([ts, ts + 5e4]), np.full(33, ts), np.array([math.nan]), np.array([ts - 1.0])
        assert fn(None, 1, C.byref(empty)) == pkg.ERR_INVALID, label
        assert fn(ok.ctypes.data, 0, C.byref(empty)) == pkg.ERR_INVALID, label
        assert fn(many.ctypes.data, 33, C.byref(empty)) == pkg.ERR_INVALID, label
        assert fn(nan.ctypes.data, 1, C.byref(empty)) == pkg.ERR_INVALID, label
        assert fn(early.ctypes.data, 1, C.byref(empty)) == pkg.ERR_INVALID, label
        assert fn(ok.ctypes.data, 2, C.byref(pkg.pred_out(-1, {}))) == pkg.ERR_INVALID, label
        e = pkg.pred_out(0, {})
        assert fn(ok.ctypes.data, 2, C.byref(e)) == pkg.ERR_CAPACITY and e.n_rows > 0, label
    # timing mode: the sequence form refuses before it looks at its outputs; the own form does not refuse
    ctx.enable_timing(True)
    try:
        assert lib.lmot_seq_predict_tracks(h, K, t.ctypes.data, 1, None) == pkg.ERR_STATE
        assert lib.lmot_seq_predict_tracks(h, -1, t.ctypes.data, 1, None) == pkg.ERR_INVALID
        assert lib.lmot_predict_tracks(h, t.ctypes.data, 1, None) == pkg.ERR_INVALID
        e = pkg.pred_out(0, {})
        now = np.array([ts])
        assert lib.lmot_predict_tracks(h, now.ctypes.data, 1, C.byref(e)) == pkg.ERR_CAPACITY
    finally:
        ctx.enable_timing(False)
    _bad_k(pkg, ctx, "predict_tracks", t.ctypes.data, 1, C.byref(empty))


# ---- tracker state: dump, load, reset, ego -------------------------------------------------------------------------------------------

def _dump(fn):
    n = C.c_int(-1)
    assert fn(None, 0, C.byref(n)) in (0, -3)
    out = np.zeros((max(n.value, 1), 236), np.float64)
    st = fn(out.ctypes.data_as(C.POINTER(C.c_double)), max(n.value, 1), C.byref(n))
    assert st == 0
    return out[: n.value]


def test_tracker_state(pkg, ctx, frames):
    for i in range(3):
        _step_own(ctx, frames, i)
        _step_seq(ctx, frames, i)
    dp = C.POINTER(C.c_double)
    for label, dump in _forms(ctx, "tracker_dump"):
        fns = {name: dict(_forms(ctx, "tracker_" + name))[label] for name in ("load", "get_ego", "set_ego", "reset")}
        d = _dump(dump)
        assert len(d) > 0, label
        n = C.c_int(-1)
        assert dump(None, -1, C.byref(n)) == pkg.ERR_INVALID, label
        short = np.zeros((1, 236))
        st = dump(short.ctypes.data_as(dp), 1, C.byref(n))
        assert st == (pkg.ERR_CAPACITY if len(d) > 1 else pkg.OK) and n.value == len(d), label
        e = np.zeros(8)
        assert fns["get_ego"](e.ctypes.data_as(dp)) == pkg.OK and e[0] == 1.0 and e[1] == frames[2][0], label
        assert fns["get_ego"](None) == pkg.ERR_INVALID, label
        # load: refused arguments leave the table alone; a dump loads back to the same dump
        cd = C.c_double
        args = (cd(frames[2][0]), cd(e[2]), cd(e[3]), cd(e[4]), cd(-math.pi / 2))
        assert fns["load"](None, -1, 1, *args) == pkg.ERR_INVALID, label
        assert fns["load"](None, 1, 1, *args) == pkg.ERR_INVALID, label
        big = np.zeros((ctx.params.max_tracks + 1, 236))
        assert fns["load"](big.ctypes.data_as(dp), ctx.params.max_tracks + 1, 1, *args) == pkg.ERR_CAPACITY, label
        assert np.array_equal(_dump(dump), d), label
        assert fns["load"](np.ascontiguousarray(d).ctypes.data_as(dp), len(d), 1, *args) == pkg.OK, label
        assert np.array_equal(_dump(dump), d), label
        e2 = np.zeros(8)
        assert fns["get_ego"](e2.ctypes.data_as(dp)) == pkg.OK, label
        assert e2[0] == 1.0 and e2[1] == frames[2][0] and list(e2[5:]) == [0.0, 0.0, -math.pi / 2], label
        # set_ego / get_ego round trip
        assert fns["set_ego"](None) == pkg.ERR_INVALID, label
        assert fns["set_ego"](e.ctypes.data_as(dp)) == pkg.OK, label
        assert fns["get_ego"](e2.ctypes.data_as(dp)) == pkg.OK and np.array_equal(e, e2), label
        # reset: an empty table without a stamp
        assert fns["reset"]() == pkg.OK, label
        assert len(_dump(dump)) == 0, label
        assert fns["get_ego"](e2.ctypes.data_as(dp)) == pkg.OK and e2[0] == 0.0, label
    for name, args in (("dump", (None, 0, C.byref(C.c_int()))), ("get_ego", (np.zeros(8).ctypes.data_as(dp),)),
                       ("set_ego", (np.zeros(8).ctypes.data_as(dp),)), ("reset", ()),
                       ("load", (None, 0, 0, C.c_double(0), C.c_double(0), C.c_double(0), C.c_double(0), C.c_double(0)))):
        _bad_k(pkg, ctx, "tracker_" + name, *args)


# ---- which calls drop uncollected sequence ticks ---------------------------------------------------------------------------------------

def _ego(ctx, k):
    e = np.zeros(8)
    if k is None:
        assert ctx.lib.lmot_tracker_get_ego(ctx.h, e.ctypes.data_as(C.POINTER(C.c_double))) == 0
    else:
        assert ctx.lib.lmot_seq_tracker_get_ego(ctx.h, k, e.ctypes.data_as(C.POINTER(C.c_double))) == 0
    return e


def _load0(lib, h, k, n):
    cd = C.c_double
    z = np.zeros((1, 236))
    args = (z.ctypes.data_as(C.POINTER(C.c_double)), n, 0, cd(0), cd(0), cd(0), cd(0), cd(-math.pi / 2))
    return lib.lmot_tracker_load(h, *args) if k is None else lib.lmot_seq_tracker_load(h, k, *args)


DROP_CASES = {
    # name: (call(ctx) -> status, expected status, ticks dropped)
    "seq_reset": (lambda c: c.lib.lmot_seq_tracker_reset(c.h, K), 0, True),
    "seq_reset_bad_k": (lambda c: c.lib.lmot_seq_tracker_reset(c.h, N_SEQ), -1, False),
    "own_reset": (lambda c: c.lib.lmot_tracker_reset(c.h), 0, False),
    "seq_load": (lambda c: _load0(c.lib, c.h, K, 0), 0, True),
    "seq_load_invalid": (lambda c: _load0(c.lib, c.h, K, -1), -1, False),
    "own_load": (lambda c: _load0(c.lib, c.h, None, 0), 0, False),
    "seq_set_ego": (lambda c: c.lib.lmot_seq_tracker_set_ego(c.h, K, _ego(c, K).ctypes.data_as(C.POINTER(C.c_double))), 0, True),
    "seq_set_ego_null": (lambda c: c.lib.lmot_seq_tracker_set_ego(c.h, K, None), -1, False),
    "own_set_ego": (lambda c: c.lib.lmot_tracker_set_ego(c.h, _ego(c, None).ctypes.data_as(C.POINTER(C.c_double))), 0, False),
}


@pytest.mark.parametrize("case", sorted(DROP_CASES))
def test_seq_ticks_dropped(pkg, ctx, frames, case):
    call, want, dropped = DROP_CASES[case]
    _step_own(ctx, frames, 0)
    _step_seq(ctx, frames, 0)
    ts, pts = frames[1]
    ctx.seq_submit([pts] * N_SEQ, [ts] * N_SEQ)
    assert call(ctx) == want
    st = ctx.lib.lmot_seq_collect(ctx.h, None)
    assert st == (pkg.ERR_STATE if dropped else pkg.OK), case


# ---- which calls forget the sweep-accumulation history ---------------------------------------------------------------------------------

FORGET_CASES = {
    # name: (form, call(ctx, pkg) -> status, expected status, history forgotten)
    "own_sensors_invalid": ("own", lambda c, p: c.lib.lmot_set_sensors(c.h, None, -1), -1, True),
    "seq_sensors_invalid": ("seq", lambda c, p: c.lib.lmot_seq_set_sensors(c.h, K, None, -1), -1, False),
    "seq_sensors_bad_k": ("seq", lambda c, p: c.lib.lmot_seq_set_sensors(c.h, N_SEQ, None, 0), -1, False),
    "seq_sensors_frame_total": ("seq", lambda c, p: c.lib.lmot_seq_set_sensors(c.h, K, _table(p, 8), 8), -1, True),
    "own_sensors_none": ("own", lambda c, p: c.lib.lmot_set_sensors(c.h, None, 0), 0, True),
    "seq_sensors_none": ("seq", lambda c, p: c.lib.lmot_seq_set_sensors(c.h, K, None, 0), 0, True),
    "own_rig_merge_invalid": ("own", lambda c, p: c.lib.lmot_set_rig_merge(c.h, 2), -1, True),
    "seq_rig_merge_invalid": ("seq", lambda c, p: c.lib.lmot_seq_set_rig_merge(c.h, K, 2), -1, True),
    "own_rig_merge_off": ("own", lambda c, p: c.lib.lmot_set_rig_merge(c.h, 0), 0, True),
    "seq_rig_merge_off": ("seq", lambda c, p: c.lib.lmot_seq_set_rig_merge(c.h, K, 0), 0, True),
    "own_load_invalid": ("own", lambda c, p: _load0(c.lib, c.h, None, -1), -1, True),
    "seq_load_invalid": ("seq", lambda c, p: _load0(c.lib, c.h, K, -1), -1, True),
    "own_set_ego_null": ("own", lambda c, p: c.lib.lmot_tracker_set_ego(c.h, None), -1, False),
    "seq_set_ego_null": ("seq", lambda c, p: c.lib.lmot_seq_tracker_set_ego(c.h, K, None), -1, False),
    "own_set_ego": ("own", lambda c, p: c.lib.lmot_tracker_set_ego(c.h, _ego(c, None).ctypes.data_as(C.POINTER(C.c_double))), 0, True),
    "seq_set_ego": ("seq", lambda c, p: c.lib.lmot_seq_tracker_set_ego(c.h, K, _ego(c, K).ctypes.data_as(C.POINTER(C.c_double))), 0, True),
    "own_accumulate_same": ("own", lambda c, p: c.lib.lmot_set_accumulate(c.h, C.byref(p._accumulate(dict(sweeps=3, max_age_s=10.0)))), 0, True),
    "seq_accumulate_same": ("seq", lambda c, p: c.lib.lmot_seq_set_accumulate(c.h, K, C.byref(p._accumulate(dict(sweeps=3, max_age_s=10.0)))), 0, True),
    "own_layers": ("own", lambda c, p: c.lib.lmot_set_layers(c.h, None), 0, False),
    "seq_tracker_params": ("seq", lambda c, p: c.lib.lmot_seq_set_tracker_params(c.h, K, None), 0, False),
    "own_other_stream": ("own", lambda c, p: c.lib.lmot_seq_set_rig_merge(c.h, K, 2), -1, False),
    "seq_other_stream": ("seq", lambda c, p: c.lib.lmot_set_rig_merge(c.h, 2), -1, False),
}


@pytest.mark.parametrize("case", sorted(FORGET_CASES))
def test_history_forgotten(pkg, ctx, frames, case):
    form, call, want, forgotten = FORGET_CASES[case]
    ctx.set_accumulate(sweeps=3, max_age_s=10.0)
    ctx.seq_set_accumulate(K, sweeps=3, max_age_s=10.0)
    for i in range(2):
        _step_own(ctx, frames, i)
        _step_seq(ctx, frames, i)
    assert call(ctx, pkg) == want, case
    if form == "own":
        _step_own(ctx, frames, 2)
        info = ctx.accumulate_info()
    else:
        _step_seq(ctx, frames, 2)
        info = ctx.seq_accumulate_info(K)
    assert len(info) == 1, case
    assert info[0]["sweeps_used"] == (0 if forgotten else 2), case
