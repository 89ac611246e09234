"""GPU parity of the sensor rig (lmot_set_sensors): each sensor of a batched tick has its own mounting pose and mounting height.

Scene: synth.py frames seen by F sensors mounted at different heights h, yaws and offsets.  Sensor k's cloud is the synth frame
with z shifted by (2 - h), so its ground sits where a sensor mounted at h sees it; its t_hmin / t_hmax are the defaults shifted by
the same amount and its h_sensor / sensor_height are h.  Oracles:
  * detection: the reference's groundRemove / componentClustering / boxFitting with its mutable globals hSeonsor, tHmin, tHmax
    (ground_removal.cpp:27,29,33) and sensorHeight (box_fitting.cpp:26, read at :123 and :385) set to the sensor's values -- they
    are exported data symbols of the compiled reference, written here through ctypes and restored afterwards;
  * the vehicle-frame list: a numpy float32 restatement of the documented arithmetic, ((r0 x + r1 y) + r2 z) + t per row;
  * the tracker: the reference's immUkfJpdaf on that list (moved on into the dead-reckoned global frame with the arithmetic of
    test_global_frame_gpu when global_frame = 1).
Bars as in test_batch_gpu: counts and boxes bit-exact, identical trackManage / static / visible flags, UKF states within 1e-4
relative on positive-definite filters.
"""
import contextlib
import ctypes as C

import numpy as np
import pytest

from test_global_frame_gpu import _ego, xf_apply, xf_pair
from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32

T_HMIN, T_HMAX, H_DEFAULT = -2.0, -0.4, 2.0


def yaw_pose(c, s, tx, ty, tz):
    """sensor -> vehicle [R | t] for a yaw with cosine c and sine s (exact values for the quarter turns used here)"""
    return np.array([[c, -s, 0, tx], [s, c, 0, ty], [0, 0, 1, tz]], f32)


# yaw 0, +pi/2, -pi/2, pi; offsets of +-1.5 m / +-0.8 m; mounting heights 2.0 / 1.2 / 0.8 / 1.8 m
RIG = [(yaw_pose(1, 0, 1.5, 0.0, 2.0), 2.0), (yaw_pose(0, 1, 0.0, 0.8, 1.2), 1.2),
       (yaw_pose(0, -1, 0.0, -0.8, 0.8), 0.8), (yaw_pose(-1, 0, -1.5, 0.0, 1.8), 1.8)]
# a second table (in-flight test): other poses, other heights
RIG_B = [(yaw_pose(0, 1, 0.3, -0.2, 1.6), 1.6), (yaw_pose(1, 0, -0.7, 0.4, 1.0), 1.0),
         (yaw_pose(-1, 0, 2.0, 0.0, 2.2), 2.2), (yaw_pose(0, -1, 0.0, 1.1, 1.4), 1.4)]


def mount(h):
    d = H_DEFAULT - h
    return dict(h_sensor=h, t_hmin=T_HMIN + d, t_hmax=T_HMAX + d, sensor_height=h)


def set_rig(ctx, rig):
    ms = [mount(h) for _, h in rig]
    ctx.set_sensors([p for p, _ in rig], **{k: [m[k] for m in ms] for k in ms[0]})


def rig_apply(m, boxes):
    """the library's contract in numpy float32: per row ((r0*x + r1*y) + r2*z) + t, one rounding per operation"""
    p = np.asarray(boxes, f32).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    rows = [((m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z) + m[r, 3] for r in range(3)]
    return np.stack(rows, 1).astype(f32).reshape(np.shape(boxes))


# lmot_sensor field -> the reference global that plays its role
REF_GLOBALS = dict(h_sensor="hSeonsor", t_hmin="tHmin", t_hmax="tHmax", sensor_height="sensorHeight")


@contextlib.contextmanager
def ref_mount(ref, h):
    """the reference runs with mounting height h while the block runs; its own values come back afterwards"""
    g = {k: C.c_float.in_dll(ref.lib, name) for k, name in REF_GLOBALS.items()}
    saved = {k: v.value for k, v in g.items()}
    assert saved == {k: float(f32(v)) for k, v in mount(H_DEFAULT).items()}, saved     # the reference's defaults: nothing leaked
    for k, v in mount(h).items():
        g[k].value = v
    try:
        yield
    finally:
        for k, v in saved.items():
            g[k].value = v


def ref_detect(ref, pts, h):
    with ref_mount(ref, h):
        e, g = ref.ground_remove(pts)
        grid, k = ref.component_clustering(e)
        b, _ = ref.box_fitting(e, grid, k)
    return (len(e), len(g), k, len(b)), b


def rig_ticks(synth, rig, n_ticks, seed=41, n_objects=30):
    """(ts, [sensor k's cloud]) per tick: scene k seen from height rig[k]'s h"""
    gens = [synth.frames(synth.SceneConfig(seed=seed + k, n_objects=n_objects, rings=32, azimuths=900), n_ticks) for k in range(len(rig))]
    for _ in range(n_ticks):
        tick = [next(g) for g in gens]
        frames = []
        for (_, p), (_, h) in zip(tick, rig):
            q = p.copy()
            q[:, 2] += f32(H_DEFAULT - h)
            frames.append(q)
        yield tick[0][0], frames


def expected_detection(ref, rig, ticks):
    """per tick: per-frame counts under each sensor's mount, and the vehicle-frame list"""
    out = []
    for ts, frames in ticks:
        per, lists = [], []
        for pts, (pose, h) in zip(frames, rig):
            c, b = ref_detect(ref, pts, h)
            per.append(c)
            lists.append(rig_apply(pose, b))
        out.append((per, np.concatenate(lists)))
    return out


def ego_sequence(pkg, ticks):
    probe = pkg.Lmot(_params(pkg, 1))        # the dead-reckoning fold the tracker will run, peeked tick by tick
    try:
        egos = []
        for f, (ts, _) in enumerate(ticks):
            v, yaw = _ego(f)
            egos.append(probe.origin_points(ts, v, yaw))
            probe.track_step(np.zeros((0, 8, 3), f32), ts, v, yaw)
        return egos
    finally:
        probe.close()


def _params(pkg, gf):
    p = pkg.default_params()
    p.global_frame = gf
    return p


def check_tick(r, per, vlist, a, back, f):
    assert list(zip(r["n_elevated"], r["n_ground"], r["num_cluster"], r["n_boxes"])) == per, f
    assert r["boxes"].shape == vlist.shape and np.array_equal(r["boxes"].view(np.uint32), vlist.view(np.uint32)), f
    for k in ("track_manage", "is_static", "is_vis"):
        assert np.array_equal(r[k], a[k]), (f, k)
    tg, vb = (a["targets"], a["vis_bb"]) if back is None else (xf_apply(back, a["targets"]), xf_apply(back, a["vis_bb"]))
    np.testing.assert_allclose(r["targets"], tg, rtol=1e-4, atol=1e-4)
    assert r["vis_bb"].shape == vb.shape
    np.testing.assert_allclose(r["vis_bb"], vb, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("gf", [0, 1])
def test_rig_parity(pkg, ref_intended, synth, gf):
    ref = ref_intended
    n_ticks = 30
    ticks = list(rig_ticks(synth, RIG, n_ticks))
    det = expected_detection(ref, RIG, ticks)
    # every sensor yields boxes, and the 0.8 m sensor's boxes depend on its own thresholds
    assert all(sum(per[k][3] for per, _ in det) > 0 for k in range(len(RIG)))
    differs = 0
    for ts, frames in ticks[:5]:
        _, b_own = ref_detect(ref, frames[2], 0.8)
        _, b_def = ref_detect(ref, frames[2], H_DEFAULT)
        differs += not (b_own.shape == b_def.shape and np.array_equal(b_own, b_def))
    assert differs > 0
    egos = ego_sequence(pkg, ticks) if gf else [None] * n_ticks
    ref.tracker_reset()
    want = []
    for f, ((ts, _), (per, vlist)) in enumerate(zip(ticks, det)):
        v, yaw = _ego(f)
        fwd, back = xf_pair(egos[f]) if gf else (None, None)
        a = ref.tracker_step(vlist if not gf else xf_apply(fwd, vlist), ts, v, yaw)
        want.append((a, back, ref.tracker_dump()))
    # synchronous ticks (lmot_batch), with the track table compared after every tick
    ctx = pkg.Lmot(_params(pkg, gf))
    try:
        set_rig(ctx, RIG)
        worst = 0.0
        for f, ((ts, frames), (per, vlist), (a, back, da)) in enumerate(zip(ticks, det, want)):
            r = ctx.batch(frames, ts, *_ego(f))
            check_tick(r, per, vlist, a, back, f)
            db = ctx.tracker_dump()
            assert np.array_equal(da[:, INTS], db[:, INTS]), f
            ok = _pd_tracks(da)
            err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
            if err.size:
                worst = max(worst, float(err.max()))
                assert err.max() < TOL, (f, float(err.max()))
        assert (want[-1][0]["track_manage"] > 0).sum() > 10
        print(f"rig of {len(RIG)} sensors, global_frame={gf}: worst relative state error (positive-definite tracks) {worst:.3g}")
    finally:
        ctx.close()
    # the same ticks pipelined from device frames (lmot_batch_dev), collected afterwards
    import torch
    ctx = pkg.Lmot(_params(pkg, gf))
    try:
        set_rig(ctx, RIG)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        with torch.cuda.stream(stream):
            dev = [[torch.from_numpy(p).cuda() for p in frames] for _, frames in ticks]
            for f, ((ts, frames), d) in enumerate(zip(ticks, dev)):
                ctx.batch_dev([(t.data_ptr(), len(p)) for t, p in zip(d, frames)], ts, *_ego(f))
        for f, ((per, vlist), (a, back, _)) in enumerate(zip(det, want)):
            check_tick(ctx.batch_collect(), per, vlist, a, back, f)
        ctx.set_stream(None)
    finally:
        ctx.close()


def test_identity_sensors_are_no_sensors(pkg, synth):
    """sensors equal to lmot_default_sensor: the same boxes, counts and track table as a context without sensors, bit for bit;
    and after lmot_set_sensors(ctx, NULL, 0) as well"""
    plain, rig = pkg.Lmot(), pkg.Lmot()
    try:
        rig.set_sensors([np.eye(3, 4, dtype=f32)] * 4)
        got = rig.get_sensors()
        d = pkg.default_params()
        assert np.array_equal(got["poses"], np.stack([np.eye(3, 4, dtype=f32)] * 4))
        assert np.all(got["h_sensor"] == f32(d.h_sensor)) and np.all(got["t_hmin"] == f32(d.t_hmin))
        assert np.all(got["t_hmax"] == f32(d.t_hmax)) and np.all(got["sensor_height"] == f32(d.sensor_height))
        ticks = list(rig_ticks(synth, [(None, H_DEFAULT)] * 4, 25, seed=7))
        n_boxes = 0
        for f, (ts, frames) in enumerate(ticks):
            if f == 20:
                rig.set_sensors(None)
                assert len(rig.get_sensors()["poses"]) == 0
            a, b = plain.batch(frames, ts, *_ego(f)), rig.batch(frames, ts, *_ego(f))
            for k in ("n_elevated", "n_ground", "num_cluster", "n_boxes"):
                assert a[k] == b[k], (f, k)
            for k in ("boxes", "targets", "vis_bb", "vandyaw", "track_manage", "is_static", "is_vis"):
                assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), (f, k)
            assert plain.tracker_dump().tobytes() == rig.tracker_dump().tobytes(), f
            n_boxes += len(a["boxes"])
        assert n_boxes > 0
    finally:
        plain.close(); rig.close()


def test_in_flight_ticks_keep_their_table(pkg, ref_intended, synth):
    """tick A submitted under table A, the table changed, tick B submitted under table B, both collected afterwards"""
    ref = ref_intended
    ctx = pkg.Lmot()
    try:
        ta = list(rig_ticks(synth, RIG, 3, seed=51))
        tb = list(rig_ticks(synth, RIG_B, 3, seed=51))
        plan = [(ta[0], RIG), (tb[1], RIG_B), (ta[2], RIG)]
        ref.tracker_reset()
        want = []
        for (ts, frames), rig in plan:
            (per, vlist), = expected_detection(ref, rig, [(ts, frames)])
            want.append((per, vlist, ref.tracker_step(vlist, ts)))
        for (ts, frames), rig in plan:
            set_rig(ctx, rig)
            ctx.batch_submit(frames, ts)
        for f, (per, vlist, a) in enumerate(want):
            check_tick(ctx.batch_collect(), per, vlist, a, None, f)
    finally:
        ctx.close()


def test_track_step_lists_dev_with_poses(pkg, ref_intended, synth):
    """three padded device lists through three poses, then one list per step (the frames-mode shape) through pose 0"""
    import torch
    ref = ref_intended
    rig = RIG[:3]
    ticks = list(rig_ticks(synth, rig, 12, seed=61, n_objects=40))
    lists = [[ref_detect(ref, p, h)[1] for p, (_, h) in zip(frames, rig)] for _, frames in ticks]
    cap = 128
    ctx = pkg.Lmot()
    try:
        set_rig(ctx, rig)
        ref.tracker_reset()
        for f, ((ts, _), ls) in enumerate(zip(ticks, lists)):
            buf = np.zeros((len(ls), cap, 8, 3), f32)
            for l, b in enumerate(ls):
                buf[l, : len(b)] = b
            d_buf = torch.from_numpy(buf).cuda()
            d_cnt = torch.tensor([len(b) for b in ls], dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            ctx.track_step_lists_dev(d_buf.data_ptr(), d_cnt.data_ptr(), len(ls), cap, ts)
            r = ctx.frame_fetch()
            vlist = np.concatenate([rig_apply(p, b) for (p, _), b in zip(rig, ls)])
            a = ref.tracker_step(vlist, ts)
            assert np.array_equal(r["boxes"].view(np.uint32), vlist.view(np.uint32)), f
            assert np.array_equal(r["track_manage"], a["track_manage"]), f
            np.testing.assert_allclose(r["targets"], a["targets"], rtol=1e-4, atol=1e-4)
        assert (a["track_manage"] > 0).sum() > 5
        # one list per step: sensor 0 for every step
        ctx.tracker_reset(); ref.tracker_reset()
        for f, ((ts, _), ls) in enumerate(zip(ticks, lists)):
            b = ls[0]
            buf = np.zeros((cap, 8, 3), f32); buf[: len(b)] = b
            d_buf = torch.from_numpy(buf).cuda()
            d_cnt = torch.tensor([len(b)], dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            ctx.track_step_lists_dev(d_buf.data_ptr(), d_cnt.data_ptr(), 1, cap, ts)
            r = ctx.frame_fetch()
            vlist = rig_apply(rig[0][0], b)
            a = ref.tracker_step(vlist, ts)
            assert np.array_equal(r["boxes"].view(np.uint32), vlist.view(np.uint32)), f
            assert np.array_equal(r["track_manage"], a["track_manage"]), f
    finally:
        ctx.close()


def test_sensor_table_validation(pkg):
    ctx = pkg.Lmot()
    try:
        set_rig(ctx, RIG)
        before = ctx.get_sensors()

        def rejected(poses, **kw):
            with pytest.raises(pkg.LmotError) as ei:
                ctx.set_sensors(poses, **kw)
            assert ei.value.status == pkg.ERR_INVALID
            after = ctx.get_sensors()
            assert all(np.array_equal(before[k], after[k]) for k in before)

        good = [p for p, _ in RIG]
        rejected([good[0]] * 9)                                       # more than LMOT_MAX_BATCH
        for bad in (np.nan, np.inf):
            p = [q.copy() for q in good]; p[1][0, 3] = bad
            rejected(p)                                               # non-finite translation
            p = [q.copy() for q in good]; p[2][2, 2] = bad
            rejected(p)                                               # non-finite rotation
            rejected(good, h_sensor=[2.0, bad, 2.0, 2.0])             # non-finite threshold
            rejected(good, sensor_height=bad)
        p = [q.copy() for q in good]; p[3][:, :3] *= f32(1.0001)
        rejected(p)                                                   # scaled: not orthonormal
        p = [q.copy() for q in good]; p[0][0, 1] = f32(1e-4)
        rejected(p)                                                   # sheared
        p = [q.copy() for q in good]; p[0][0, 1] = f32(4e-6)
        ctx.set_sensors(p)                                            # within 1e-5: accepted
        assert len(ctx.get_sensors()["poses"]) == 4
        import torch
        # more frames / lists than sensors
        set_rig(ctx, RIG[:3])
        pts = torch.zeros((16, 4), device="cuda")
        with pytest.raises(pkg.LmotError) as ei:
            ctx.batch_dev([(pts.data_ptr(), 16)] * 4, 1e5)
        assert ei.value.status == pkg.ERR_INVALID
        with pytest.raises(pkg.LmotError) as ei:
            ctx.batch([np.zeros((16, 4), f32)] * 4, 1e5)
        assert ei.value.status == pkg.ERR_INVALID
        d_cnt = torch.zeros(4, dtype=torch.int32, device="cuda")
        d_buf = torch.zeros((4, 8, 8, 3), device="cuda")
        with pytest.raises(pkg.LmotError) as ei:
            ctx.track_step_lists_dev(d_buf.data_ptr(), d_cnt.data_ptr(), 4, 8, 1e5)
        assert ei.value.status == pkg.ERR_INVALID
        ctx.set_sensors(None)
        ctx.batch([np.zeros((16, 4), f32)] * 4, 1e5)                  # no sensors: any frame count again
    finally:
        ctx.close()
