"""Sweep accumulation of batched rigs and sequence ticks (include/lmot.h, lmot_set_accumulate / lmot_seq_set_accumulate): every unit's
history and pose, a merging rig's E_acc through the stage entry points, sequences against lmot_frame twins under FRAMES / LISTS / SKIP /
RESTART schedules, the remaining reset rules and a setting change while ticks are in flight."""
import numpy as np
import pytest

from accumulate_scenes import e_acc, pose_ref, rig_apply, sparse_frames

pytestmark = pytest.mark.gpu
f32 = np.float32

# two sensors: the forward one as mounted, the other turned a quarter to the left and offset (mounting heights as lmot_params' h_sensor,
# so each sensor's ground removal is a plain context's)
POSES = [np.array([[1, 0, 0, 0.5], [0, 1, 0, 0.0], [0, 0, 1, 0.0]], f32), np.array([[0, -1, 0, -0.4], [1, 0, 0, 0.3], [0, 0, 1, 0.0]], f32)]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _params(pkg, depth=None):
    p = pkg.default_params()
    p.max_points = 1 << 17
    if depth:
        p.pipeline_depth = depth
    return p


def _same(a, b, keys=("boxes", "targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")):
    for k in keys:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k


@pytest.mark.parametrize("merge", [False, True])
def test_rig_batch_dev(pkg, synth, merge):
    """a 2-sensor rig through lmot_batch_dev: each unit's pose D = M^-1 A M (merge unit: M = identity), |E_acc| from the units' own
    clouds, n_elevated unchanged; merging: boxes and tracks equal a plain context stepping E_acc of the merged cloud"""
    import torch
    frames = sparse_frames(pkg, synth, "turn", 8)
    a, plain, twin = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        for c in (a, plain):
            c.set_sensors(POSES)
            c.set_rig_merge(merge)
        a.set_accumulate(sweeps=3, max_age_s=1.0)
        hist = []                                   # merging: (merged cloud, ts, fold) newest first; else per sensor
        hist_u = [[], []]
        dev = []
        for ts, v, yaw, pts, _, _ in frames:
            # the two sensors see the same scene from their mounts: sensor j's frame = pose_j^-1 applied to the vehicle-frame cloud
            sens = []
            for P in POSES:
                R, t = P[:, :3].astype(np.float64), P[:, 3].astype(np.float64)
                q = pts.copy()
                q[:, :3] = ((pts[:, :3].astype(np.float64) - t) @ R).astype(f32)
                sens.append(np.ascontiguousarray(q))
            d = [torch.from_numpy(x).cuda() for x in sens]
            dev.append(d)
            torch.cuda.synchronize()
            a.batch_dev([(x.data_ptr(), x.shape[0]) for x in d], ts, v, yaw)
            got = a.batch_fetch()
            info = a.accumulate_info()
            want = plain.batch(sens, ts, v, yaw)
            assert got["n_elevated"] == want["n_elevated"] and got["n_ground"] == want["n_ground"]
            e = [plain.ground_remove(x)["elevated"] for x in sens]
            fold_t = twin.origin_points(ts, v, yaw)[:3].copy()
            if merge:
                m = np.concatenate([rig_apply(P, ej) for P, ej in zip(POSES, e)])
                acc, used = e_acc(m, ts, fold_t, hist, 1.0, 1 << 17)
                grid, k = twin.component_cluster(acc)
                boxes, _ = twin.box_fit(acc, grid, k)
                tr = twin.track_step(boxes, ts, v, yaw)
                tr["boxes"] = boxes
                _same(got, tr)
                assert got["num_cluster"][0] == k
                assert len(info) == 1 and info[0]["n_points"] == len(acc) and info[0]["sweeps_used"] == len(used)
                for j, (ts_s, D) in enumerate(used):
                    assert info[0]["stamp_us"][j] == ts_s and np.array_equal(info[0]["pose"][j].view(np.uint32), D.view(np.uint32))
                f = twin.tracker_get_ego()[5:8].copy()
                hist = ([(m, ts, f)] + hist)[:2]
            else:
                twin.track_step(np.zeros((0, 8, 3), f32), ts, v, yaw)
                f = twin.tracker_get_ego()[5:8].copy()
                assert len(info) == 2
                for j in range(2):
                    acc, used = e_acc(e[j], ts, fold_t, hist_u[j], 1.0, 1 << 17)
                    assert info[j]["n_points"] == len(acc) and info[j]["sweeps_used"] == len(used)
                    for i, (ts_s, _) in enumerate(used):
                        fs = [h[2] for h in hist_u[j]][i]
                        D = pose_ref(fs, fold_t, POSES[j])
                        assert info[j]["stamp_us"][i] == ts_s and np.array_equal(info[j]["pose"][i].view(np.uint32), D.view(np.uint32))
                    hist_u[j] = ([(e[j], ts, f)] + hist_u[j])[:2]
        assert max(u["sweeps_used"] for u in info) == 2
    finally:
        a.close(); plain.close(); twin.close()


def test_sequences_mixed_schedules(pkg, synth):
    """sequence 0 accumulates (FRAMES every tick), 1 is plain, 2 accumulates under FRAMES / LISTS / SKIP / RESTART: each equals its own
    lmot_frame twin with the same setting (a LISTS step is lmot_track_step, a restart lmot_tracker_reset)"""
    fr = [sparse_frames(pkg, synth, kind, 10, seed=s) for kind, s in (("turn", 3), ("straight", 4), ("turn", 5))]
    sched = ["F", "F", "L", "F", "S", "F", "R", "F", "F", "L"]
    ctx = pkg.Lmot(_params(pkg))
    tw = [pkg.Lmot(_params(pkg)) for _ in range(3)]
    try:
        ctx.seq_open(3, ring=4)
        for k in (0, 2):
            ctx.seq_set_accumulate(k, sweeps=3, max_age_s=1.0)
            tw[k].set_accumulate(sweeps=3, max_age_s=1.0)
        assert ctx.seq_get_accumulate(0) == dict(sweeps=3, max_age_s=1.0) and ctx.seq_get_accumulate(1)["sweeps"] == 1
        lists = np.zeros((0, 8, 3), f32)
        for t in range(10):
            entries, want = [], []
            for k in range(3):
                ts, v, yaw, pts, _, _ = fr[k][t]
                s = sched[t] if k == 2 else "F"
                if s == "S":
                    entries.append(None); want.append(None)
                    continue
                if s == "L":
                    entries.append(dict(lists=[lists], timestamp=ts, v_gps=v, yaw_gps=yaw))
                    want.append(tw[k].track_step(lists, ts, v, yaw))
                    continue
                if s == "R":
                    tw[k].tracker_reset()
                entries.append(dict(frames=pts, timestamp=ts, v_gps=v, yaw_gps=yaw, restart=s == "R"))
                want.append(tw[k].frame(pts, ts, v, yaw))
            got = ctx.seq_tick(entries)
            for k in range(3):
                if want[k] is None:
                    assert got[k] is None
                    continue
                _same(got[k], want[k], ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb"))
                if entries[k].get("frames") is not None:
                    _same(got[k], want[k], ("boxes",))
                    assert got[k]["n_elevated"] == want[k]["n_elevated"] and got[k]["num_cluster"] == want[k]["num_cluster"]
                    gi, wi = ctx.seq_accumulate_info(k), tw[k].accumulate_info()
                    assert len(gi) == len(wi)
                    for x, y in zip(gi, wi):
                        assert x["n_points"] == y["n_points"] and x["sweeps_used"] == y["sweeps_used"]
                        assert np.array_equal(x["pose"], y["pose"]) and np.array_equal(x["stamp_us"], y["stamp_us"])
                else:
                    assert ctx.seq_accumulate_info(k) == []
        for k in range(3):
            assert np.array_equal(ctx.seq_tracker_dump(k), tw[k].tracker_dump())
    finally:
        ctx.close()
        for c in tw:
            c.close()


def test_more_reset_rules(pkg, synth):
    """lmot_tracker_load, lmot_tracker_set_ego, lmot_set_rig_merge and their sequence forms start the history afresh; a change of the
    units (a 2-sensor batched tick between frames) too"""
    frames = sparse_frames(pkg, synth, "straight", 12)
    a = pkg.Lmot(_params(pkg))
    try:
        a.set_accumulate(sweeps=3)
        it = iter(frames)

        def step():
            ts, v, yaw, pts, _, _ = next(it)
            a.frame(pts, ts, v, yaw)
            return a.accumulate_info()[0]["sweeps_used"]

        assert step() == 0 and step() == 1
        a.tracker_set_ego(a.tracker_get_ego())
        assert step() == 0 and step() == 1
        a.tracker_load(a.tracker_dump(), 1, frames[3][0], ego_point_yaw=float(a.tracker_get_ego()[7]))
        assert step() == 0 and step() == 1
        a.set_rig_merge(False)
        assert step() == 0 and step() == 1
        ts, v, yaw, pts, _, _ = frames[8]
        a.batch([pts, pts], ts, v, yaw)              # two units: another layout
        assert len(a.accumulate_info()) == 2 and all(u["sweeps_used"] == 0 for u in a.accumulate_info())
        ts, v, yaw, pts, _, _ = frames[9]
        a.frame(pts, ts, v, yaw)
        assert a.accumulate_info()[0]["sweeps_used"] == 0
        a.seq_open(2)
        a.seq_set_accumulate(0, sweeps=3, max_age_s=100.0)
        clock = [2e7]
        _, v, yaw, pts, _, _ = frames[11]

        def tick():
            clock[0] += 1e5
            a.seq_tick([dict(frames=pts, timestamp=clock[0], v_gps=v, yaw_gps=yaw), None])
            return a.seq_accumulate_info(0)[0]["sweeps_used"]

        assert tick() == 0 and tick() == 1
        for reset in (lambda: a.seq_tracker_reset(0), lambda: a.seq_set_rig_merge(0, False), lambda: a.seq_set_sensors(0, None),
                      lambda: a.seq_tracker_set_ego(0, a.seq_tracker_get_ego(0)),
                      lambda: a.seq_tracker_load(0, a.seq_tracker_dump(0), 1, clock[0], ego_point_yaw=float(a.seq_tracker_get_ego(0)[7]))):
            reset()
            assert tick() == 0 and tick() == 1
        a.seq_open(2)                                 # a new set: settings off, history gone
        assert a.seq_get_accumulate(0)["sweeps"] == 1
    finally:
        a.close()


def test_setting_change_in_flight(pkg, synth):
    """submitted frames keep the setting they were submitted with: a change between submissions equals the same change between
    synchronous frames"""
    frames = sparse_frames(pkg, synth, "turn", 10)
    a, b = pkg.Lmot(_params(pkg, depth=4)), pkg.Lmot(_params(pkg))
    try:
        got, want = [], []
        for c in (a, b):
            c.set_accumulate(sweeps=4, max_age_s=1.0)
        for i, (ts, v, yaw, pts, _, _) in enumerate(frames):
            if i == 5:
                a.set_accumulate(sweeps=2, max_age_s=1.0)
                b.set_accumulate(sweeps=2, max_age_s=1.0)
            a.frame_submit(pts, ts, v, yaw)
            want.append((b.frame(pts, ts, v, yaw), b.accumulate_info()))
            if a.frames_in_flight() >= 4:
                got.append((a.frame_collect(), a.accumulate_info()))
        while a.frames_in_flight() > 0:
            got.append((a.frame_collect(), a.accumulate_info()))
        for (g, gi), (w, wi) in zip(got, want):
            _same(g, w)
            assert [u["sweeps_used"] for u in gi] == [u["sweeps_used"] for u in wi]
            assert [u["n_points"] for u in gi] == [u["n_points"] for u in wi]
        assert [u["sweeps_used"] for _, wi in want for u in wi][4:7] == [3, 0, 1]
    finally:
        a.close(); b.close()
