"""Sensor tables for independent sequences (lmot_seq_set_sensors): each sequence of a tick brings one frame per sensor of its own rig.

Contract (include/lmot.h): sequence k with a table gives bit for bit what a separate context with the same lmot_params and
lmot_set_sensors(that table) gives when it receives sequence k's frames through lmot_batch -- per-frame and summed counts, the
vehicle-frame box list, targets, vandyaw, trackManage, static / visible flags, vis_bb, the status and the track-table dump.  A sequence
without a table gives what such a context gives through lmot_frame.  Every test compares against these twin contexts; one case also
anchors sequence 0 to the reference, as test_rig_parity does.
"""
import ctypes as C

import numpy as np
import pytest

from test_sensor_rig_gpu import H_DEFAULT, RIG, RIG_B, mount, ref_detect, rig_apply, yaw_pose
from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32

N_TICKS = 30
FIELDS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb", "boxes")
COUNTS = ("n_elevated", "n_ground", "num_cluster", "n_boxes")


def _params(pkg, global_frame=0, max_tracks=512, max_boxes=None):
    p = pkg.default_params()
    p.max_points = 1 << 16
    p.max_tracks = max_tracks
    p.pipeline_depth = 2
    p.result_ring = 4
    p.global_frame = global_frame
    if max_boxes is not None:
        p.max_boxes = max_boxes
    return p


def _table_kw(rig):
    ms = [mount(h) for _, h in rig]
    return dict(poses=[p for p, _ in rig], **{k: [m[k] for m in ms] for k in ms[0]})


def set_seq_rig(ctx, k, rig):
    if rig is None:
        ctx.seq_set_sensors(k, None)
    else:
        ctx.seq_set_sensors(k, **_table_kw(rig))


class _RigSeq:
    """Sequence k: its sensor table (None: no table, one frame from the default height), one synth scene per sensor seen from that
    sensor's height, and its own start stamp, frame interval, ego speed and yaw rate (as _Seq in test_sequences_gpu)."""

    def __init__(self, synth, k, rig, n_ticks=N_TICKS, seed=500, n_objects=24, n_sensors=None):
        self.rig = rig
        heights = [h for _, h in rig] if rig else [H_DEFAULT]
        n_sensors = n_sensors or len(heights)
        heights = (heights * n_sensors)[:n_sensors]
        gens = [synth.frames(synth.SceneConfig(seed=seed + 17 * k + j, n_objects=n_objects, rings=32, azimuths=900), n_ticks)
                for j in range(n_sensors)]
        self.frames = []
        for _ in range(n_ticks):
            fr = []
            for g, h in zip(gens, heights):
                q = next(g)[1].copy()
                q[:, 2] += f32(H_DEFAULT - h)
                fr.append(q)
            self.frames.append(fr)
        self.t0 = 1.0e6 * (1 + k) + 1234.5 * k
        self.dt = 100000.0 + 5000.0 * k
        self.v = 1.5 * k
        self.rate = 0.02 * (k - 3)

    def ts(self, f):
        return self.t0 + f * self.dt

    def ego(self, f):
        return self.v + 0.1 * f, 0.3 * (self.rate != 0) + self.rate * f


def _entry(frames, rig):
    """a sequence's entry of a tick: a list of frames with a table, one frame without"""
    return list(frames[: len(rig)]) if rig else frames[0]


class _Twin:
    """the oracle of one sequence: lmot_batch with set_sensors(rig), or lmot_frame without a table"""

    def __init__(self, pkg, prm, rig):
        self.pkg, self.ctx, self.rig = pkg, pkg.Lmot(prm), None
        self.set(rig)

    def set(self, rig):
        self.rig = rig
        if rig is None:
            self.ctx.set_sensors(None)
        else:
            self.ctx.set_sensors(**_table_kw(rig))

    def step(self, frames, ts, v, yaw):
        """-> (status, result dict, per-frame counts), through the raw calls so that an error status keeps its outputs"""
        c = self.ctx
        if self.rig:
            ptrs, ns, F, stride, keep = c._batch_args(list(frames[: len(self.rig)]), False)
            bo, bufs = c._batch_out(c.params.max_tracks)
            st = c.lib.lmot_batch(c.h, ptrs, ns, F, stride, C.c_double(ts), C.c_double(v), C.c_double(yaw), C.byref(bo))
            r = c._batch_result(bo, bufs)
            counts = [tuple(int(r[k][i]) for k in COUNTS) for i in range(F)]
            r.update({k: int(sum(r[k])) for k in ("n_elevated", "n_ground", "num_cluster")})
        else:
            p, n, s = self.pkg._pts(frames[0])
            fo, bufs = c._frame_out(c.params.max_tracks)
            st = c.lib.lmot_frame(c.h, self.pkg._fp(p), n, s, C.c_double(ts), C.c_double(v), C.c_double(yaw), C.byref(fo))
            r = c._frame_result(fo, bufs)
            counts = [(r["n_elevated"], r["n_ground"], r["num_cluster"], fo.n_boxes)]
        return st, r, counts

    def close(self):
        self.ctx.close()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


def _same(got, fc, want, what):
    """got: the sequence's dict, fc: its seq_frame_counts rows; want: the twin's (status, dict, per-frame counts)"""
    _, w, wc = want
    assert [tuple(int(x) for x in row) for row in fc] == wc, (what, "frame counts")
    assert (got["n_elevated"], got["n_ground"], got["num_cluster"]) == (w["n_elevated"], w["n_ground"], w["num_cluster"]), what
    for key in FIELDS:
        assert got[key].shape == w[key].shape and np.array_equal(_bits(got[key]), _bits(w[key])), (what, key)


def _same_tables(ctx, twins, what):
    for k, t in enumerate(twins):
        a, b = ctx.seq_tracker_dump(k), t.ctx.tracker_dump()
        assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (what, k, "dump")
        assert np.array_equal(ctx.seq_tracker_get_ego(k), t.ctx.tracker_get_ego()), (what, k, "ego")


def _seq_raw(ctx, entries, ts, v, yaw):
    """lmot_seq through the raw call: -> (status, per-sequence dicts)"""
    ptrs, ns, S, stride, keep = ctx._seq_args(entries, False)
    so, sets = ctx._seq_out(ctx.params.max_tracks)
    ptrs, ns, S, t_, v_, y_ = ctx._seq_call_args((ptrs, ns, S), ts, v, yaw)
    st = ctx.lib.lmot_seq(ctx.h, ptrs, ns, S, stride, t_, v_, y_, C.byref(so))
    return st, ctx._seq_result(so, sets)


def _run(ctx, seqs, tables, n_ticks, mode, twins, before=None):
    """n_ticks ticks of every sequence -- `tables(f)` gives each sequence's table at tick f, `before(f)` runs before tick f is
    submitted -- through lmot_seq (sync) or pipelined lmot_seq_dev (dev, collected afterwards); every tick is compared with the twins,
    which step tick by tick.  -> per tick the list of sequence results"""
    import torch
    S = len(seqs)
    want, done = [], []
    stream = None
    keep = []
    for f in range(n_ticks):
        if before:
            before(f)
        rigs = tables(f)
        entries = [_entry(s.frames[f], r) for s, r in zip(seqs, rigs)]
        ts = [s.ts(f) for s in seqs]
        v = [s.ego(f)[0] for s in seqs]
        yaw = [s.ego(f)[1] for s in seqs]
        want.append([twins[k].step(seqs[k].frames[f], ts[k], v[k], yaw[k]) for k in range(S)])
        if mode == "sync":
            got = ctx.seq(entries, ts, v, yaw)
            done.append((got, [ctx.seq_frame_counts(k) for k in range(S)]))
        else:
            if stream is None:
                stream = torch.cuda.Stream()
                ctx.set_stream(stream.cuda_stream)
            with torch.cuda.stream(stream):
                dev = []
                for e in entries:
                    ts_ = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in (e if isinstance(e, list) else [e])]
                    keep.append(ts_)
                    tup = [(t.data_ptr(), len(t)) for t in ts_]
                    dev.append(tup if isinstance(e, list) else tup[0])
                ctx.seq_dev(dev, ts, v, yaw)
    if mode == "dev":
        for f in range(n_ticks):
            got = ctx.seq_collect()
            done.append((got, [ctx.seq_frame_counts(k) for k in range(S)]))
        ctx.set_stream(None)
    for f, ((got, fcs), w) in enumerate(zip(done, want)):
        for k in range(S):
            _same(got[k], fcs[k], w[k], (f, k))
    return [g for g, _ in done]


LAYOUTS = {"2x4": [RIG, RIG_B], "mixed": [RIG, RIG_B[1:2], None, RIG_B[2:4]]}


@pytest.mark.parametrize("mode", ["sync", "dev"])
@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("layout", ["2x4", "mixed"])
def test_seq_rig_parity(pkg, synth, ref_intended, layout, gf, mode):
    """30 ticks with moving egos: 2 sequences x 4 sensors, or 4 + 1 (with a table) + 1 (no table) + 2 frames; every sequence equals its
    twin on every tick and in its final table.  2x4 / gf 0 / sync also anchors sequence 0 to the reference."""
    rigs = LAYOUTS[layout]
    seqs = [_RigSeq(synth, k, r) for k, r in enumerate(rigs)]
    prm = _params(pkg, gf)
    ctx = pkg.Lmot(prm)
    twins = [_Twin(pkg, _params(pkg, gf), r) for r in rigs]
    try:
        ctx.seq_open(len(rigs), ring=N_TICKS if mode == "dev" else 4)
        for k, r in enumerate(rigs):
            set_seq_rig(ctx, k, r)
        got = _run(ctx, seqs, lambda f: rigs, N_TICKS, mode, twins)
        _same_tables(ctx, twins, layout)
        assert ctx.tracker_num_tracks() == 0                  # the context's own table is untouched
        assert sum(len(g[0]["boxes"]) for g in got) > 0 and (got[-1][0]["track_manage"] > 0).sum() > 5
        if layout == "2x4" and gf == 0 and mode == "sync":
            ref = ref_intended
            ref.tracker_reset()
            s = seqs[0]
            worst = 0.0
            for f in range(N_TICKS):
                per, lists = [], []
                for p, (pose, h) in zip(s.frames[f], RIG):
                    c, b = ref_detect(ref, p, h)
                    per.append(c)
                    lists.append(rig_apply(pose, b))
                vlist = np.concatenate(lists)
                a = ref.tracker_step(vlist, s.ts(f), *s.ego(f))
                r = got[f][0]
                assert (r["n_elevated"], r["n_ground"], r["num_cluster"]) == tuple(sum(c[i] for c in per) for i in range(3)), f
                assert r["boxes"].shape == vlist.shape and np.array_equal(r["boxes"].view(np.uint32), vlist.view(np.uint32)), f
                assert np.array_equal(r["track_manage"], a["track_manage"]), f
                np.testing.assert_allclose(r["targets"], a["targets"], rtol=1e-4, atol=1e-4)
            da, db = ref.tracker_dump(), ctx.seq_tracker_dump(0)
            assert np.array_equal(da[:, INTS], db[:, INTS])
            ok = _pd_tracks(da)
            err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
            if err.size:
                worst = float(err.max())
                assert worst < TOL, worst
            print(f"sequence 0 against the reference: worst relative state error {worst:.3g}")
    finally:
        ctx.close()
        for t in twins:
            t.close()


# eight single-LiDAR vehicles: eight mounting heights, yaws and offsets
FLEET = [(yaw_pose(1, 0, 0.0, 0.0, 2.0), 2.0), (yaw_pose(1, 0, 1.2, 0.0, 1.73), 1.73), (yaw_pose(0, 1, 0.0, 0.5, 1.2), 1.2),
         (yaw_pose(0, -1, 0.3, -0.4, 0.8), 0.8), (yaw_pose(-1, 0, -1.0, 0.2, 1.5), 1.5), (yaw_pose(1, 0, 0.8, 0.8, 2.2), 2.2),
         (yaw_pose(0, 1, -0.6, 0.0, 1.0), 1.0), (yaw_pose(-1, 0, 0.0, -0.9, 1.8), 1.8)]


def test_heterogeneous_fleet(pkg, synth):
    """8 sequences with one sensor each, at 8 heights and poses: each equals its own one-sensor twin."""
    rigs = [[s] for s in FLEET]
    seqs = [_RigSeq(synth, k, r, seed=800) for k, r in enumerate(rigs)]
    ctx = pkg.Lmot(_params(pkg, 1))
    twins = [_Twin(pkg, _params(pkg, 1), r) for r in rigs]
    try:
        ctx.seq_open(8, ring=4)
        for k, r in enumerate(rigs):
            set_seq_rig(ctx, k, r)
        assert all(len(ctx.seq_get_sensors(k)["poses"]) == 1 for k in range(8))
        got = _run(ctx, seqs, lambda f: rigs, 15, "sync", twins)
        _same_tables(ctx, twins, "fleet")
        assert all(sum(len(g[k]["boxes"]) for g in got) > 0 for k in range(8))
    finally:
        ctx.close()
        for t in twins:
            t.close()


def test_no_table_is_todays_path(pkg, synth):
    """Tables set, ticks run with them, then cleared and every sequence reset: the ticks equal a fresh set that never had a table (and
    lmot_frame twins), bit for bit, with the context's own lmot_set_sensors table set all along."""
    seqs = [_RigSeq(synth, k, None, seed=900, n_sensors=2) for k in range(4)]
    a, b = pkg.Lmot(_params(pkg, 0)), pkg.Lmot(_params(pkg, 0))
    twins = [_Twin(pkg, _params(pkg, 0), None) for _ in range(4)]
    try:
        a.set_sensors(**_table_kw(RIG))
        a.seq_open(4, ring=4); b.seq_open(4, ring=4)
        with_tables = [RIG[:2], None, RIG_B[:1], None]
        for k, r in enumerate(with_tables):
            set_seq_rig(a, k, r)
        for f in range(3):
            a.seq([_entry(s.frames[f], r) for s, r in zip(seqs, with_tables)], [s.ts(f) for s in seqs])
        assert a.seq_frame_counts(0).shape == (2, 4)
        for k in range(4):
            set_seq_rig(a, k, None)
            a.seq_tracker_reset(k)
            assert len(a.seq_get_sensors(k)["poses"]) == 0
        for f in range(3, 11):
            entries = [s.frames[f][0] for s in seqs]
            ts = [s.ts(f) for s in seqs]
            v = [s.ego(f)[0] for s in seqs]
            yaw = [s.ego(f)[1] for s in seqs]
            ga, gb = a.seq(entries, ts, v, yaw), b.seq(entries, ts, v, yaw)
            for k in range(4):
                w = twins[k].step(seqs[k].frames[f], ts[k], v[k], yaw[k])
                fa, fb = a.seq_frame_counts(k), b.seq_frame_counts(k)
                _same(ga[k], fa, w, (f, k, "cleared"))
                _same(gb[k], fb, w, (f, k, "fresh"))
                assert fa.shape == (1, 4) and tuple(fa[0]) == (ga[k]["n_elevated"], ga[k]["n_ground"], ga[k]["num_cluster"], len(ga[k]["boxes"]))
        _same_tables(a, twins, "cleared")
        _same_tables(b, twins, "fresh")
    finally:
        a.close(); b.close()
        for t in twins:
            t.close()


def test_ticks_in_flight_keep_their_tables(pkg, synth):
    """lmot_seq_dev with sequence 0's table changed between submissions (2 -> 3 sensors, then another 2-sensor table) and sequence 1 on
    a fixed one-sensor table: every tick, collected after all were submitted, equals twins whose tables changed at the same tick."""
    plan = [RIG[:2]] * 3 + [RIG[:3]] * 3 + [RIG_B[:2]] * 2
    fixed = RIG_B[1:2]
    seqs = [_RigSeq(synth, 0, RIG, seed=700), _RigSeq(synth, 1, fixed, seed=700)]
    ctx = pkg.Lmot(_params(pkg, 1))
    twins = [_Twin(pkg, _params(pkg, 1), plan[0]), _Twin(pkg, _params(pkg, 1), fixed)]
    try:
        ctx.seq_open(2, ring=len(plan))
        set_seq_rig(ctx, 1, fixed)

        def before(f):
            set_seq_rig(ctx, 0, plan[f])
            twins[0].set(plan[f])

        _run(ctx, seqs, lambda f: [plan[f], fixed], len(plan), "dev", twins, before)
        _same_tables(ctx, twins, "in flight")
    finally:
        ctx.close()
        for t in twins:
            t.close()


def test_seq_sensor_table_validation(pkg, synth):
    import torch
    ctx = pkg.Lmot(_params(pkg, 0))
    try:
        good = _table_kw(RIG)
        for call in (lambda: ctx.seq_set_sensors(0, **good), lambda: ctx.seq_get_sensors(0), lambda: ctx.seq_frame_counts(0)):
            with pytest.raises(pkg.LmotError) as e:
                call()                                                  # no open set
            assert e.value.status == pkg.ERR_INVALID
        ctx.seq_open(3, ring=2)
        assert ctx.seq_frame_counts(0).shape == (0, 4)                  # nothing collected yet
        set_seq_rig(ctx, 0, RIG)
        set_seq_rig(ctx, 2, RIG_B[:2])

        def tables():
            return [ctx.seq_get_sensors(k) for k in range(3)]

        before = tables()

        def rejected(fn):
            with pytest.raises(pkg.LmotError) as e:
                fn()
            assert e.value.status == pkg.ERR_INVALID
            after = tables()
            assert all(all(np.array_equal(x[key], y[key]) for key in x) for x, y in zip(before, after))

        poses = [p for p, _ in RIG]
        rejected(lambda: ctx.seq_set_sensors(3, poses))                 # k out of range
        rejected(lambda: ctx.seq_set_sensors(-1, poses))
        rejected(lambda: ctx.seq_get_sensors(3))
        rejected(lambda: ctx.seq_frame_counts(-1))
        rejected(lambda: ctx.seq_set_sensors(1, poses[:3]))             # 4 + 3 + 2 = 9 frames per tick
        rejected(lambda: ctx.seq_set_sensors(2, poses))                 # 4 + 1 + 4 = 9
        rejected(lambda: ctx.seq_set_sensors(0, [poses[0]] * 9))        # more than LMOT_MAX_BATCH in one table
        for bad in (np.nan, np.inf):
            p = [q.copy() for q in poses]; p[1][0, 3] = bad
            rejected(lambda: ctx.seq_set_sensors(0, p))                 # non-finite translation
            p = [q.copy() for q in poses]; p[2][1, 1] = bad
            rejected(lambda: ctx.seq_set_sensors(0, p))                 # non-finite rotation
            rejected(lambda: ctx.seq_set_sensors(1, poses[:1], h_sensor=bad))    # non-finite threshold
        p = [q.copy() for q in poses]; p[3][:, :3] *= f32(1.0001)
        rejected(lambda: ctx.seq_set_sensors(0, p))                     # scaled: not orthonormal
        p = [q.copy() for q in poses]; p[0][0, 1] = f32(1e-4)
        rejected(lambda: ctx.seq_set_sensors(0, p))                     # sheared
        assert ctx.lib.lmot_seq_set_sensors(ctx.h, 1, None, 2) == pkg.ERR_INVALID      # null table with n > 0
        assert tables()[1]["poses"].shape == (0, 3, 4)
        # a table that fits exactly: 4 + 2 + 2 = 8 frames
        ctx.seq_set_sensors(1, poses[:2])
        assert [len(t["poses"]) for t in tables()] == [4, 2, 2]
        got = tables()[0]
        assert np.array_equal(got["poses"], np.stack(poses)) and np.array_equal(got["h_sensor"], f32([h for _, h in RIG]))
        # a tick with fewer frames than its tables call for is refused (n_seq counts sequences, the frames follow the tables)
        fr = [np.zeros((16, 4), f32)] * 8
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq([fr[:4], fr[:2]], [1e6] * 2)                        # 2 entries for a set of 3
        assert e.value.status == pkg.ERR_INVALID
        d = torch.zeros((16, 4), device="cuda")
        ptrs = (C.c_void_p * 8)(*([d.data_ptr()] * 7 + [None]))
        ns = (C.c_int * 8)(*([16] * 8))
        dd = (C.c_double * 3)(1e6, 1e6, 1e6)
        assert ctx.lib.lmot_seq_dev(ctx.h, ptrs, ns, 3, dd, dd, dd) == pkg.ERR_INVALID  # the 8th frame (sequence 2's last) is null
        # timing mode is still refused
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq([fr[:4], fr[:2], fr[:2]], [1e6] * 3)
        assert e.value.status == pkg.ERR_STATE
        ctx.enable_timing(False)
        # reopening clears every table; n = 0 clears one
        ctx.seq_open(3, ring=2)
        assert [len(t["poses"]) for t in tables()] == [0, 0, 0]
        set_seq_rig(ctx, 1, RIG)
        ctx.seq_set_sensors(1, None)
        assert [len(t["poses"]) for t in tables()] == [0, 0, 0]
        ctx.seq_open(0, 0)
        with pytest.raises(pkg.LmotError):
            ctx.seq_get_sensors(0)
    finally:
        ctx.close()


def test_capacity_of_one_sequence(pkg, synth):
    """max_boxes below what sequence 0's four frames find together: its status and outputs equal its twin's (LMOT_ERR_CAPACITY, list
    cut at max_boxes); the other sequences of each tick equal their twins."""
    rigs = [RIG, None, RIG_B[1:2]]
    seqs = [_RigSeq(synth, k, r, seed=600, n_objects=30) for k, r in enumerate(rigs)]
    mb = 32
    ctx = pkg.Lmot(_params(pkg, 0, max_boxes=mb))
    twins = [_Twin(pkg, _params(pkg, 0, max_boxes=mb), r) for r in rigs]
    try:
        ctx.seq_open(3, ring=2)
        for k, r in enumerate(rigs):
            set_seq_rig(ctx, k, r)
        over = 0
        for f in range(8):
            entries = [_entry(s.frames[f], r) for s, r in zip(seqs, rigs)]
            ts = [s.ts(f) for s in seqs]
            v = [s.ego(f)[0] for s in seqs]
            yaw = [s.ego(f)[1] for s in seqs]
            want = [twins[k].step(seqs[k].frames[f], ts[k], v[k], yaw[k]) for k in range(3)]
            st, got = _seq_raw(ctx, entries, ts, v, yaw)
            errs = [w[0] for w in want if w[0] < 0]
            warns = [w[0] for w in want if w[0] > 0]
            assert st == (errs[0] if errs else (warns[0] if warns else 0)), (f, st, [w[0] for w in want])
            for k in range(3):
                _same(got[k], ctx.seq_frame_counts(k), want[k], (f, k))
            if sum(c[3] for c in want[0][2]) > mb:
                over += 1
                assert want[0][0] == pkg.ERR_CAPACITY and len(got[0]["boxes"]) == mb
        assert over > 0
        _same_tables(ctx, twins, "capacity")
    finally:
        ctx.close()
        for t in twins:
            t.close()
