"""Tracking-only sequence ticks (lmot_seq_track*): each sequence's track table stepped from a caller box list, S tables in one chain.

Contract (include/lmot.h): sequence k gives bit for bit what a separate context with the same lmot_params gives -- lmot_track_step on
its list without a sensor table, lmot_set_sensors(table) + lmot_track_step_lists_dev on its lists with one -- targets, vandyaw,
trackManage, static / visible flags, vis_bb, the status and the track-table dump; its boxes are the list that was tracked, its
detection counts 0.  Every test compares against such twin contexts; the teacher-forced test compares against the reference.

Each docstring names the one-line breakage the test is meant to catch.  These breakages were reasoned out; none was injected and run.
"""
import ctypes as C

import numpy as np
import pytest

from test_sensor_rig_gpu import RIG, RIG_B, mount
from test_tracker_gpu import INTS, STATE, TOL, _boxes_sequence, _rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32
OFF = -0.63035 - np.pi / 2          # firstEgoYawOffset_, imm_ukf_jpda.cpp:70
N_TICKS = 30
TRACK_FIELDS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")


# ------------------------------------------------------------------------------------------------ box lists (numpy)
def boxes_at(centres, half_extent=(1.0, 0.5)):
    """axis-aligned boxes (B, 8, 3) around `centres` (B, 2) (as test_tracker_regimes_gpu.boxes_at)"""
    c = np.asarray(centres, np.float64).reshape(-1, 2)
    h = np.broadcast_to(np.asarray(half_extent, np.float64), c.shape)
    out = np.zeros((len(c), 8, 3), f32)
    sign = np.array([[-1.0, -1.0], [-1.0, 1.0], [1.0, 1.0], [1.0, -1.0]])
    for k in range(4):
        out[:, k, :2] = c + sign[k] * h; out[:, k, 2] = -2.0
        out[:, 4 + k, :2] = c + sign[k] * h; out[:, 4 + k, 2] = 0.0
    return out


class _ListSeq:
    """Sequence k's box lists: n_obj moving objects (a count of its own), clutter that changes every tick, an empty list on some ticks;
    its own start stamp, frame interval, ego speed and yaw rate (none for sequence 0).  n_lists > 1: one list per sensor, the objects
    split between them.  ref_boxes: a list of box arrays replacing the synthetic ones (the reference's own detections)."""

    def __init__(self, k, n_ticks=N_TICKS, n_lists=1, seed=0, ref_boxes=None, n_obj=None):
        rng = np.random.default_rng(seed + 31 * k)
        n_obj = n_obj or 5 + 3 * k
        start = rng.uniform((8.0, -30.0), (40.0, 30.0), (n_obj, 2))
        vel = rng.uniform(-1.5, 1.5, (n_obj, 2))
        self.lists = []
        for f in range(n_ticks):
            if ref_boxes is not None:
                b = ref_boxes[f]
            elif (f + 2 * k) % 9 == 4:
                b = np.zeros((0, 8, 3), f32)
            else:
                c = start + vel * 0.1 * f + rng.normal(0, 0.03, start.shape)
                junk = rng.uniform((-60.0, -60.0), (-20.0, 60.0), (int(rng.integers(0, 4)), 2))
                b = boxes_at(np.concatenate([c, junk]))
            self.lists.append([b[j::n_lists] for j in range(n_lists)] if n_lists > 1 else b)
        self.t0 = 1.0e6 * (1 + k) + 1234.5 * k
        self.dt = 100000.0 + 5000.0 * k
        self.k = k

    def ts(self, f):
        return self.t0 + f * self.dt

    def ego(self, f):
        k = self.k
        return (1.5 * k + 0.1 * f, 0.3 + 0.02 * (k - 3) * f) if k else (0.0, 0.0)


def _params(pkg, gf=0, max_boxes=None, max_tracks=2048):
    p = pkg.default_params()
    p.max_points = 1 << 16
    p.max_tracks = max_tracks
    p.pipeline_depth = 2
    p.result_ring = 4
    p.global_frame = gf
    if max_boxes is not None:
        p.max_boxes = max_boxes
    return p


def _table_kw(rig):
    ms = [mount(h) for _, h in rig]
    return dict(poses=[p for p, _ in rig], **{k: [m[k] for m in ms] for k in ms[0]})


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


class _Twin:
    """the oracle of one sequence: a context stepped with lmot_track_step (no table) or lmot_set_sensors(table) +
    lmot_track_step_lists_dev + lmot_frame_fetch (table).  step -> (status, dict with the track outputs and `boxes`)"""

    def __init__(self, pkg, prm, rig=None):
        self.pkg, self.ctx, self.rig = pkg, pkg.Lmot(prm), rig
        if rig:
            self.ctx.set_sensors(**_table_kw(rig))

    def step(self, lists, ts, v, yaw, counts=None, cap=None):
        c = self.ctx
        if not self.rig:
            b = np.ascontiguousarray(lists, f32).reshape(-1, 8, 3)
            m = len(b)
            to, bufs = c._track_out(c.params.max_tracks)
            st = c.lib.lmot_track_step(c.h, self.pkg._fp(b if m else np.zeros((1, 8, 3), f32)), m, C.c_double(ts), C.c_double(v),
                                       C.c_double(yaw), C.byref(to))
            r = c._track_result(to, bufs)
            r["boxes"] = b
            return st, r
        import torch
        lists = lists if isinstance(lists, list) else [lists]
        d_lists, d_counts, cap = _pad_lists(lists, counts, cap)
        c.set_stream(None)
        c.lib.lmot_track_step_lists_dev(c.h, C.c_void_p(d_lists.data_ptr()), C.c_void_p(d_counts.data_ptr()), len(lists), int(cap),
                                        C.c_double(ts), C.c_double(v), C.c_double(yaw))
        fo, bufs = c._frame_out(c.params.max_tracks)
        torch.cuda.synchronize()
        st = c.lib.lmot_frame_fetch(c.h, C.byref(fo))
        return st, c._frame_result(fo, bufs)

    def close(self):
        self.ctx.close()


def _pad_lists(lists, counts=None, cap=None):
    """host box lists -> (device padded lists, device int32 counts, cap) in lmot_track_step_lists_dev's layout; `counts` overrides the
    lengths written to the device (clamping tests)"""
    import torch
    cap = cap or max(1, max(len(b) for b in lists))
    pad = np.zeros((len(lists), cap, 8, 3), f32)
    for i, b in enumerate(lists):
        pad[i, : min(len(b), cap)] = b[:cap]
    n = np.array(counts if counts is not None else [len(b) for b in lists], np.int32)
    d, dn = torch.from_numpy(pad).cuda(), torch.from_numpy(n).cuda()
    torch.cuda.synchronize()                 # (the contexts run on streams of their own)
    return d, dn, cap


def _same(got, fc, want, what, lists=None):
    """got: a sequence's result dict, fc: its seq_frame_counts; want: its twin's (status, dict)"""
    _, w = want
    assert (got["n_elevated"], got["n_ground"], got["num_cluster"]) == (0, 0, 0), what
    if lists is not None:
        ls = lists if isinstance(lists, list) else [lists]
        assert [tuple(int(x) for x in row) for row in fc] == [(0, 0, 0, len(b)) for b in ls], (what, "frame counts")
    for key in TRACK_FIELDS + ("boxes",):
        assert got[key].shape == w[key].shape and np.array_equal(_bits(got[key]), _bits(w[key])), (what, key)


def _same_tables(ctx, twins, what, seqs=None):
    for k, t in enumerate(twins):
        j = k if seqs is None else seqs[k]
        a, b = ctx.seq_tracker_dump(j), t.ctx.tracker_dump()
        assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (what, k, "dump")
        assert np.array_equal(ctx.seq_tracker_get_ego(j), t.ctx.tracker_get_ego()), (what, k, "ego")


def _track_raw(ctx, lists, ts, v, yaw):
    """lmot_seq_track through the raw call: -> (status, per-sequence dicts)"""
    ptrs, ms, S, keep = ctx._seq_lists(lists)
    so, sets = ctx._seq_out(ctx.params.max_tracks)
    ptrs, ms, S, t_, v_, y_ = ctx._seq_call_args((ptrs, ms, S), ts, v, yaw)
    st = ctx.lib.lmot_seq_track(ctx.h, ptrs, ms, S, t_, v_, y_, C.byref(so))
    return st, ctx._seq_result(so, sets)


def _flat(entries):
    out = []
    for e in entries:
        out.extend(e if isinstance(e, list) else [e])
    return out


def _collect_raw(ctx):
    so, sets = ctx._seq_out(ctx.params.max_tracks)
    st = ctx.lib.lmot_seq_collect(ctx.h, C.byref(so))
    return st, ctx._seq_result(so, sets)


def _run(pkg, ctx, seqs, twins, mode, n_ticks, dumps_every_tick=False):
    """n_ticks tracking ticks through lmot_seq_track (sync), pipelined lmot_seq_track_submit or pipelined lmot_seq_track_dev (torch
    device lists on the context's stream), every tick compared with the twins.  -> per tick the sequence results"""
    import torch
    S = len(seqs)
    want, done, keep = [], [], []
    stream = None
    for f in range(n_ticks):
        entries = [s.lists[f] for s in seqs]
        ts = [s.ts(f) for s in seqs]
        v = [s.ego(f)[0] for s in seqs]
        yaw = [s.ego(f)[1] for s in seqs]
        want.append([twins[k].step(entries[k], ts[k], v[k], yaw[k]) for k in range(S)])
        if mode == "sync":
            st, got = _track_raw(ctx, entries, ts, v, yaw)
            done.append((st, got, [ctx.seq_frame_counts(k) for k in range(S)]))
            if dumps_every_tick:
                _same_tables(ctx, twins, ("tick", f))
        elif mode == "submit":
            ctx.seq_track_submit(entries, ts, v, yaw)
        else:
            if stream is None:
                stream = torch.cuda.Stream()
                ctx.set_stream(stream.cuda_stream)
            flat = _flat(entries)
            cap = max(1, max(len(b) for b in flat)) + 3         # padded: the pack kernel must stride by cap, not by length
            pad = np.zeros((len(flat), cap, 8, 3), f32)
            for i, b in enumerate(flat):
                pad[i, : len(b)] = b
            with torch.cuda.stream(stream):
                d = torch.from_numpy(pad).cuda(non_blocking=False)
                n = torch.tensor([len(b) for b in flat], dtype=torch.int32).cuda()
            keep.append((d, n))
            ctx.seq_track_dev(d.data_ptr(), n.data_ptr(), cap, ts, v, yaw)
    if mode != "sync":
        for f in range(n_ticks):
            st, got = _collect_raw(ctx)
            done.append((st, got, [ctx.seq_frame_counts(k) for k in range(S)]))
        ctx.set_stream(None)
    for f, ((st, got, fcs), w) in enumerate(zip(done, want)):
        errs = [x[0] for x in w if x[0] < 0]
        warns = [x[0] for x in w if x[0] > 0]
        assert st == (errs[0] if errs else (warns[0] if warns else 0)), (f, st)
        for k in range(S):
            _same(got[k], fcs[k], w[k], (f, k), seqs[k].lists[f])
    return [g for _, g, _ in done]


# ------------------------------------------------------------------------------------------------ 1. parity with lmot_track_step
_REF_DETECTIONS = []


def _ref_detections(ref, synth):
    """the reference's own detections of N_TICKS synth frames (computed once per session: the CPU detection is the slow part)"""
    if not _REF_DETECTIONS:
        _REF_DETECTIONS.extend(b for _, b in _boxes_sequence(ref, synth, seed=3, n_frames=N_TICKS, n_objects=48))
    return _REF_DETECTIONS


@pytest.mark.parametrize("mode", ["sync", "submit", "dev"])
@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("S", [8, 3])
def test_seq_track_equals_track_step(pkg, synth, ref_intended, S, gf, mode):
    """S sequences of 30 ticks (own stamps and ego motion, empty lists, clutter; with S = 3 sequence 0 tracks the reference's own
    detections of synth frames) equal their lmot_track_step twins after every tick, in outputs and in the table; sequence 0 (no ego
    motion) with global_frame 0 also equals the reference's tracker.  Catches: a pack CTA reading another sequence's list range or count,
    or the host staging buffer indexed by sequence instead of by list."""
    ref_boxes = _ref_detections(ref_intended, synth) if S == 3 else None
    seqs = [_ListSeq(k, seed=100, ref_boxes=ref_boxes if k == 0 else None) for k in range(S)]
    ctx = pkg.Lmot(_params(pkg, gf))
    twins = [_Twin(pkg, _params(pkg, gf)) for _ in range(S)]
    try:
        ctx.seq_open(S, ring=N_TICKS if mode != "sync" else 4)
        got = _run(pkg, ctx, seqs, twins, mode, N_TICKS, dumps_every_tick=(mode == "sync"))
        _same_tables(ctx, twins, "final")
        assert ctx.tracker_num_tracks() == 0                  # the context's own table is untouched
        assert (got[-1][0]["track_manage"] > 0).sum() >= 1
        if gf == 0:
            ref = ref_intended
            ref.tracker_reset()
            s = seqs[0]
            for f in range(N_TICKS):
                a = ref.tracker_step(s.lists[f], s.ts(f))
                assert np.array_equal(got[f][0]["track_manage"], a["track_manage"]), f
                np.testing.assert_allclose(got[f][0]["targets"], a["targets"], rtol=1e-4, atol=1e-4)
    finally:
        ctx.close()
        for t in twins:
            t.close()


# ------------------------------------------------------------------------------------------------ 2. sensor tables
LAYOUTS = {"2x4": [RIG, RIG_B], "mixed": [RIG, RIG_B[1:2], None, RIG_B[2:4]]}


@pytest.mark.parametrize("mode", ["sync", "dev"])
@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("layout", ["2x4", "mixed"])
def test_seq_track_with_sensor_tables(pkg, layout, gf, mode):
    """2 sequences x 4 sensors, or 4 + 1 + 1 (no table) + 2 lists: a sequence with a table equals a lmot_set_sensors(table) twin fed by
    lmot_track_step_lists_dev (vehicle-frame boxes, per-list counts, outputs, table), the table-less one its lmot_track_step twin.
    Catches: poses indexed by sequence instead of by list, or a table-less sequence's list being transformed."""
    rigs = LAYOUTS[layout]
    seqs = [_ListSeq(k, n_ticks=20, n_lists=len(r) if r else 1, seed=200) for k, r in enumerate(rigs)]
    ctx = pkg.Lmot(_params(pkg, gf))
    twins = [_Twin(pkg, _params(pkg, gf), r) for r in rigs]
    try:
        ctx.seq_open(len(rigs), ring=20 if mode == "dev" else 4)
        for k, r in enumerate(rigs):
            if r:
                ctx.seq_set_sensors(k, **_table_kw(r))
        got = _run(pkg, ctx, seqs, twins, mode, 20)
        _same_tables(ctx, twins, layout)
        assert sum(len(g[0]["boxes"]) for g in got) > 0 and (got[-1][0]["track_manage"] > 0).sum() >= 3
        # the table's poses moved the boxes: sequence 0's published list is not the caller's
        assert not np.array_equal(got[1][0]["boxes"], np.concatenate(seqs[0].lists[1]))
    finally:
        ctx.close()
        for t in twins:
            t.close()


# ------------------------------------------------------------------------------------------------ 3. detection and tracking ticks mixed
PATTERN = "DTTDdTtDDTdtTTDt"     # D: lmot_seq, d: lmot_seq_dev (detection); T: host lists, t: device lists (tracking)


def _frame_twin(pkg, twin, pts, ts, v, yaw):
    c = twin.ctx
    p, n, s = pkg._pts(pts)
    fo, bufs = c._frame_out(c.params.max_tracks)
    st = c.lib.lmot_frame(c.h, pkg._fp(p), n, s, C.c_double(ts), C.c_double(v), C.c_double(yaw), C.byref(fo))
    return st, c._frame_result(fo, bufs)


@pytest.mark.parametrize("mode", ["sync", "pipelined"])
def test_track_and_detect_ticks_interleave(pkg, synth, mode):
    """One set of 3 sequences alternates detection ticks (host and device frames) with tracking ticks (host and device lists) in an
    irregular pattern, synchronously or all in flight at once (both kinds in the ring and on both banks); every tick equals twins that
    alternate lmot_frame and lmot_track_step.  Catches: a bank's staging or measurement list reused before the previous tick on that bank
    was consumed, or the two front ends disagreeing about which bank comes next."""
    import torch
    S, gf = 3, (1 if mode == "pipelined" else 0)
    n = len(PATTERN)
    gens = [synth.frames(synth.SceneConfig(seed=300 + 7 * k, n_objects=24, rings=32, azimuths=900), n) for k in range(S)]
    frames = [[next(g)[1] for _ in range(n)] for g in gens]
    seqs = [_ListSeq(k, n_ticks=n, seed=300) for k in range(S)]
    ctx = pkg.Lmot(_params(pkg, gf))
    twins = [_Twin(pkg, _params(pkg, gf)) for _ in range(S)]
    stream = torch.cuda.Stream()
    keep, want, done = [], [], []
    try:
        ctx.seq_open(S, ring=n if mode == "pipelined" else 4)
        ctx.set_stream(stream.cuda_stream)
        for f, kind in enumerate(PATTERN):
            ts = [s.ts(f) for s in seqs]
            v = [s.ego(f)[0] for s in seqs]
            yaw = [s.ego(f)[1] for s in seqs]
            if kind in "Dd":
                want.append([_frame_twin(pkg, twins[k], frames[k][f], ts[k], v[k], yaw[k]) for k in range(S)])
                if kind == "D":
                    ctx.seq_submit([frames[k][f] for k in range(S)], ts, v, yaw)
                else:
                    with torch.cuda.stream(stream):
                        d = [torch.from_numpy(np.ascontiguousarray(frames[k][f])).cuda() for k in range(S)]
                    keep.append(d)
                    ctx.seq_dev([(t.data_ptr(), len(t)) for t in d], ts, v, yaw)
            else:
                lists = [s.lists[f] for s in seqs]
                want.append([twins[k].step(lists[k], ts[k], v[k], yaw[k]) for k in range(S)])
                if kind == "T":
                    ctx.seq_track_submit(lists, ts, v, yaw)
                    keep.append(ctx._keep)
                else:
                    cap = max(1, max(len(b) for b in lists))
                    pad = np.zeros((S, cap, 8, 3), f32)
                    for i, b in enumerate(lists):
                        pad[i, : len(b)] = b
                    with torch.cuda.stream(stream):
                        dl = torch.from_numpy(pad).cuda()
                        dn = torch.tensor([len(b) for b in lists], dtype=torch.int32).cuda()
                    keep.append((dl, dn))
                    ctx.seq_track_dev(dl.data_ptr(), dn.data_ptr(), cap, ts, v, yaw)
            if mode == "sync":
                done.append(_collect_raw(ctx) + ([ctx.seq_frame_counts(k) for k in range(S)],))
        if mode == "pipelined":
            for f in range(n):
                done.append(_collect_raw(ctx) + ([ctx.seq_frame_counts(k) for k in range(S)],))
        ctx.set_stream(None)
        for f, ((st, got, fcs), w) in enumerate(zip(done, want)):
            assert st == next((x[0] for x in w if x[0] != 0), 0), (f, st)
            for k in range(S):
                if PATTERN[f] in "Dd":
                    _, wk = w[k]
                    assert (got[k]["n_elevated"], got[k]["n_ground"], got[k]["num_cluster"]) == \
                        (wk["n_elevated"], wk["n_ground"], wk["num_cluster"]), (f, k)
                    for key in TRACK_FIELDS + ("boxes",):
                        assert np.array_equal(_bits(got[k][key]), _bits(wk[key])), (f, k, key)
                else:
                    _same(got[k], fcs[k], w[k], (f, k), seqs[k].lists[f])
        _same_tables(ctx, twins, mode)
        assert all(sum(len(d[1][k]["boxes"]) for d, kind in zip(done, PATTERN) if kind in "Dd") > 0 for k in range(S))
    finally:
        ctx.set_stream(None)
        ctx.close()
        for t in twins:
            t.close()


# ------------------------------------------------------------------------------------------------ 4. teacher-forced, mixed regimes
def _mature(ref, sites, n_frames, ts0, rng, noise=0.02):
    """the reference's table after observing every site for n_frames frames from scratch -> (state, last stamp)"""
    ref.tracker_reset()
    ts = ts0
    for _ in range(n_frames):
        ts += 1e5
        ref.tracker_step(boxes_at(sites + rng.normal(0, noise, sites.shape)), ts)
    return ref.tracker_dump(), ts


def test_seq_teacher_forced(pkg, synth, ref_intended):
    """Six sequences loaded with six different reference states (lmot_seq_tracker_load, then lmot_seq_tracker_set_ego where the ego
    moves), then ONE tracking tick that mixes regimes: more than 512 active tracks (spawn_output's general path), a track gating more than
    32 boxes, an empty list, a compat first frame after lmot_seq_tracker_reset.  Each sequence equals the reference stepped from its own
    state: identical integers, UKF state within 1e-4 relative.  Catches: the load helper writing the context's own table, or leaving
    act_valid set (the side arrays of the previous table)."""
    ref = ref_intended
    rng = np.random.default_rng(7)
    seq_a = _boxes_sequence(ref, synth, seed=11, n_frames=9, n_objects=60)
    seq_b = _boxes_sequence(ref, synth, seed=12, n_frames=9, n_objects=60)
    cases = []          # (state, init, prev_ts, ego load args, boxes, ts, v, yaw)

    def from_run(seq, n, v=0.0, yaw=0.0):
        ref.tracker_reset()
        for ts, b in seq[:n]:
            ref.tracker_step(b, ts)
        return ref.tracker_dump(), seq[n - 1][0]

    st, pts = from_run(seq_a, 8)
    cases.append((st, 1, pts, seq_a[8][1], seq_a[8][0], 0.0, 0.0))                       # 0: synth detections
    st, pts = from_run(seq_b, 7)
    cases.append((st, 1, pts, seq_b[7][1], seq_b[7][0], 3.0, 0.05))                      # 1: moving ego
    lat = np.stack(np.meshgrid(np.arange(32) * 8.0 - 124.0, np.arange(32) * 8.0 - 124.0, indexing="ij"), -1).reshape(-1, 2)
    st, pts = _mature(ref, lat, 8, 0.0, rng)
    assert (st[:, 0] > 0).sum() > 512
    sel = np.sort(rng.choice(len(lat), 256, replace=False))
    cases.append((st, 1, pts, boxes_at(lat[sel] + rng.normal(0, 0.15, (256, 2))), pts + 1e5, 0.0, 0.0))   # 2: > 512 active tracks
    sites = np.array([[20.0, 5.0], [35.0, -12.0], [50.0, 20.0]])
    st, pts = _mature(ref, sites, 6, 5e6, rng)
    r = 0.08 * np.sqrt(rng.random(40)); a = rng.random(40) * 2 * np.pi
    crowd = sites[0] + np.stack([r * np.cos(a), r * np.sin(a)], 1)
    cases.append((st, 1, pts, boxes_at(np.concatenate([crowd, sites[1:]])), pts + 1e5, 1.0, 0.02))       # 3: 40 boxes in one gate
    st, pts = from_run(seq_a, 5)
    cases.append((st, 1, pts, np.zeros((0, 8, 3), f32), seq_a[5][0], 0.0, 0.0))          # 4: empty list
    cases.append((None, 0, 0.0, seq_b[0][1], seq_b[0][0], 0.0, 0.0))                     # 5: first frame after a reset
    S = len(cases)
    want = []
    for state, init, pts, boxes, ts, v, yaw in cases:
        if state is None:
            ref.tracker_reset()
        else:
            ref.tracker_load(state, init, pts, 0.0, OFF, OFF, -np.pi / 2)
        want.append((ref.tracker_step(boxes, ts, v, yaw), ref.tracker_dump()))
    ctx = pkg.Lmot(_params(pkg, 0, max_tracks=4096))
    try:
        ctx.seq_open(S, ring=2)
        # a first tick on different data, so that every table has history the load must replace
        ctx.seq_track([seq_b[1][1]] * S, [1e5] * S)
        for k, (state, init, pts, boxes, ts, v, yaw) in enumerate(cases):
            if state is None:
                ctx.seq_tracker_reset(k)
            elif v != 0.0 or yaw != 0.0:
                # loaded with the wrong ego, corrected by set_ego to what the reference's load left
                ctx.seq_tracker_load(k, state, init, pts + 5.0, 9.0, 0.7, 0.1, 0.2)
                ctx.seq_tracker_set_ego(k, [1.0, pts, 0.0, OFF, OFF, 0.0, 0.0, -np.pi / 2])
            else:
                ctx.seq_tracker_load(k, state, init, pts, 0.0, OFF, OFF, -np.pi / 2)
        own_before = ctx.tracker_num_tracks()
        got = ctx.seq_track([c[3] for c in cases], [c[4] for c in cases], [c[5] for c in cases], [c[6] for c in cases])
        assert ctx.tracker_num_tracks() == own_before == 0
        for k, ((a, da), b) in enumerate(zip(want, got)):
            for key in ("track_manage", "is_static", "is_vis"):
                assert np.array_equal(a[key], b[key]), (k, key)
            db = ctx.seq_tracker_dump(k)
            assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), k
            live = da[:, 0] > 0
            err = _rel_err(da[live][:, STATE], db[live][:, STATE])
            assert err.size == 0 or err.max() < TOL, (k, float(err.max()))
            np.testing.assert_allclose(b["targets"], a["targets"], rtol=1e-5, atol=1e-5)
        print("active tracks per sequence:", [int((ctx.seq_tracker_dump(k)[:, 0] > 0).sum()) for k in range(S)])
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 5. checkpoints move between contexts
def test_seq_checkpoint_migrates(pkg):
    """Sequence 1's dump + ego of context A, loaded with load + set_ego into sequence 2 of context B and into context C's own tracker:
    10 further ticks give bit-identical outputs, tables and ego on all three."""
    seqs = [_ListSeq(k, n_ticks=16, seed=500) for k in range(3)]
    j, k2 = 1, 2
    A, B, Cc = pkg.Lmot(_params(pkg, 1)), pkg.Lmot(_params(pkg, 1)), pkg.Lmot(_params(pkg, 1))
    try:
        A.seq_open(3, ring=4); B.seq_open(3, ring=4)
        for f in range(6):
            A.seq_track([s.lists[f] for s in seqs], [s.ts(f) for s in seqs], [s.ego(f)[0] for s in seqs], [s.ego(f)[1] for s in seqs])
        dump, ego = A.seq_tracker_dump(j), A.seq_tracker_get_ego(j)
        assert len(dump) > 3 and abs(ego[7] + np.pi / 2) > 1e-3          # a real table, a turned ego
        B.seq_tracker_load(k2, dump, 1, seqs[j].ts(5)); B.seq_tracker_set_ego(k2, ego)
        Cc.tracker_load(dump, 1, seqs[j].ts(5)); Cc.tracker_set_ego(ego)
        s = seqs[j]
        for f in range(6, 16):
            ts, (v, yaw) = s.ts(f), s.ego(f)
            ga = A.seq_track([q.lists[f] for q in seqs], [q.ts(f) for q in seqs], [q.ego(f)[0] for q in seqs], [q.ego(f)[1] for q in seqs])[j]
            lb = [np.zeros((0, 8, 3), f32)] * 3
            lb[k2] = s.lists[f]
            tb = [1e5 * (f + 1)] * 3
            tb[k2] = ts
            vb, yb = [0.0] * 3, [0.0] * 3
            vb[k2], yb[k2] = v, yaw
            gb = B.seq_track(lb, tb, vb, yb)[k2]
            gc = Cc.track_step(s.lists[f], ts, v, yaw)
            for key in TRACK_FIELDS:
                assert np.array_equal(_bits(ga[key]), _bits(gb[key])) and np.array_equal(_bits(ga[key]), _bits(gc[key])), (f, key)
        da, db, dc = A.seq_tracker_dump(j), B.seq_tracker_dump(k2), Cc.tracker_dump()
        assert np.array_equal(_bits(da), _bits(db)) and np.array_equal(_bits(da), _bits(dc))
        ea = A.seq_tracker_get_ego(j)
        assert np.array_equal(ea, B.seq_tracker_get_ego(k2)) and np.array_equal(ea, Cc.tracker_get_ego())
    finally:
        A.close(); B.close(); Cc.close()


# ------------------------------------------------------------------------------------------------ 6. validation and capacity
def test_seq_track_validation_and_capacity(pkg):
    """Every rejection of lmot_seq_track_submit / _dev leaves the ring as it was; a sequence whose lists exceed max_boxes reports what its
    lists_dev twin reports while its neighbours are unaffected; device counts are clamped like the twin's; a full ring refuses host lists
    and drops the oldest tick for device lists; timing mode is refused; load / set_ego check k and n."""
    import torch
    mb = 32
    lib = None
    ctx = pkg.Lmot(_params(pkg, 0, max_boxes=mb, max_tracks=64))
    try:
        lib, h = ctx.lib, ctx.h
        one = boxes_at([[10.0, 0.0]])
        dd = (C.c_double * 3)(1e6, 1e6, 1e6)

        def host(lists):
            ptrs, ms, S, keep = ctx._seq_lists(lists)
            return ptrs, ms, S, keep

        ptrs, ms, S, keep = host([one, one, one])
        assert lib.lmot_seq_track_submit(h, ptrs, ms, 3, dd, dd, dd) == pkg.ERR_INVALID          # no open set
        ctx.seq_open(3, ring=2)
        assert lib.lmot_seq_track_submit(h, ptrs, ms, 3, dd, dd, dd) == 0                        # one tick in the ring
        d = torch.zeros((3, 4, 8, 3), device="cuda")
        dn = torch.tensor([1, 1, 1], dtype=torch.int32, device="cuda")
        rejections = [
            (lambda: lib.lmot_seq_track_submit(h, ptrs, ms, 2, dd, dd, dd), pkg.ERR_INVALID),     # n_seq != the set's
            (lambda: lib.lmot_seq_track_submit(h, None, ms, 3, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, ptrs, None, 3, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, ptrs, ms, 3, None, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, ptrs, ms, 3, dd, None, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, ptrs, ms, 3, dd, dd, None), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, (C.c_void_p * 3)(ptrs[0], None, ptrs[2]), ms, 3, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, ptrs, (C.c_int * 3)(1, -1, 1), 3, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_submit(h, ptrs, (C.c_int * 3)(1, mb + 1, 1), 3, dd, dd, dd), pkg.ERR_CAPACITY),
            (lambda: lib.lmot_seq_track_dev(h, None, C.c_void_p(dn.data_ptr()), 3, 4, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_dev(h, C.c_void_p(d.data_ptr()), None, 3, 4, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_dev(h, C.c_void_p(d.data_ptr()), C.c_void_p(dn.data_ptr()), 3, 0, dd, dd, dd), pkg.ERR_INVALID),
            (lambda: lib.lmot_seq_track_dev(h, C.c_void_p(d.data_ptr()), C.c_void_p(dn.data_ptr()), 4, 4, dd, dd, dd), pkg.ERR_INVALID),
        ]
        big = boxes_at(np.stack([np.arange(mb + 1) * 3.0 + 10.0, np.zeros(mb + 1)], 1))
        bp, bm, _, bkeep = host([one, big, one])
        rejections.append((lambda: lib.lmot_seq_track_submit(h, bp, bm, 3, dd, dd, dd), pkg.ERR_CAPACITY))   # a real list above max_boxes
        for i, (call, status) in enumerate(rejections):
            assert call() == status, i
        ctx.enable_timing(True)
        assert lib.lmot_seq_track_submit(h, ptrs, ms, 3, dd, dd, dd) == pkg.ERR_STATE
        assert lib.lmot_seq_track_dev(h, C.c_void_p(d.data_ptr()), C.c_void_p(dn.data_ptr()), 3, 4, dd, dd, dd) == pkg.ERR_STATE
        ctx.enable_timing(False)
        st, got = _collect_raw(ctx)                                                              # exactly the one tick
        assert st == 0 and [len(g["boxes"]) for g in got] == [1, 1, 1]
        assert _collect_raw(ctx)[0] == pkg.ERR_STATE

        # a full ring: host lists are refused, device lists drop the oldest tick
        lens = [[1, 2, 3], [2, 3, 4], [3, 4, 1]]
        lists = [[boxes_at(np.stack([np.arange(n) * 4.0 + 10.0, np.full(n, 2.0 * k)], 1)) for k, n in enumerate(l)] for l in lens]
        ctx.seq_track_submit(lists[0], [2e6] * 3)
        ctx.seq_track_submit(lists[1], [2.1e6] * 3)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_track_submit(lists[2], [2.2e6] * 3)
        assert e.value.status == pkg.ERR_STATE
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        with torch.cuda.stream(stream):
            pad = np.zeros((3, 4, 8, 3), f32)
            for i, b in enumerate(lists[2]):
                pad[i, : len(b)] = b
            d2 = torch.from_numpy(pad).cuda()
            n2 = torch.tensor(lens[2], dtype=torch.int32).cuda()
        ctx.seq_track_dev(d2.data_ptr(), n2.data_ptr(), 4, [2.2e6] * 3)
        ctx.set_stream(None)
        assert [len(g["boxes"]) for g in ctx.seq_collect()] == lens[1]                           # the oldest was dropped
        assert [len(g["boxes"]) for g in ctx.seq_collect()] == lens[2]

        # load / set_ego
        dump = np.zeros((1, pkg.TRACK_DUMP_DOUBLES))
        for k in (-1, 3):
            assert lib.lmot_seq_tracker_load(h, k, dump.ctypes.data_as(C.POINTER(C.c_double)), 1, 1, C.c_double(0), C.c_double(0),
                                             C.c_double(0), C.c_double(0), C.c_double(0)) == pkg.ERR_INVALID
            assert lib.lmot_seq_tracker_set_ego(h, k, np.zeros(8).ctypes.data_as(C.POINTER(C.c_double))) == pkg.ERR_INVALID
        many = np.zeros((65, pkg.TRACK_DUMP_DOUBLES))
        assert lib.lmot_seq_tracker_load(h, 0, many.ctypes.data_as(C.POINTER(C.c_double)), 65, 1, C.c_double(0), C.c_double(0),
                                         C.c_double(0), C.c_double(0), C.c_double(0)) == pkg.ERR_CAPACITY
    finally:
        ctx.close()

    # capacity of one sequence and clamped device counts, against lists_dev / track_step twins
    rigs = [RIG, None, RIG_B[1:2]]
    ctx = pkg.Lmot(_params(pkg, 0, max_boxes=mb))
    twins = [_Twin(pkg, _params(pkg, 0, max_boxes=mb), r) for r in rigs]
    try:
        ctx.seq_open(3, ring=2)
        for k, r in enumerate(rigs):
            if r:
                ctx.seq_set_sensors(k, **_table_kw(r))
        seqs = [_ListSeq(k, n_ticks=6, n_lists=len(r) if r else 1, seed=600, n_obj=40 if k == 0 else 8) for k, r in enumerate(rigs)]
        over = 0
        for f in range(6):
            entries = [s.lists[f] for s in seqs]
            ts = [s.ts(f) for s in seqs]
            v = [s.ego(f)[0] for s in seqs]
            yaw = [s.ego(f)[1] for s in seqs]
            want = [t.step(e, ts[k], v[k], yaw[k]) for k, (t, e) in enumerate(zip(twins, entries))]
            st, got = _track_raw(ctx, entries, ts, v, yaw)
            errs = [w[0] for w in want if w[0] < 0]
            assert st == (errs[0] if errs else next((w[0] for w in want if w[0] > 0), 0)), (f, st)
            for k in range(3):
                _same(got[k], ctx.seq_frame_counts(k), want[k], (f, k), entries[k])
            if sum(len(b) for b in entries[0]) > mb:
                over += 1
                assert want[0][0] == pkg.ERR_CAPACITY and len(got[0]["boxes"]) == mb
        assert over > 0
        # device counts below 0 and above cap_per_list are clamped as lmot_track_step_lists_dev clamps them
        f = 5
        entries = [s.lists[f] for s in seqs]
        flat = _flat(entries)
        cap = 6
        counts = [-3, 99, 2, 6, 0, 4][: len(flat)]
        counts = counts + [3] * (len(flat) - len(counts))
        ts = [s.ts(f) + 1e5 for s in seqs]
        clamped = [b[: max(0, min(c, cap))] for b, c in zip(flat, counts)]
        want = [twins[0].step(entries[0], ts[0], 0.0, 0.0, counts=counts[:4], cap=cap),
                twins[1].step(clamped[4], ts[1], 0.0, 0.0), twins[2].step(entries[2], ts[2], 0.0, 0.0, counts=counts[5:], cap=cap)]
        d, n, _ = _pad_lists(flat, counts, cap)
        ctx.seq_track_dev(d.data_ptr(), n.data_ptr(), cap, ts, 0.0, 0.0)
        st, got = _collect_raw(ctx)
        torch.cuda.synchronize()
        rows = [ctx.seq_frame_counts(k) for k in range(3)]
        assert [int(r[3]) for r in rows[0]] == [max(0, min(c, cap)) for c in counts[:4]]
        for k in range(3):
            _same(got[k], rows[k], want[k], ("clamp", k))
        _same_tables(ctx, twins, "capacity")
    finally:
        ctx.close()
        for t in twins:
            t.close()
