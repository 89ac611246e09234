"""Independent sequences (lmot_seq_*): one frame of each of S sequences per tick, S track tables, one tracker chain per tick.

Contract (include/lmot.h): sequence k of a tick gives bit for bit what a separate context with the same lmot_params gives when it
receives sequence k's frames through lmot_frame -- counts, boxes, targets, vandyaw, trackManage, static / visible flags, vis_bb and
the track-table dump.  Every test below compares against such twin contexts; sequence 0 is also anchored to the reference pipeline.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_TICKS = 30
FIELDS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb", "boxes")


def _params(pkg, global_frame=0, max_tracks=512):
    p = pkg.default_params()
    p.max_points = 1 << 16
    p.max_tracks = max_tracks
    p.pipeline_depth = 2
    p.result_ring = 4
    p.global_frame = global_frame
    return p


class _Seq:
    """Sequence k: its own synth scene, start stamp, frame interval, ego speed and yaw rate."""

    def __init__(self, synth, k, n_ticks=N_TICKS):
        cfg = synth.SceneConfig(seed=101 + 7 * k, n_objects=18 + 3 * k, rings=32, azimuths=900)
        self.frames = [p for _, p in synth.frames(cfg, n_ticks)]
        self.t0 = 1.0e6 * (1 + k) + 1234.5 * k
        self.dt = 100000.0 + 5000.0 * k
        self.v = 1.5 * k
        self.rate = 0.02 * (k - 3)

    def ts(self, f):
        return self.t0 + f * self.dt

    def ego(self, f):
        return self.v + 0.1 * f, 0.3 * (self.rate != 0) + self.rate * f


_CACHE = {}


def _seqs(synth, S):
    for k in range(S):
        if k not in _CACHE:
            _CACHE[k] = _Seq(synth, k)
    return [_CACHE[k] for k in range(S)]


def _tick_args(seqs, f, frames=None):
    frames = frames if frames is not None else [s.frames[f] for s in seqs]
    ts = [s.ts(f) for s in seqs]
    v = [s.ego(f)[0] for s in seqs]
    yaw = [s.ego(f)[1] for s in seqs]
    return frames, ts, v, yaw


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


def _same(got, want, what):
    assert (got["n_elevated"], got["n_ground"], got["num_cluster"]) == (want["n_elevated"], want["n_ground"], want["num_cluster"]), what
    for key in FIELDS:
        assert got[key].shape == want[key].shape and np.array_equal(_bits(got[key]), _bits(want[key])), (what, key)


def _same_dump(a, b, what):
    assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (what, "dump")


@pytest.mark.parametrize("S,global_frame,mode", [(8, 0, "sync"), (8, 1, "dev"), (3, 1, "sync"), (3, 0, "dev")])
def test_sequences_equal_separate_contexts(pkg, synth, ref_intended, S, global_frame, mode):
    """30 ticks through lmot_seq (tick at a time) or pipelined lmot_seq_dev (all submitted, collected afterwards): every output and
    every dump row of every sequence equals its twin context fed through lmot_frame.  Sequence 0 (no ego motion, global_frame 0)
    also equals the reference chain, with the bars of test_full_pipeline_frame_matches_chained_reference."""
    import torch
    seqs = _seqs(synth, S)
    prm = _params(pkg, global_frame)
    ctx = pkg.Lmot(prm)
    twins = [pkg.Lmot(_params(pkg, global_frame)) for _ in range(S)]
    anchor = global_frame == 0 and mode == "sync"
    try:
        ctx.seq_open(S, ring=N_TICKS if mode == "dev" else 4)
        if anchor:
            ref_intended.tracker_reset()
        want = []
        for f in range(N_TICKS):
            frames, ts, v, yaw = _tick_args(seqs, f)
            if anchor:
                v[0] = yaw[0] = 0.0
            want.append([twins[k].frame(frames[k], ts[k], v[k], yaw[k]) for k in range(S)])
            if mode == "sync":
                got = ctx.seq(frames, ts, v, yaw)
                for k in range(S):
                    _same(got[k], want[f][k], (f, k))
                if anchor:
                    e, g = ref_intended.ground_remove(frames[0])
                    grid, nc = ref_intended.component_clustering(e)
                    boxes, _ = ref_intended.box_fitting(e, grid, nc)
                    a = ref_intended.tracker_step(boxes, ts[0])
                    r = got[0]
                    assert (r["n_elevated"], r["n_ground"], r["num_cluster"]) == (len(e), len(g), nc)
                    assert r["boxes"].shape == boxes.shape and np.array_equal(r["boxes"].view(np.uint32), boxes.view(np.uint32))
                    assert np.array_equal(r["track_manage"], a["track_manage"]), f
                    np.testing.assert_allclose(r["targets"], a["targets"], rtol=1e-4, atol=1e-4)
            else:
                if f == 0:
                    stream = torch.cuda.Stream()
                    ctx.set_stream(stream.cuda_stream)
                    dev = []
                with torch.cuda.stream(stream):
                    d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in frames]
                    dev.append(d)
                    ctx.seq_dev([(t.data_ptr(), len(p)) for t, p in zip(d, frames)], ts, v, yaw)
        if mode == "dev":
            for f in range(N_TICKS):
                got = ctx.seq_collect()
                for k in range(S):
                    _same(got[k], want[f][k], (f, k))
            ctx.set_stream(None)
        for k in range(S):
            _same_dump(ctx.seq_tracker_dump(k), twins[k].tracker_dump(), k)
            assert np.array_equal(ctx.seq_tracker_get_ego(k), twins[k].tracker_get_ego()), k
        assert ctx.tracker_num_tracks() == 0          # the context's own table is untouched
    finally:
        ctx.close()
        for t in twins:
            t.close()


def _crowd(f, seed=1):
    """432 pillars on a 2.2 m lattice over a flat ground grid: 432 boxes per frame, > 256 active tracks from the third tick on."""
    rng = np.random.default_rng(seed * 100 + f)
    g = np.arange(-24.0, 24.0, 0.3)
    gx, gy = np.meshgrid(g, g, indexing="ij")
    ground = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, -1.73), np.full(gx.size, 0.2)], 1)
    c = np.arange(-22.0, 22.01, 2.2)
    cx, cy = np.meshgrid(c, c, indexing="ij")
    cen = np.stack([cx.ravel(), cy.ravel()], 1)
    cen = cen[np.hypot(cen[:, 0], cen[:, 1]) > 4.0] + 0.05 * f
    u = rng.uniform(size=(len(cen), 80, 3))
    obj = np.concatenate([cen[:, None, :] + (u[..., :2] - 0.5) * 0.6, (-1.45 + 1.3 * u[..., 2:])], -1).reshape(-1, 3)
    obj = np.concatenate([obj, np.full((len(obj), 1), 0.8)], 1)
    return np.concatenate([ground, obj]).astype(np.float32)


@pytest.mark.parametrize("tc_wide", [None, "0", "1"])
def test_mixed_regimes_in_one_launch_and_reset(pkg, synth, monkeypatch, tc_wide):
    """One tick in which sequence 0 has > 256 active tracks (TC's general path at 256 threads, its wide fast path at 512), sequence 1
    an empty frame and sequence 2 its compat first frame after lmot_seq_tracker_reset(2), and sequence 3 runs normally: each equals
    its twin; the reset sequence equals a fresh context, the others their undisturbed twins."""
    if tc_wide is not None:
        monkeypatch.setenv("LMOT_TC_WIDE", tc_wide)
    seqs = _seqs(synth, 4)
    ctx = pkg.Lmot(_params(pkg, 0, max_tracks=2048))
    twins = [pkg.Lmot(_params(pkg, 0, max_tracks=2048)) for _ in range(4)]
    try:
        ctx.seq_open(4, ring=2)
        n_act_seen = 0
        for f in range(8):
            frames, ts, v, yaw = _tick_args(seqs, f)
            frames[0] = _crowd(f)
            if f == 4:
                frames[1] = frames[1][:0]
                ctx.seq_tracker_reset(2)
                twins[2].tracker_reset()
                assert ctx.seq_tracker_get_ego(2)[0] == 0.0
            want = [twins[k].frame(frames[k], ts[k], v[k], yaw[k]) for k in range(4)]
            got = ctx.seq(frames, ts, v, yaw)
            for k in range(4):
                _same(got[k], want[k], (f, k))
            n_act_seen = max(n_act_seen, int(np.sum((got[0]["track_manage"] != 0) | (got[0]["is_vis"] != 0))))
            if f == 4:
                assert len(got[1]["boxes"]) == 0 and len(got[2]["track_manage"]) <= 1
        assert n_act_seen > 256, n_act_seen
        for k in range(4):
            _same_dump(ctx.seq_tracker_dump(k), twins[k].tracker_dump(), k)
    finally:
        ctx.close()
        for t in twins:
            t.close()


def test_sequences_are_isolated(pkg, synth):
    """A different frame for sequence 2 in one tick leaves the outputs and dumps of every other sequence bit-identical."""
    seqs = _seqs(synth, 4)
    a, b = pkg.Lmot(_params(pkg, 1)), pkg.Lmot(_params(pkg, 1))
    try:
        a.seq_open(4, 2); b.seq_open(4, 2)
        changed = False
        for f in range(8):
            frames, ts, v, yaw = _tick_args(seqs, f)
            ra = a.seq(frames, ts, v, yaw)
            if f == 3:
                frames = list(frames)
                frames[2] = seqs[0].frames[f]
            rb = b.seq(frames, ts, v, yaw)
            for k in (0, 1, 3):
                _same(ra[k], rb[k], (f, k))
            changed |= not np.array_equal(ra[2]["boxes"], rb[2]["boxes"])
        assert changed
        for k in (0, 1, 3):
            _same_dump(a.seq_tracker_dump(k), b.seq_tracker_dump(k), k)
    finally:
        a.close(); b.close()


def test_interleaved_with_frame_and_batch_calls(pkg, synth):
    """Sequence ticks mixed with lmot_frame and lmot_batch on one context: the context's own tracker equals a twin that receives only
    the frame / batch calls, and every sequence equals its twin."""
    seqs = _seqs(synth, 3)
    own_frames = _seqs(synth, 6)[3:]
    ctx = pkg.Lmot(_params(pkg, 0))
    own = pkg.Lmot(_params(pkg, 0))
    twins = [pkg.Lmot(_params(pkg, 0)) for _ in range(3)]
    try:
        ctx.seq_open(3, 4)
        for f in range(10):
            frames, ts, v, yaw = _tick_args(seqs, f)
            want = [twins[k].frame(frames[k], ts[k], v[k], yaw[k]) for k in range(3)]
            got = ctx.seq(frames, ts, v, yaw)
            for k in range(3):
                _same(got[k], want[k], (f, k))
            ts_own = 5.0e5 + 1.0e5 * f
            if f % 2 == 0:
                r, w = ctx.frame(own_frames[0].frames[f], ts_own, 2.0, 0.01 * f), own.frame(own_frames[0].frames[f], ts_own, 2.0, 0.01 * f)
                _same(r, w, ("own frame", f))
            else:
                fr = [s.frames[f] for s in own_frames]
                r, w = ctx.batch(fr, ts_own), own.batch(fr, ts_own)
                for key in ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb", "boxes"):
                    assert np.array_equal(_bits(r[key]), _bits(w[key])), ("own batch", f, key)
        _same_dump(ctx.tracker_dump(), own.tracker_dump(), "own")
        for k in range(3):
            _same_dump(ctx.seq_tracker_dump(k), twins[k].tracker_dump(), k)
    finally:
        ctx.close(); own.close()
        for t in twins:
            t.close()


def test_ring_validation_and_reopen(pkg, synth):
    import ctypes as C
    import torch
    seqs = _seqs(synth, 3)
    prm = _params(pkg, 0)
    ctx = pkg.Lmot(prm)
    try:
        frames, ts, v, yaw = _tick_args(seqs[:2], 0)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq(frames, ts)                              # no open set
        assert e.value.status == pkg.ERR_INVALID
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_open(9, 2)
        assert e.value.status == pkg.ERR_INVALID
        ctx.seq_open(2, ring=2)
        # host submissions into a full ring are refused; collect returns them oldest first
        for f in range(2):
            fr, ts, v, yaw = _tick_args(seqs[:2], f)
            ctx.seq_submit(fr, ts, v, yaw)
        fr, ts, v, yaw = _tick_args(seqs[:2], 2)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_submit(fr, ts, v, yaw)
        assert e.value.status == pkg.ERR_STATE
        c0, c1 = ctx.seq_collect(), ctx.seq_collect()
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_collect()
        assert e.value.status == pkg.ERR_STATE
        # device submissions drop the oldest tick; fetch returns the most recent
        dev = []
        for f in range(2, 5):
            fr, ts, v, yaw = _tick_args(seqs[:2], f)
            d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in fr]
            dev.append(d)
            torch.cuda.synchronize()
            ctx.seq_dev([(t.data_ptr(), len(p)) for t, p in zip(d, fr)], ts, v, yaw)
        r3, r4 = ctx.seq_collect(), ctx.seq_collect()
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_collect()
        assert e.value.status == pkg.ERR_STATE
        twin = pkg.Lmot(_params(pkg, 0))
        try:
            want = [twin.frame(*((seqs[0].frames[f], seqs[0].ts(f)) + seqs[0].ego(f))) for f in range(6)]
            for f, r in ((0, c0), (1, c1), (3, r3), (4, r4)):
                _same(r[0], want[f], f)
            fr, ts, v, yaw = _tick_args(seqs[:2], 5)
            ctx.seq_submit(fr, ts, v, yaw)
            _same(ctx.seq_fetch()[0], want[5], 5)
            with pytest.raises(pkg.LmotError):
                ctx.seq_collect()                            # fetch dropped everything older
        finally:
            twin.close()
        # validation
        fr, ts, v, yaw = _tick_args(seqs, 6)
        for call in (lambda: ctx.seq(fr, ts, v, yaw),                                   # 3 frames for a set of 2
                     lambda: ctx.seq_tracker_reset(2), lambda: ctx.seq_tracker_dump(-1), lambda: ctx.seq_tracker_get_ego(2)):
            with pytest.raises(pkg.LmotError) as e:
                call()
            assert e.value.status == pkg.ERR_INVALID
        d = torch.zeros((1024, 4), device="cuda")
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_dev([(d.data_ptr() + 4, 100), (d.data_ptr(), 100)], [1e6, 1e6])   # misaligned
        assert e.value.status == pkg.ERR_INVALID
        lib = ctx.lib
        ptrs = (C.c_void_p * 2)(None, d.data_ptr())
        ns = (C.c_int * 2)(100, 100)
        dd = (C.c_double * 2)(1e6, 1e6)
        assert lib.lmot_seq_dev(ctx.h, ptrs, ns, 2, dd, dd, dd) == pkg.ERR_INVALID                 # null frame with points
        assert lib.lmot_seq_dev(ctx.h, None, ns, 2, dd, dd, dd) == pkg.ERR_INVALID
        assert lib.lmot_seq_dev(ctx.h, ptrs, ns, 2, None, dd, dd) == pkg.ERR_INVALID
        big = np.zeros((prm.max_points + 1, 4), np.float32)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq([big, fr[1]], ts[:2], v[:2], yaw[:2])
        assert e.value.status == pkg.ERR_CAPACITY
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq(fr[:2], ts[:2], v[:2], yaw[:2])
        assert e.value.status == pkg.ERR_STATE
        ctx.enable_timing(False)
        # reopening with another count starts every sequence from scratch
        ctx.seq_open(3, 2)
        twins = [pkg.Lmot(_params(pkg, 0)) for _ in range(3)]
        try:
            for f in range(3):
                fr, ts, v, yaw = _tick_args(seqs, f)
                got = ctx.seq(fr, ts, v, yaw)
                for k in range(3):
                    _same(got[k], twins[k].frame(fr[k], ts[k], v[k], yaw[k]), (f, k))
        finally:
            for t in twins:
                t.close()
        ctx.seq_open(0, 0)
        with pytest.raises(pkg.LmotError):
            ctx.seq(fr, ts, v, yaw)
    finally:
        ctx.close()
