"""Track retirement and track IDs on the GPU (lmot_set_track_retirement, lmot_track_ids): the retire-capable TC against the erasing
reference (the reference's sources + ref_tracker_retire of oracle/ref_retire.cpp after every step), against twin contexts, and the default path unchanged.

Bars as in test_tracker_gpu: identical integers and flags, targets / vandyaw / vis_bb as in test_teacher_forced_steps, UKF state
within 1e-4 relative; free-running comparisons leave out filters that are not positive definite (_pd_tracks).  IDs must equal a Python
bookkeeping of the table: erase where trackManage == 0, append the next ordinals.  Each docstring names the breakage the test is meant
to catch; those breakages were reasoned out, not injected.
"""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest

from test_seq_track_gpu import _ListSeq, _params, _same, _same_tables, _Twin, _bits, _track_raw, _collect_raw, boxes_at
from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err
from test_track_retire_cpu import _contains

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OFF = -0.63035 - np.pi / 2
FLAGS = ("track_manage", "is_static", "is_vis")
OUT_KEYS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")
TUNED = dict(gamma_g=7.5, std_a=[1.5, 2.5, 3.5], std_las_x=0.2, mode_prob0=[0.4, 0.35, 0.25], p0_diag=[0.4, 0.6, 2.5, 8.0, 1.2])


@pytest.fixture(scope="module")
def ref():
    from oracle import ref, ref_retire
    if not ref.have_ref("intended") or not ref_retire.have_retire("intended"):
        pytest.skip("oracle/_ref not built")
    r = ref.RefOracle("intended")
    r.tracker_retire = ref_retire.retirer(r)
    return r


@pytest.fixture(scope="module")
def ref_tunable():
    from oracle import ref_retire
    from oracle import ref_tunable as rt
    if not rt.have_ref("tunable") or not ref_retire.have_retire("tunable"):
        pytest.skip("oracle/_ref/libref_tunable.so not built")
    r = rt.RefTunable()
    r.tracker_retire = ref_retire.retirer(r)
    yield r
    r.set_tracker_params(None)


def bench_scene(n, seed=0):
    """the tracking-only bench workload of scripts/seq_track_measure.py (clutter that spawns and dies every step), moving ego"""
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    try:
        stm = importlib.import_module("seq_track_measure")
    finally:
        sys.path.pop(0)
    lists = stm.bench_lists(seed, n)
    return [(1e6 + 1e5 * f, lists[f], 2.0 + 0.5 * np.sin(0.03 * f), 0.4 + 0.004 * f) for f in range(n)]


class _Ids:
    """the ID bookkeeping of one table: the rows retained after the previous step, then this step's spawns"""

    def __init__(self):
        self.ids, self.next = [], 0

    def step(self, track_manage, retire=True):
        n_new = len(track_manage) - len(self.ids)
        self.ids += list(range(self.next, self.next + n_new))
        self.next += n_new
        out = np.asarray(self.ids, np.int64)
        if retire:
            self.ids = [i for i, tm in zip(self.ids, track_manage) if tm != 0]
        return out


def _ctx(pkg, retire=True, max_points=None, **kw):
    p = _params(pkg, **kw)
    if max_points:
        p.max_points = max_points
    c = pkg.Lmot(p)
    c.set_track_retirement(retire)
    return c


def _vs_ref(a, b, da, db, what, teacher=False):
    """a / da: the reference's outputs / dump, b / db: this library's"""
    for k in FLAGS:
        assert np.array_equal(a[k], b[k]), (what, k)
    assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (what, "dump")
    ok = (da[:, 0] > 0) if teacher else _pd_tracks(da)
    err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
    assert err.size == 0 or err.max() < TOL, (what, float(err.max()))
    if teacher:
        np.testing.assert_allclose(b["targets"], a["targets"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(b["vandyaw"], a["vandyaw"], rtol=1e-4, atol=1e-6)
    assert a["vis_bb"].shape == b["vis_bb"].shape, what
    if teacher:
        np.testing.assert_allclose(b["vis_bb"], a["vis_bb"], rtol=1e-5, atol=1e-5)


def _same_outputs(a, b, what):
    for k in OUT_KEYS:
        assert a[k].shape == b[k].shape and np.array_equal(_bits(a[k]), _bits(b[k])), (what, k)


_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
from test_track_retire_gpu import bench_scene
scene = bench_scene(12)
names = {}
for arm in ("never", "off", "on"):
    c = pkg.Lmot()
    if arm != "never":
        c.set_track_retirement(arm == "on")
    for f, (ts, b, v, y) in enumerate(scene[:10]):
        c.track_step(b, ts, v, y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for ts, b, v, y in scene[10:]:
            c.track_step(b, ts, v, y)
        torch.cuda.synchronize()
    names[arm] = sorted({e.name for e in prof.events() if "spawn_output" in e.name or "publish" in e.name})
    c.close()
print(json.dumps(names))
"""


# ------------------------------------------------------------------------------------------------ 1. off is today's path
def test_off_runs_the_default_kernels(pkg):
    """Catches a context that never called the API, or switched retirement off, running the tuned kernels, the retire-capable TC or the
    ID publication (kernel names through torch.profiler, in a process of its own), outputs that differ from such a context, and IDs
    that are not the row indices.  A retiring context runs the sequence family's TC at S = 1 and publishes its IDs."""
    import json
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, ROOT, here], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    print(names)
    for arm in ("never", "off"):
        assert names[arm] and not any("tuned" in n or "retire" in n or "publish_ids" in n for n in names[arm]), (arm, names[arm])
    assert any("spawn_output_seq_tuned" in n for n in names["on"]) and any("publish_ids" in n for n in names["on"]), names["on"]
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_track_retirement(False)
        assert not b.get_track_retirement()
        for f, (ts, boxes, v, y) in enumerate(bench_scene(40)):
            ra, rb = a.track_step(boxes, ts, v, y), b.track_step(boxes, ts, v, y)
            _same_outputs(ra, rb, f)
            assert np.array_equal(b.track_ids(), np.arange(len(rb["track_manage"]))), f
        assert np.array_equal(_bits(a.tracker_dump()), _bits(b.tracker_dump()))
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ 2. parity with the erasing reference
def _state_err(da, db):
    ok = _pd_tracks(da)
    err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
    return float(err.max()) if err.size else 0.0


@pytest.mark.parametrize("tuned", [False, True])
def test_track_step_equals_erasing_reference(pkg, ref, ref_tunable, tuned):
    """Catches a compaction that loses, reorders or duplicates a record, position or ID; a retire phase that misses a row that died in
    this step (merge, guard, track-number machine); and IDs that drift from the bookkeeping -- 150 free-running frames of the bench
    scene with a moving ego, with the default parameters and with tuned ones (the retire kernels read the tuned source).
    Against the erasing reference: identical flags and dump integers every frame.  Against an unbounded context (the default path):
    the retained rows bit for bit, outputs and records -- so the UKF states are within the bar wherever the default path is; the
    free-running drift of this scene's long-lived filters (libm ulps accumulated over ~100 steps) is the default path's own, and the
    test prints both.  The comparison with the unbounded context ends at the first difference, which must be a frame with a ghost
    containment (a dead track's frozen position inside a visible box: the one documented deviation)."""
    oracle = ref_tunable if tuned else ref
    scene = bench_scene(150)
    if tuned:
        ref_tunable.set_tracker_params(TUNED)
    off, on = _ctx(pkg, retire=False, max_tracks=8192), _ctx(pkg)
    try:
        if tuned:
            off.set_tracker_params(**TUNED)
            on.set_tracker_params(**TUNED)
        # the unbounded reference against the default path
        oracle.tracker_reset()
        full, err_off = [], []
        for f, (ts, boxes, v, y) in enumerate(scene):
            a = oracle.tracker_step(boxes, ts, v, y)
            b = off.track_step(boxes, ts, v, y)
            for k in FLAGS:
                assert np.array_equal(a[k], b[k]), ("unbounded", f, k)
            db = off.tracker_dump()
            err_off.append(_state_err(oracle.tracker_dump(), db))
            full.append((b, db))
        # the erasing reference against retirement
        oracle.tracker_reset()
        ids = _Ids()
        err_on = []
        diverged = None
        for f, (ts, boxes, v, y) in enumerate(scene):
            a = oracle.tracker_step(boxes, ts, v, y)
            b = on.track_step(boxes, ts, v, y)
            want_ids = ids.step(a["track_manage"])
            oracle.tracker_retire()
            for k in FLAGS:
                assert np.array_equal(a[k], b[k]), (f, k)
            da, db = oracle.tracker_dump(), on.tracker_dump()
            assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (f, "dump")
            err_on.append(_state_err(da, db))
            assert np.array_equal(on.track_ids(), want_ids), f
            assert on.tracker_num_tracks() == len(ids.ids), f
            if diverged is not None:
                continue
            fb, fdb = full[f]
            same = all(np.array_equal(_bits(b[k]), _bits(fb[k][want_ids])) for k in OUT_KEYS[:-1])
            same = same and np.array_equal(_bits(b["vis_bb"]), _bits(fb["vis_bb"]))
            same = same and np.array_equal(_bits(db), _bits(fdb[np.asarray(ids.ids, np.int64)]))
            if not same:
                dead = np.nonzero(full[f - 1][0]["track_manage"] == 0)[0] if f else np.zeros(0, np.int64)
                ghost = any(np.any(_contains(fb["vis_bb"][slot, :4, :2], fdb[dead, 4], fdb[dead, 5]) & (dead != i))
                            for slot, i in enumerate(np.nonzero(fb["is_vis"])[0]))
                assert ghost, (f, "differs from the unbounded context without a ghost containment")
                diverged = f
                continue
            assert err_on[-1] <= max(TOL, err_off[f]), (f, err_on[-1], err_off[f])
        print(f"\nstate error vs the reference, max over 150 frames: default path {max(err_off):.2e} "
              f"(first frame above {TOL}: {next((f for f, e in enumerate(err_off) if e > TOL), None)}), retirement {max(err_on):.2e}; "
              f"equal to the unbounded context until frame {diverged} (a ghost containment)")
    finally:
        off.close(); on.close()
        if tuned:
            ref_tunable.set_tracker_params(None)


@pytest.mark.parametrize("gf", [0, 1])
def test_pipelined_frames_equal_sync_twin(pkg, synth, gf):
    """Catches IDs of a pipelined result that belong to another step (the pinned block is reused by later submissions; the IDs are
    copied at collect), a prev-block seed that breaks once rows move, and _fetch with dropped results -- lmot_frame_submit / _collect
    and _fetch against a twin stepped by lmot_frame, global_frame 0 and 1, 110 frames with a moving ego."""
    cfg = synth.SceneConfig(seed=5, n_objects=60)
    frames = list(synth.frames(cfg, 110))
    ego = [(1.0 + 0.02 * f, 0.2 + 0.005 * f) for f in range(len(frames))]
    a, b = _ctx(pkg, gf=gf, max_points=1 << 20), _ctx(pkg, gf=gf, max_points=1 << 20)
    try:
        want = []
        for f, (ts, pts) in enumerate(frames):
            r = a.frame(pts, ts, *ego[f])
            want.append((r, a.track_ids()))
        got = []
        f = 0
        while f < len(frames):
            k = min(3, len(frames) - f)
            for j in range(k):
                ts, pts = frames[f + j]
                b.frame_submit(pts, ts, *ego[f + j])
            if f % 2 == 0:
                for j in range(k):
                    got.append((f + j, b.frame_collect(), b.track_ids()))
            else:
                got.append((f + k - 1, b.frame_fetch(), b.track_ids()))     # the older ones are dropped
            f += k
        for i, r, ids in got:
            for key in OUT_KEYS:
                assert np.array_equal(_bits(r[key]), _bits(want[i][0][key])), (i, key)
            assert np.array_equal(ids, want[i][1]), i
        assert np.array_equal(_bits(a.tracker_dump()), _bits(b.tracker_dump()))
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ 3. a long run on a small table
def test_long_run_on_small_table(pkg, ref):
    """Catches a table that still fills (the warning, at the frame the spawn count predicts without retirement), a bound on n_tracks
    that does not hold, and drift over a long run: 1,000 frames of the bench scene on max_tracks 128 -- flags equal to the erasing
    reference every frame, outputs and retained records equal to an unbounded context bit for bit."""
    scene = bench_scene(1000, seed=3)
    big = _ctx(pkg, retire=False, max_tracks=16384)
    off = _ctx(pkg, retire=False, max_tracks=128)
    on = _ctx(pkg, retire=True, max_tracks=128)
    try:
        predicted = warned = None
        ref.tracker_reset()
        ids = _Ids()
        n_max = 0
        for f, (ts, boxes, v, y) in enumerate(scene):
            rb = big.track_step(boxes, ts, v, y)
            assert big.last_warning == 0, f
            if predicted is None and len(rb["track_manage"]) > 128:
                predicted = f
            if warned is None:
                off.track_step(boxes, ts, v, y)
                if off.last_warning == pkg.WARN_TRACK_TABLE_FULL:
                    warned = f
            a = ref.tracker_step(boxes, ts, v, y)
            b = on.track_step(boxes, ts, v, y)
            assert on.last_warning == 0, f
            want_ids = ids.step(a["track_manage"])
            ref.tracker_retire()
            n_max = max(n_max, len(b["track_manage"]))
            for k in FLAGS:
                assert np.array_equal(a[k], b[k]), (f, k)
            assert np.array_equal(on.track_ids(), want_ids), f
            for k in OUT_KEYS[:-1]:
                assert np.array_equal(_bits(b[k]), _bits(rb[k][want_ids])), (f, k, "vs unbounded")
            if f % 50 == 0 or f == len(scene) - 1:
                da, db = ref.tracker_dump(), on.tracker_dump()
                assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (f, "dump")
                assert np.array_equal(_bits(db), _bits(big.tracker_dump()[np.asarray(ids.ids, np.int64)])), (f, "records vs unbounded")
        print(f"\nmax_tracks 128: without retirement the table is full at frame {warned} (predicted {predicted}); with it at most "
              f"{n_max} rows per step, {ids.next} tracks spawned in {len(scene)} frames")
        assert predicted is not None and warned == predicted
        assert n_max <= 128 and ids.next > 1000
    finally:
        big.close(); off.close(); on.close()


# ------------------------------------------------------------------------------------------------ 4. regimes
def _lattice(n, spacing=4.0):
    side = int(np.ceil(np.sqrt(n)))
    g = np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2)[:n] * spacing
    return g + np.array([5.0, -side * spacing / 2])


_STATES = {}


def _mature_state(ref, n):
    """n mature tracks on a lattice (the reference's own table after 8 observed frames)"""
    if n not in _STATES:
        rng = np.random.default_rng(n)
        sites = _lattice(n)
        ref.tracker_reset()
        ts = 1e6
        for _ in range(8):
            ts += 1e5
            ref.tracker_step(boxes_at(sites + rng.normal(0, 0.02, sites.shape)), ts)
        _STATES[n] = (ref.tracker_dump(), ts, sites)
    return _STATES[n]


@pytest.mark.parametrize("n", [256, 257, 512, 513])
@pytest.mark.parametrize("deaths", ["first", "middle", "last", "all", "none"])
def test_regimes_teacher_forced(pkg, ref, n, deaths):
    """Catches tile-boundary mistakes of the in-place compaction (tables of 256, 257, 512 and 513 rows: TC's 256 / 512 variants and
    their general paths) with deaths at the first row, the middle, the last row, every row and no row, from a reference state with dead
    rows loaded first (TC's `full` path); then three more teacher-forced steps against the erasing reference."""
    state, ts, sites = _mature_state(ref, n)
    state = state.copy()
    kill = {"first": [0], "middle": [n // 2], "last": [n - 1], "all": list(range(n)), "none": []}[deaths]
    state[kill, 0] = 0
    rng = np.random.default_rng(7)
    lm = _ctx(pkg, max_tracks=2048)
    try:
        for step in range(4):
            ref.tracker_load(state, 1, ts, 0.0, OFF, OFF, -np.pi / 2)
            lm.tracker_load(state, 1, ts, 0.0, OFF, OFF, -np.pi / 2)
            ts += 1e5
            pick = sites[np.sort(rng.choice(len(sites), int(0.8 * len(sites)), replace=False))]
            boxes = boxes_at(pick + rng.normal(0, 0.03, pick.shape))
            a = ref.tracker_step(boxes, ts)
            b = lm.track_step(boxes, ts)
            assert np.array_equal(lm.track_ids(), np.arange(len(a["track_manage"]))), (deaths, step)   # loaded rows: 0..n-1, then spawns
            ref.tracker_retire()
            state = ref.tracker_dump()
            _vs_ref(a, b, state, lm.tracker_dump(), (n, deaths, step), teacher=True)
    finally:
        lm.close()


def test_lattice_general_path_moves_many_records(pkg, ref):
    """Catches record moves that overlap across tiles of the general path: the 1,024-track lattice with 256 boxes per step, where most
    tracks die within a few steps and hundreds of records move per step; free-running against the erasing reference with IDs."""
    rng = np.random.default_rng(11)
    sites = _lattice(1024, 8.0)
    lm = _ctx(pkg, max_tracks=4096)
    try:
        ref.tracker_reset()
        ids = _Ids()
        ts = 1e6
        for f in range(14):
            ts += 1e5
            pick = sites if f < 6 else sites[np.sort(rng.choice(len(sites), 256, replace=False))]
            boxes = boxes_at(pick + rng.normal(0, 0.03, pick.shape))
            a = ref.tracker_step(boxes, ts)
            b = lm.track_step(boxes, ts)
            want = ids.step(a["track_manage"])
            ref.tracker_retire()
            _vs_ref(a, b, ref.tracker_dump(), lm.tracker_dump(), f)
            assert np.array_equal(lm.track_ids(), want), f
        assert ids.next >= 1024 and len(ids.ids) < 1024
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ 5. sequences
def test_seq_mixed_settings_equal_twins(pkg):
    """Catches a sequence that takes another's flags, IDs or parameters in a tick that mixes retirement on / off, default / tuned
    parameters and a table whose IDs are no longer its rows; and lmot_seq_track_ids reading the wrong sequence.  S = 8 tracking-only
    ticks, sync and pipelined (_submit / _collect), global_frame 0 and 1, each sequence against a twin context with the same
    settings."""
    for gf in (0, 1):
        S, n_ticks = 8, 40
        seqs = [_ListSeq(k, n_ticks=n_ticks) for k in range(S)]
        ctx = pkg.Lmot(_params(pkg, gf=gf))
        twins = [_Twin(pkg, _params(pkg, gf=gf)) for _ in range(S)]
        try:
            ctx.seq_open(S, ring=4)
            retire = [k % 2 == 0 for k in range(S)]
            for k in range(S):
                ctx.seq_set_track_retirement(k, retire[k])
                twins[k].ctx.set_track_retirement(retire[k])
                if k % 3 == 1:
                    ctx.seq_set_tracker_params(k, **TUNED)
                    twins[k].ctx.set_tracker_params(**TUNED)
            for f in range(n_ticks):
                if f == 20:                                  # sequence 2 retired; off now, its IDs stay its own
                    ctx.seq_set_track_retirement(2, False); twins[2].ctx.set_track_retirement(False); retire[2] = False
                lists = [s.lists[f] for s in seqs]
                ts = [s.ts(f) for s in seqs]
                v = [s.ego(f)[0] for s in seqs]
                y = [s.ego(f)[1] for s in seqs]
                want = [twins[k].step(lists[k], ts[k], v[k], y[k]) for k in range(S)]
                want_ids = [twins[k].ctx.track_ids() for k in range(S)]
                if f % 2 == 0:
                    st, got = _track_raw(ctx, lists, ts, v, y)
                else:
                    ctx.seq_track_submit(lists, ts, v, y)
                    st, got = _collect_raw(ctx)
                for k in range(S):
                    _same(got[k], ctx.seq_frame_counts(k), want[k], (gf, f, k), lists[k])
                    assert np.array_equal(ctx.seq_track_ids(k), want_ids[k]), (gf, f, k)
            _same_tables(ctx, twins, ("final", gf))
            assert [ctx.seq_get_track_retirement(k) for k in range(S)] == retire
        finally:
            ctx.close()
            for t in twins:
                t.close()


# ------------------------------------------------------------------------------------------------ 6. lifecycle
def test_switching_in_flight_reset_load_reopen(pkg):
    """Catches a switch that reaches steps already in flight, IDs that go wrong when retirement is switched off after retiring, and
    reset / load / reopen that do not return the IDs to the row indices or the switch to its documented state."""
    scene = bench_scene(60, seed=5)
    a, b = _ctx(pkg, retire=False), _ctx(pkg, retire=False)       # a: the switch flipped between submissions; b: synchronous twin
    try:
        pattern = [f // 7 % 2 == 1 for f in range(len(scene))]
        for f, (ts, boxes, v, y) in enumerate(scene):
            a.set_track_retirement(pattern[f])
            b.set_track_retirement(pattern[f])
            want = b.track_step(boxes, ts, v, y)
            want_ids = b.track_ids()
            # a: submit through the list entry point without waiting, flip the switch, then fetch
            import torch
            pad = torch.from_numpy(np.ascontiguousarray(boxes.reshape(1, -1, 8, 3) if len(boxes) else np.zeros((1, 1, 8, 3), np.float32))).cuda()
            n = torch.tensor([len(boxes)], dtype=torch.int32).cuda()
            torch.cuda.synchronize()
            a.set_stream(None)
            assert a.lib.lmot_track_step_lists_dev(a.h, C.c_void_p(pad.data_ptr()), C.c_void_p(n.data_ptr()), 1, max(1, len(boxes)),
                                                   C.c_double(ts), C.c_double(v), C.c_double(y)) == 0
            a.set_track_retirement(not pattern[f])          # must not reach the step just submitted
            got = a.frame_fetch()
            for key in ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb"):
                assert np.array_equal(_bits(got[key]), _bits(want[key])), (f, key)
            assert np.array_equal(a.track_ids(), want_ids), f
        assert not np.array_equal(b.track_ids(), np.arange(len(want_ids))), "the IDs never left the row indices"
        assert np.array_equal(_bits(a.tracker_dump()), _bits(b.tracker_dump()))
        # reset: IDs restart at 0, the switch is kept
        b.set_track_retirement(True)
        b.tracker_reset()
        assert b.get_track_retirement()
        book = _Ids()
        for ts, boxes, v, y in scene[:3]:
            r = b.track_step(boxes, 1e9 + ts, v, y)
            assert np.array_equal(b.track_ids(), book.step(r["track_manage"])), "IDs after reset"
        n_rows = len(r["track_manage"])
        # load: rows 0..n-1, the counter continues at n
        dump = b.tracker_dump()
        b.tracker_load(dump, 1, 1e9 + scene[2][0], 0.0, OFF, OFF, -np.pi / 2)
        ts, boxes, v, y = scene[3]
        r = b.track_step(boxes, 1e9 + ts, v, y)
        assert np.array_equal(b.track_ids(), np.arange(len(r["track_manage"]))), "IDs after load"
        assert b.get_track_retirement() and n_rows > 0
        # reopen: every sequence off
        b.seq_open(3, ring=2)
        b.seq_set_track_retirement(1, True)
        b.seq_tracker_reset(1)
        assert b.seq_get_track_retirement(1)
        b.seq_open(3, ring=2)
        assert [b.seq_get_track_retirement(k) for k in range(3)] == [False, False, False]
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ 7. timing mode
@pytest.mark.parametrize("gf", [0, 1])
def test_timing_mode_kernel_times(pkg, gf):
    """Catches a tuned or retiring table whose tracker chain marks a different set of kernels in timing mode (lmot_enable_timing: TA, TB
    and TC each followed by an event, launched without programmatic dependence) than a table at the defaults, and timing mode changing a
    result.  lmot_track_step over 30 frames of the bench scene with a moving ego, compat first frame included: a default, a tuned (every
    association at 99 m also happens at 1e9 m) and a retiring context, timed, each against an untimed twin with the same settings."""
    scene = bench_scene(30)
    arms = ("default", "tuned", "retire")
    ctx = {}
    try:
        for arm in arms:
            for timed in (True, False):
                c = _ctx(pkg, retire=arm == "retire", gf=gf)
                if arm == "tuned":
                    c.set_tracker_params(distance_thres=1e9)
                c.enable_timing(timed)
                ctx[arm, timed] = c
        for f, (ts, boxes, v, y) in enumerate(scene):
            out, n_times = {}, {}
            for arm in arms:
                out[arm] = ctx[arm, True].track_step(boxes, ts, v, y)
                n_times[arm] = len(ctx[arm, True].last_kernel_ms())
                _same_outputs(out[arm], ctx[arm, False].track_step(boxes, ts, v, y), (arm, f))
                assert np.array_equal(ctx[arm, True].track_ids(), ctx[arm, False].track_ids()), (arm, f)
            _same_outputs(out["tuned"], out["default"], ("tuned vs default", f))
            assert n_times["default"] > 0 and n_times["tuned"] == n_times["default"] == n_times["retire"], (f, n_times)
        for arm in arms:
            assert np.array_equal(_bits(ctx[arm, True].tracker_dump()), _bits(ctx[arm, False].tracker_dump())), arm
    finally:
        for c in ctx.values():
            c.close()


# ------------------------------------------------------------------------------------------------ 8. validation
def test_validation(pkg):
    """Catches a missing argument check of the new calls."""
    c = pkg.Lmot(_params(pkg))
    L = c.lib
    try:
        n = C.c_int(0)
        ids = (C.c_int64 * 4)()
        on = C.c_int(0)
        for fn in (L.lmot_track_ids, L.lmot_seq_track_ids, L.lmot_set_track_retirement, L.lmot_get_track_retirement,
                   L.lmot_seq_set_track_retirement, L.lmot_seq_get_track_retirement):
            fn.argtypes = None
        assert L.lmot_track_ids(c.h, ids, 4, C.byref(n)) == pkg.ERR_STATE                 # no result yet
        assert L.lmot_track_ids(None, ids, 4, C.byref(n)) == pkg.ERR_INVALID
        assert L.lmot_track_ids(c.h, ids, 4, None) == pkg.ERR_INVALID
        assert L.lmot_track_ids(c.h, None, 4, C.byref(n)) == pkg.ERR_INVALID
        assert L.lmot_track_ids(c.h, ids, -1, C.byref(n)) == pkg.ERR_INVALID
        assert L.lmot_set_track_retirement(None, 1) == pkg.ERR_INVALID
        assert L.lmot_get_track_retirement(c.h, None) == pkg.ERR_INVALID
        assert L.lmot_get_track_retirement(None, C.byref(on)) == pkg.ERR_INVALID
        for k in (-1, 0, 8):                                 # no open set
            assert L.lmot_seq_set_track_retirement(c.h, k, 1) == pkg.ERR_INVALID
            assert L.lmot_seq_get_track_retirement(c.h, k, C.byref(on)) == pkg.ERR_INVALID
            assert L.lmot_seq_track_ids(c.h, k, ids, 4, C.byref(n)) == pkg.ERR_INVALID
        c.seq_open(2, ring=2)
        assert L.lmot_seq_track_ids(c.h, 0, ids, 4, C.byref(n)) == pkg.ERR_STATE
        assert L.lmot_seq_track_ids(c.h, 2, ids, 4, C.byref(n)) == pkg.ERR_INVALID
        assert L.lmot_seq_get_track_retirement(c.h, 1, None) == pkg.ERR_INVALID
        assert L.lmot_seq_set_track_retirement(c.h, 1, 1) == 0
        assert L.lmot_seq_get_track_retirement(c.h, 1, C.byref(on)) == 0 and on.value == 1
        c.track_step(boxes_at(np.array([[10.0, 0.0], [20.0, 5.0]])), 1e6)
        assert L.lmot_track_ids(c.h, None, 0, C.byref(n)) == 0 and 1 <= n.value <= 2
        assert L.lmot_track_ids(c.h, ids, 4, C.byref(n)) == 0 and list(ids[: n.value]) == list(range(n.value))
    finally:
        c.close()
