"""lmot_tracker_params on the GPU: the tuned kernels against the default ones, against twin contexts and against the reference with
the same constants (oracle/_ref/libref_tunable.so).

Bars as in test_tracker_gpu: identical integers and flags, targets / vandyaw / vis_bb as in test_teacher_forced_steps, UKF state
within 1e-4 relative; free-running comparisons leave out filters that are not positive definite (_pd_tracks).  Each docstring names
the breakage the test is meant to catch; those breakages were reasoned out, not injected.
"""
import numpy as np
import pytest

from test_seq_track_gpu import N_TICKS, RIG, _ListSeq, _params, _run, _same_tables, _Twin, _bits, boxes_at
from test_tracker_gpu import INTS, STATE, TOL, _boxes_sequence, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu

OFF = -0.63035 - np.pi / 2          # firstEgoYawOffset_, imm_ukf_jpda.cpp:70
OUT_KEYS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")

# the reference's own commented-out alternatives (imm_ukf_jpda.cpp:31-42, ukf.cpp:53-58, :92-95, :156-166, :263-267)
REF_ALT = dict(gamma_g=5.99, p_g=0.95, distance_thres=1.0, lifetime_thres=8, std_a=[0.8, 0.8, 5.0], std_yawdd=[0.8, 0.8, 3.0],
               std_las_x=0.3, std_las_y=0.3, trans=[[0.8, 0.1, 0.1], [0.8, 0.1, 0.1], [0.1, 0.1, 0.8]], p0_diag=[0.5, 0.5, 1.0, 1.0, 1.0])
REF_ALT2 = dict(gamma_g=15.22, std_a=[3.0, 3.0, 3.0], std_yawdd=[3.0, 3.0, 3.0], distance_thres=0.25, p0_diag=[0.5, 0.5, 3.0, 1.0, 1.0])
# every field moved
ALL_MOVED = dict(gamma_g=7.5, p_g=0.97, p_d=0.85, distance_thres=2.0, lifetime_thres=2, bb_yaw_change_thres=0.3, second_init_v=1.5,
                 static_lifetime=6, static_dist=4.0, std_a=[1.5, 2.5, 3.5], std_yawdd=[1.0, 1.8, 2.6], std_las_x=0.2, std_las_y=0.12,
                 trans=[[0.85, 0.1, 0.05], [0.07, 0.88, 0.05], [0.1, 0.05, 0.85]], mode_prob0=[0.4, 0.35, 0.25],
                 p0_diag=[0.4, 0.6, 2.5, 8.0, 1.2])
NOOP = dict(distance_thres=1e9)     # tuned, but every box association that happens at 99 m also happens at 1e9 m


@pytest.fixture(scope="module")
def ref_tunable():
    from oracle import ref_tunable as rt
    if not rt.have_ref("tunable"):
        pytest.skip("oracle/_ref/libref_tunable.so not built")
    r = rt.RefTunable()
    yield r
    r.set_tracker_params(None)


def _ctx(pkg, **kw):
    return pkg.Lmot(_params(pkg, **kw))


def _kernel_names(fn):
    """names of the CUDA kernels `fn` launches (torch.profiler; the library's kernels show up by their mangled names)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "imm_" in e.name or "spawn_output" in e.name]


def _same_outputs(a, b, what):
    for k in OUT_KEYS:
        assert a[k].shape == b[k].shape and np.array_equal(_bits(a[k]), _bits(b[k])), (what, k)


def _lattice(n, spacing=4.0):
    side = int(np.ceil(np.sqrt(n)))
    g = np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2)[:n] * spacing
    return g + np.array([5.0, -side * spacing / 2])


# ------------------------------------------------------------------------------------------------ the default path stays
def test_defaults_are_todays_path(pkg):
    """Catches a selection that takes the tuned kernels for a table at the defaults (set to the defaults, or restored with NULL), and
    a restore that leaves a value behind."""
    ctxs = [_ctx(pkg) for _ in range(3)]
    try:
        ctxs[1].set_tracker_params(**pkg.default_tracker_params())
        ctxs[2].set_tracker_params(**ALL_MOVED)
        ctxs[2].set_tracker_params()                       # NULL: the defaults again
        for c in ctxs[1:]:
            assert c.get_tracker_params() == pkg.default_tracker_params()
        seq = _ListSeq(3, n_ticks=N_TICKS)
        names = []
        for f in range(N_TICKS):
            v, yaw = seq.ego(f)
            outs = []
            for i, c in enumerate(ctxs):
                step = lambda: outs.append(c.track_step(seq.lists[f], seq.ts(f), v, yaw))
                if f == 5 and i > 0:
                    names += _kernel_names(step)
                else:
                    step()
            for i in (1, 2):
                _same_outputs(outs[0], outs[i], (f, i))
        for i in (1, 2):
            assert np.array_equal(_bits(ctxs[0].tracker_dump()), _bits(ctxs[i].tracker_dump())), i
        print("kernels at the defaults:", sorted(set(names)))
        assert names, "the profiler recorded none of the tracker's kernels"
        assert not any("tuned" in n for n in names), names
    finally:
        for c in ctxs:
            c.close()


def test_noop_tuned_values(pkg, synth):
    """Catches the tuned kernels misreading any field other than the one changed (distance_thres = 1e9 changes nothing the scenes can
    reach), free-running on caller lists with ego motion, on the synth scene (40 frames), on 100 frames of the bench scene and on a
    denser scene whose active count crosses TC's 256 / 512 variants."""
    scenes = {"lists": [(_ListSeq(2, n_ticks=N_TICKS).lists[f], 1.0e6 + 1.0e5 * f, 1.0, 0.2 + 0.01 * f) for f in range(N_TICKS)]}
    det = pkg.Lmot()                          # the scenes' boxes: this library's detection of the synthetic frames
    try:
        for name, cfg, n in (("synth", synth.SceneConfig(seed=2, n_objects=72), 40),
                             ("bench scene", synth.SceneConfig(n_objects=150, lattice_pitch=3.8, ped_fraction=0.65, seed=1), 100)):
            scenes[name] = [(det.frame(pts, ts)["boxes"].copy(), ts, 0.0, 0.0) for ts, pts in synth.frames(cfg, n)]
    finally:
        det.close()
    rng = np.random.default_rng(3)
    base = _lattice(600, 3.0)
    scenes["dense"] = [(boxes_at(base[: 150 + 45 * f] + rng.normal(0, 0.02, (150 + 45 * f, 2))), 2.0e6 + 1.0e5 * f, 0.0, 0.0)
                       for f in range(11)]
    for name, scene in scenes.items():
        a, b = _ctx(pkg), _ctx(pkg)
        try:
            b.set_tracker_params(**NOOP)
            names = []
            for f, (boxes, ts, v, yaw) in enumerate(scene):
                ra = a.track_step(boxes, ts, v, yaw)
                if f == 3:
                    out = []
                    names = _kernel_names(lambda: out.append(b.track_step(boxes, ts, v, yaw)))
                    rb = out[0]
                else:
                    rb = b.track_step(boxes, ts, v, yaw)
                _same_outputs(ra, rb, (name, f))
            assert np.array_equal(_bits(a.tracker_dump()), _bits(b.tracker_dump())), name
            print(name, "tuned kernels:", sorted(set(names)))
            assert names, "the profiler recorded none of the tracker's kernels"
            assert all("tuned" in n for n in names), names
        finally:
            a.close(); b.close()


# ------------------------------------------------------------------------------------------------ against the reference
def _teacher_forced(lm, ref, seq, what):
    ref.tracker_reset(); lm.tracker_reset()
    prev_ts = None
    for f, (ts, boxes) in enumerate(seq):
        if f > 0:
            state = ref.tracker_dump()
            lm.tracker_load(state, 1, prev_ts, 0.0, OFF, OFF, -np.pi / 2)
            ref.tracker_load(state, 1, prev_ts, 0.0, OFF, OFF, -np.pi / 2)
        a = ref.tracker_step(boxes, ts)
        b = lm.track_step(boxes, ts)
        for k in ("track_manage", "is_static", "is_vis"):
            assert np.array_equal(a[k], b[k]), (what, f, k)
        da, db = ref.tracker_dump(), lm.tracker_dump()
        assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (what, f)
        live = da[:, 0] > 0
        err = _rel_err(da[live][:, STATE], db[live][:, STATE])
        assert err.size == 0 or err.max() < TOL, (what, f, float(err.max()))
        np.testing.assert_allclose(b["targets"], a["targets"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(b["vandyaw"], a["vandyaw"], rtol=1e-4, atol=1e-6)
        assert a["vis_bb"].shape == b["vis_bb"].shape, (what, f)
        np.testing.assert_allclose(b["vis_bb"], a["vis_bb"], rtol=1e-5, atol=1e-5)
        prev_ts = ts


def _free_running(lm, ref, seq, what, ego=False):
    ref.tracker_reset(); lm.tracker_reset()
    worst = 0.0
    for f, (ts, boxes) in enumerate(seq):
        v, yaw = (1.0 + 0.05 * f, 0.2 + 0.01 * f) if ego else (0.0, 0.0)
        a = ref.tracker_step(boxes, ts, v, yaw)
        b = lm.track_step(boxes, ts, v, yaw)
        for k in ("track_manage", "is_static", "is_vis"):
            assert np.array_equal(a[k], b[k]), (what, f, k)
        da, db = ref.tracker_dump(), lm.tracker_dump()
        assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (what, f)
        ok = _pd_tracks(da)
        err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
        if err.size:
            worst = max(worst, float(err.max()))
            assert err.max() < TOL, (what, f, float(err.max()))
    return worst


@pytest.mark.parametrize("name", ["ref_alt", "ref_alt2", "all_moved"])
def test_params_match_tunable_reference(pkg, synth, ref_tunable, name):
    """Catches a field wired to the wrong model, row or stage (the values differ per model and per row), and a compat first frame that
    spawns with the literals.  40 frames, teacher-forced and free-running (with ego motion), against the reference with the same
    constants."""
    prm = {"ref_alt": REF_ALT, "ref_alt2": REF_ALT2, "all_moved": ALL_MOVED}[name]
    seq = _boxes_sequence(ref_tunable, synth, seed=11, n_frames=40)
    lm = _ctx(pkg)
    try:
        lm.set_tracker_params(**prm)
        ref_tunable.set_tracker_params(prm)
        _teacher_forced(lm, ref_tunable, seq, (name, "teacher-forced"))
        worst = _free_running(lm, ref_tunable, seq, (name, "free-running"), ego=True)
        print(name, "free-running worst relative state error:", worst)
    finally:
        ref_tunable.set_tracker_params(None)
        lm.close()


REGIME_SET = dict(ALL_MOVED, static_lifetime=4, static_dist=6.0)     # slow lattice: the static thresholds decide within 14 frames


@pytest.mark.parametrize("n_tracks", [400, 700])
def test_tuned_regimes_on_sequence_tc(pkg, ref_tunable, n_tracks):
    """Catches a TC path or width that still uses the literals.  Free-running from a reset over 14 frames of a slowly moving lattice:
    a compat first frame (ukf_initialize's p0_diag and mode_prob0), then more than 256 active tracks (400: the 512-thread fast path,
    emit_values) or more than 512 (700: the general path, emit_track), where every track turns static (static_lifetime /
    static_dist decide when).  Then teacher-forced from the same lattice: every step follows a table load, so TC rebuilds from the
    records on its general path."""
    rng = np.random.default_rng(n_tracks)
    base = _lattice(n_tracks)
    seq = [(3.0e6 + 1.0e5 * f, boxes_at(base + 0.02 * f + rng.normal(0, 0.02, base.shape))) for f in range(14)]
    lm = _ctx(pkg)
    try:
        lm.set_tracker_params(**REGIME_SET)
        ref_tunable.set_tracker_params(REGIME_SET)
        ref_tunable.tracker_reset(); lm.tracker_reset()
        names = []
        for f, (ts, boxes) in enumerate(seq):
            a = ref_tunable.tracker_step(boxes, ts)
            if f == 8:
                out = []
                names = _kernel_names(lambda: out.append(lm.track_step(boxes, ts)))
                b = out[0]
            else:
                b = lm.track_step(boxes, ts)
            for k in ("track_manage", "is_static", "is_vis"):
                assert np.array_equal(a[k], b[k]), (n_tracks, f, k)
            da, db = ref_tunable.tracker_dump(), lm.tracker_dump()
            assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (n_tracks, f)
            ok = _pd_tracks(da)
            err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
            assert err.size == 0 or err.max() < TOL, (n_tracks, f, float(err.max()))
        assert b["is_static"].sum() > 0, "the scene never reaches the static thresholds"
        print(n_tracks, "tracks: TC kernels", sorted({n.split("(")[0] for n in names if "spawn_output" in n}),
              "static at the end:", int(b["is_static"].sum()))
        assert names, "the profiler recorded none of the tracker's kernels"
        assert any("spawn_output_seq_tuned_kernel<512>" in n for n in names), names
        _teacher_forced(lm, ref_tunable, seq[:8], ("lattice, teacher-forced", n_tracks))
    finally:
        ref_tunable.set_tracker_params(None)
        lm.close()


# ------------------------------------------------------------------------------------------------ sequences
SEQ_SETS = [None, REF_ALT, ALL_MOVED, NOOP, REF_ALT2, dict(p_d=0.8, second_init_v=1.0), dict(static_lifetime=4, static_dist=6.0),
            dict(std_las_x=0.25, mode_prob0=[0.5, 0.3, 0.2])]


@pytest.mark.parametrize("mode", ["sync", "dev"])
@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("table", [False, True])
def test_seq_params_equal_twins(pkg, ref_tunable, mode, gf, table):
    """Catches a CTA reading sequence 0's parameter slice (every sequence has its own set), and a sequence at the defaults disturbed by
    a tick that runs the tuned kernels (sequence 0).  Sequence 7 has a sensor table in one case.  Sequence 2 is also checked against
    the reference with its constants."""
    if table and mode == "dev" and gf == 1:
        pytest.skip("covered by the other table cases")
    S = 8
    prm = _params(pkg, gf=gf)
    ctx = pkg.Lmot(prm)
    rigs = [None] * S
    if table:
        rigs[7] = RIG[:1]
    twins = [_Twin(pkg, prm, rigs[k]) for k in range(S)]
    try:
        ctx.seq_open(S, ring=N_TICKS + 1)
        if table:
            from test_seq_track_gpu import _table_kw
            ctx.seq_set_sensors(7, **_table_kw(rigs[7]))
        for k, p in enumerate(SEQ_SETS):
            if p:
                ctx.seq_set_tracker_params(k, **p)
                twins[k].ctx.set_tracker_params(**p)
        seqs = [_ListSeq(k) for k in range(S)]
        got = _run(pkg, ctx, seqs, twins, mode, N_TICKS)
        _same_tables(ctx, twins, ("final", mode, gf, table))
        if gf == 0 and mode == "sync":
            ref_tunable.set_tracker_params(SEQ_SETS[2])
            try:
                ref_tunable.tracker_reset()
                s = seqs[2]
                for f in range(N_TICKS):
                    v, yaw = s.ego(f)
                    a = ref_tunable.tracker_step(s.lists[f], s.ts(f), v, yaw)
                    assert np.array_equal(a["track_manage"], got[f][2]["track_manage"]), f
                da, db = ref_tunable.tracker_dump(), ctx.seq_tracker_dump(2)
                assert np.array_equal(da[:, INTS], db[:, INTS])
                ok = _pd_tracks(da)
                err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
                assert err.size == 0 or err.max() < TOL, float(err.max())
            finally:
                ref_tunable.set_tracker_params(None)
    finally:
        ctx.close()
        for t in twins:
            t.close()


@pytest.mark.parametrize("gf", [0, 1])
def test_seq_detection_ticks_with_params(pkg, synth, gf):
    """Catches detection ticks (pipelined lmot_seq_dev) that step the tables without their parameters: four sequences, three with
    their own sets, 30 ticks, every output and dump row equal to a twin context with the same parameters fed through lmot_frame."""
    import torch
    from test_sequences_gpu import _params as _seq_params, _same, _same_dump, _seqs, _tick_args
    S = 4
    sets = [None, REF_ALT, ALL_MOVED, dict(static_lifetime=4, static_dist=6.0, p_d=0.8)]
    seqs = _seqs(synth, S)
    ctx = pkg.Lmot(_seq_params(pkg, gf))
    twins = [pkg.Lmot(_seq_params(pkg, gf)) for _ in range(S)]
    try:
        ctx.seq_open(S, ring=N_TICKS)
        for k, p in enumerate(sets):
            if p:
                ctx.seq_set_tracker_params(k, **p)
                twins[k].set_tracker_params(**p)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        want, keep = [], []
        for f in range(N_TICKS):
            frames, ts, v, yaw = _tick_args(seqs, f)
            want.append([twins[k].frame(frames[k], ts[k], v[k], yaw[k]) for k in range(S)])
            with torch.cuda.stream(stream):
                d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in frames]
                keep.append(d)
                ctx.seq_dev([(t.data_ptr(), len(p)) for t, p in zip(d, frames)], ts, v, yaw)
        for f in range(N_TICKS):
            got = ctx.seq_collect()
            for k in range(S):
                _same(got[k], want[f][k], (f, k))
        ctx.set_stream(None)
        for k in range(S):
            _same_dump(ctx.seq_tracker_dump(k), twins[k].tracker_dump(), k)
    finally:
        ctx.close()
        for t in twins:
            t.close()


def test_in_flight_and_midrun_change(pkg, ref_tunable):
    """Catches a submission that reads the parameters at execution instead of copying them (ticks in flight when they change must
    keep the old values), and a change that does not reach the tracks that already exist.  A mid-run change equals the reference
    reloaded from the dump under the new constants."""
    S, n1, n2 = 2, 8, 12
    prm = _params(pkg)
    ctx = pkg.Lmot(prm)
    twins = [_Twin(pkg, prm) for _ in range(S)]
    seqs = [_ListSeq(0, n_ticks=n1 + n2, seed=5), _ListSeq(1, n_ticks=n1 + n2, seed=6)]
    try:
        ctx.seq_open(S, ring=n1 + n2)
        want = []
        for f in range(n1 + n2):
            if f == n1:
                ctx.seq_set_tracker_params(0, **ALL_MOVED)      # ticks 0..n1-1 are still in flight
                twins[0].ctx.set_tracker_params(**ALL_MOVED)
            ts = [s.ts(f) for s in seqs]
            v = [s.ego(f)[0] for s in seqs]
            yaw = [s.ego(f)[1] for s in seqs]
            ctx.seq_track_submit([s.lists[f] for s in seqs], ts, v, yaw)
            want.append([twins[k].step(seqs[k].lists[f], ts[k], v[k], yaw[k])[1] for k in range(S)])
        for f in range(n1 + n2):
            got = ctx.seq_collect()
            for k in range(S):
                _same_outputs(got[k], want[f][k], (f, k))
        _same_tables(ctx, twins, "final")
    finally:
        ctx.close()
        for t in twins:
            t.close()
    # the reference: n1 steps at the defaults, dump, reload under the new constants, n2 more steps
    s = seqs[0]
    lm = _ctx(pkg)
    try:
        ref_tunable.set_tracker_params(None)
        ref_tunable.tracker_reset()
        for f in range(n1):
            ref_tunable.tracker_step(s.lists[f], s.ts(f))
            lm.track_step(s.lists[f], s.ts(f))
        state = ref_tunable.tracker_dump()
        ref_tunable.set_tracker_params(ALL_MOVED)
        ref_tunable.tracker_load(state, 1, s.ts(n1 - 1), 0.0, OFF, OFF, -np.pi / 2)
        lm.set_tracker_params(**ALL_MOVED)
        for f in range(n1, n1 + n2):
            a = ref_tunable.tracker_step(s.lists[f], s.ts(f))
            b = lm.track_step(s.lists[f], s.ts(f))
            assert np.array_equal(a["track_manage"], b["track_manage"]), f
            da, db = ref_tunable.tracker_dump(), lm.tracker_dump()
            assert np.array_equal(da[:, INTS], db[:, INTS]), f
            ok = _pd_tracks(da)
            err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
            assert err.size == 0 or err.max() < TOL, (f, float(err.max()))
    finally:
        ref_tunable.set_tracker_params(None)
        lm.close()


def test_tracker_params_validation(pkg):
    """Catches a rejection that leaves a partial change behind, a getter that does not return what was set, and a reopened set that
    keeps the old parameters."""
    ctx = _ctx(pkg)
    try:
        d = pkg.default_tracker_params()
        bad = [dict(gamma_g=float("nan")), dict(gamma_g=0.0), dict(p_g=0.0), dict(p_g=1.5), dict(p_d=-0.1), dict(std_a=[2, 0, 3]),
               dict(std_yawdd=[2, 2, -1]), dict(std_las_x=0.0), dict(std_las_y=float("inf")), dict(p0_diag=[0.5, 0.5, 0, 10, 1]),
               dict(mode_prob0=[0.33, 0.0, 0.33]), dict(trans=[[1.2, 0, 0], [0, 1, 0], [0, 0, 1]]),
               dict(trans=[[0.9, 0, 0.1], [0.1, 0, 0.9], [0.5, 0, 0.5]]), dict(trans=[[0.9, -0.1, 0.2], [0, 1, 0], [0, 0, 1]]),
               dict(lifetime_thres=-1), dict(static_lifetime=-2), dict(distance_thres=float("nan")), dict(second_init_v=float("inf"))]
        ctx.set_tracker_params(**REF_ALT)
        want = dict(d, **REF_ALT)
        assert ctx.get_tracker_params() == want
        for b in bad:
            with pytest.raises(pkg.LmotError):
                ctx.set_tracker_params(**b)
            assert ctx.get_tracker_params() == want, b
        ctx.seq_open(3, ring=2)
        ctx.seq_set_tracker_params(1, **ALL_MOVED)
        got = ctx.seq_get_tracker_params(1)
        assert got["gamma_g"] == ALL_MOVED["gamma_g"] and got["trans"] == ALL_MOVED["trans"] and got["p0_diag"] == ALL_MOVED["p0_diag"]
        assert ctx.seq_get_tracker_params(0) == d and ctx.seq_get_tracker_params(2) == d
        for b in bad:
            with pytest.raises(pkg.LmotError):
                ctx.seq_set_tracker_params(1, **b)
            assert ctx.seq_get_tracker_params(1) == got, b
        for k in (-1, 3):
            with pytest.raises(pkg.LmotError):
                ctx.seq_set_tracker_params(k, **REF_ALT)
            with pytest.raises(pkg.LmotError):
                ctx.seq_get_tracker_params(k)
        ctx.seq_tracker_reset(1)
        assert ctx.seq_get_tracker_params(1) == got                  # reset keeps them
        ctx.seq_open(3, ring=2)
        assert all(ctx.seq_get_tracker_params(k) == d for k in range(3))   # reopening resets them
        ctx.seq_open(0)
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_tracker_params(0, **REF_ALT)                  # no open set
        ctx.set_tracker_params()
        assert ctx.get_tracker_params() == d
    finally:
        ctx.close()
