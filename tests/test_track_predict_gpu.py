"""Track prediction on the GPU (lmot_predict_tracks*, predict_tracks_kernel) against the reference's own prediction (oracle/ref_predict.cpp:
ProcessIMMUKF + findMaxZandS + PostProcessIMMUKF({1, 1, 1}) on copies of the reference's rows), against the host forms and twin
contexts, and the tracker chain unchanged by it.

Bars as in test_tracker_gpu: flags, IDs and trackManage identical; x, P, mode_prob, gate_z and gate_S within 1e-4 relative (NaN where
the oracle has NaN); free-running comparisons leave out rows whose covariance is not positive definite (_pd_tracks).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from test_seq_track_gpu import _ListSeq, _bits, _pad_lists, _params, boxes_at
from test_track_retire_gpu import _Ids, bench_scene
from test_global_frame_gpu import xf_apply, xf_pair
from test_tracker_gpu import _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OFF = -0.63035 - np.pi / 2
TOL = 1e-4
AFTER = (0.0, 1.0, 5e4, 1e5, 5e5, 1e6, 3e6, 1e7)
VALUES = ("x", "P", "mode_prob", "gate_z", "gate_S")
TUNED = dict(gamma_g=7.5, std_a=[1.5, 2.5, 3.5], std_yawdd=[1.0, 2.5, 4.0], std_las_x=0.2, std_las_y=0.1,
             trans=[[0.8, 0.15, 0.05], [0.1, 0.85, 0.05], [0.05, 0.05, 0.9]])
WORST = {}


@pytest.fixture(scope="module")
def ref():
    from oracle import ref, ref_predict
    if not ref.have_ref("intended") or not ref_predict.have_predict("intended"):
        pytest.skip("oracle/_ref not built")
    r = ref.RefOracle("intended")
    r.tracker_predict = ref_predict.predictor(r)
    return r


@pytest.fixture(scope="module")
def ref_tunable():
    from oracle import ref_predict
    from oracle import ref_tunable as rt
    if not rt.have_ref("tunable") or not ref_predict.have_predict("tunable"):
        pytest.skip("oracle/_ref/libref_tunable.so not built")
    r = rt.RefTunable()
    r.tracker_predict = ref_predict.predictor(r)
    yield r
    r.set_tracker_params(None)


def _vs_oracle(got, want, what, rows=None):
    """got: Lmot.predict_tracks' dict, want: the oracle's (no ids); rows: the rows whose values are compared (default: all)"""
    n = len(want["track_manage"])
    assert np.array_equal(got["track_manage"], want["track_manage"]), (what, "track_manage")
    sel = np.ones(n, bool) if rows is None else rows
    assert np.array_equal(got["flags"][:, sel], want["flags"][:, sel]), (what, "flags")
    worst = 0.0
    for k in VALUES:
        a, b = want[k][:, sel], got[k][:, sel]
        assert a.shape == b.shape, (what, k)
        assert np.array_equal(np.isnan(a), np.isnan(b)), (what, k, "NaN pattern")
        err = _rel_err(a, b)
        if err.size:
            worst = max(worst, float(err.max()))
    WORST[what] = worst
    print(f"{what}: worst relative error {worst:.3g}")
    assert worst < TOL, (what, worst)


def _run_ref(r, scene):
    r.tracker_reset()
    for ts, b, v, y in scene:
        r.tracker_step(b, ts, v, y)
    return scene[-1][0]


def _load_both(lm, r, dumps, ts):
    lm.tracker_load(dumps, 1, ts, 0.0, OFF, OFF, -np.pi / 2)
    r.tracker_load(dumps, 1, ts, 0.0, OFF, OFF, -np.pi / 2)


def _lattice_table(r, n=1024):
    """the stress table of test_tracker_gpu: 1024 mature tracks on a 32 x 32 lattice"""
    rng = np.random.default_rng(0)
    gx, gy = np.meshgrid(np.arange(32) * 8.0 - 124.0, np.arange(32) * 8.0 - 124.0, indexing="ij")
    pos = np.stack([gx.ravel(), gy.ravel()], 1)[:n]
    r.tracker_reset()
    ts = 0.0
    for _ in range(8):
        ts += 1e5
        r.tracker_step(boxes_at(pos + rng.normal(0, 0.02, pos.shape)), ts)
    return r.tracker_dump(), ts


class _Dev:
    """device outputs of n_t times x cap rows (torch), as lmot_pred_out"""

    def __init__(self, pkg, n_t, cap, gate=True):
        import torch
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device="cuda")
        self.t = {"ids": z(cap, torch.int64), "track_manage": z(cap, torch.int32), "flags": z((n_t, cap), torch.uint8),
                  "x": z((n_t, cap, 5), torch.float64), "P": z((n_t, cap, 5, 5), torch.float64), "mode_prob": z((n_t, cap, 3), torch.float64)}
        if gate:
            self.t["gate_z"] = z((n_t, cap, 2), torch.float64)
            self.t["gate_S"] = z((n_t, cap, 4), torch.float64)
        self.n = z(1, torch.int32)
        self.out = pkg.pred_out(cap, {k: v.data_ptr() for k, v in self.t.items()})
        torch.cuda.synchronize()

    def host(self):
        import torch
        torch.cuda.synchronize()
        n = int(self.n.cpu()[0])
        h = {k: v.cpu().numpy() for k, v in self.t.items()}
        return {k: (a[:n] if k in ("ids", "track_manage") else a[:, :n]) for k, a in h.items()}


def _frame_params(pkg):
    p = _params(pkg)
    p.max_points = 1 << 18
    return p


def _same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(_bits(a[k]), _bits(b[k])), (what, k)


# ------------------------------------------------------------------------------------------------ teacher-forced
@pytest.mark.parametrize("table", ["bench20", "bench60", "stress1024"])
def test_teacher_forced_against_the_oracle(pkg, ref, table):
    """a table loaded from the reference, predicted at ts_last + 0 .. 10 s in one call, against the oracle on the same table"""
    if table == "stress1024":
        dumps, ts = _lattice_table(ref)
    else:
        ts = _run_ref(ref, bench_scene(int(table[5:])))
        dumps = ref.tracker_dump()
    lm = pkg.Lmot(_params(pkg, max_tracks=4096))
    try:
        _load_both(lm, ref, dumps, ts)
        times = [ts + d for d in AFTER]
        got, want = lm.predict_tracks(times), ref.tracker_predict(times)
        assert np.array_equal(got["ids"], np.arange(len(dumps)))
        assert (want["flags"] & 1).sum() > 0
        _vs_oracle(got, want, "teacher " + table)
        before = lm.tracker_dump()
        d = _Dev(pkg, len(times), len(dumps))
        lm.predict_tracks_dev(times, d.out, d.n.data_ptr())
        _same(d.host(), got, "dev form")
        assert np.array_equal(_bits(before), _bits(lm.tracker_dump()))          # the table is never written
    finally:
        lm.close()


def test_teacher_forced_tuned_parameters(pkg, ref_tunable):
    """a table with its own parameters against libref_predict_tunable with the same values as globals"""
    ref_tunable.set_tracker_params(TUNED)
    try:
        ts = _run_ref(ref_tunable, bench_scene(30))
        dumps = ref_tunable.tracker_dump()
        lm = pkg.Lmot(_params(pkg))
        try:
            lm.set_tracker_params(**TUNED)
            _load_both(lm, ref_tunable, dumps, ts)
            times = [ts + d for d in AFTER]
            _vs_oracle(lm.predict_tracks(times), ref_tunable.tracker_predict(times), "teacher tuned")
        finally:
            lm.close()
    finally:
        ref_tunable.set_tracker_params(None)


# ------------------------------------------------------------------------------------------------ free-running, pipelined
@pytest.mark.parametrize("gf", [0, 1])
def test_free_running_lists_dev_with_a_prediction_after_every_step(pkg, ref, gf):
    """50 bench steps through lmot_track_step_lists_dev, each followed by lmot_predict_tracks_dev (n_t = 4) into its own buffers, all
    submitted before anything is read; against the reference stepped on the same boxes (global_frame 1: fed the transformed boxes,
    whose ego pose it then shares, as in test_global_frame_gpu).  (Beyond ~55 free-running steps of this scene the two tables drift
    apart by more than the bar in a few well-conditioned rows, and a 1 s prediction amplifies that: the drift is the step's, which
    test_tracker_gpu bounds.)"""
    import torch
    scene = bench_scene(50)
    lm = pkg.Lmot(_params(pkg, gf=gf))
    lm.set_stream(None)
    try:
        ref.tracker_reset()
        wants, devs, pd = [], [], []
        for f, (ts, b, v, y) in enumerate(scene):
            fwd = xf_pair(lm.origin_points(ts, v, y))[0] if gf else None
            d_lists, d_counts, cap = _pad_lists([b])
            lm.track_step_lists_dev(d_lists.data_ptr(), d_counts.data_ptr(), 1, cap, ts, v, y)
            times = [ts, ts + 5e4, ts + 1e5, ts + 1e6]
            d = _Dev(pkg, len(times), 2048, gate=(f % 2 == 0))
            lm.predict_tracks_dev(times, d.out, d.n.data_ptr())
            devs.append((d, d_lists, d_counts))
            ref.tracker_step(xf_apply(fwd, b) if gf else b, ts, v, y)
            wants.append(ref.tracker_predict(times))
            pd.append(_pd_tracks(ref.tracker_dump()))
            if f % 8 == 7:
                torch.cuda.synchronize()
                lm.frame_fetch()
        for f, (d, _, _) in enumerate(devs):
            got = d.host()
            if f % 2:
                got.update({k: wants[f][k] for k in ("gate_z", "gate_S")})
            keep = pd[f] | (wants[f]["track_manage"] == 0)
            _vs_oracle(got, wants[f], f"free lists_dev gf={gf} step {f}", rows=keep)
    finally:
        lm.close()


def test_free_running_frame_dev_pipelined(pkg, ref, synth):
    """30 synthetic frames through lmot_frame_dev (detection overlapping the chain), a prediction after every submission; against the
    reference's detection + tracker on the same frames"""
    import torch
    frames = list(synth.frames(synth.SceneConfig(seed=3, n_objects=40), 30))
    lm = pkg.Lmot(_frame_params(pkg))
    try:
        ref.tracker_reset()
        wants, devs, pd, keep_pts = [], [], [], []
        for ts, pts in frames:
            e, _ = ref.ground_remove(pts)
            g, k = ref.component_clustering(e)
            b, _ = ref.box_fitting(e, g, k)
            ref.tracker_step(b, ts)
            times = [ts + 1e5, ts + 2e5]
            wants.append(ref.tracker_predict(times))
            pd.append(_pd_tracks(ref.tracker_dump()))
            x = torch.from_numpy(np.ascontiguousarray(pts[:, :4], np.float32)).cuda()
            torch.cuda.synchronize()
            keep_pts.append(x)
            lm.frame_dev(x.data_ptr(), len(pts), ts)
            d = _Dev(pkg, len(times), 2048)
            lm.predict_tracks_dev(times, d.out, d.n.data_ptr())
            devs.append(d)
            torch.cuda.synchronize()
            lm.frame_fetch()
        for f, d in enumerate(devs):
            _vs_oracle(d.host(), wants[f], f"free frame_dev step {f}", rows=pd[f] | (wants[f]["track_manage"] == 0))
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ predicting changes nothing
def _frames_arm(pkg, frames, predict):
    """frame_dev pipelined (gated chain); predict: None, 'after' (after every submission) or 'between' (every other one, host form)"""
    import torch
    lm = pkg.Lmot(_frame_params(pkg))
    lm.set_track_retirement(True)
    outs, ids, dumps, keep = [], [], [], []
    try:
        for f, (ts, pts) in enumerate(frames):
            x = torch.from_numpy(np.ascontiguousarray(pts[:, :4], np.float32)).cuda()
            torch.cuda.synchronize()
            keep.append(x)
            lm.frame_dev(x.data_ptr(), len(pts), ts)
            if predict == "after":
                d = _Dev(pkg, 8, 2048)
                lm.predict_tracks_dev([ts + 1e5 * j for j in range(8)], d.out, d.n.data_ptr())
                keep.append(d)
            elif predict == "between" and f % 2:
                lm.predict_tracks([ts + 3e5])
            if f % 3 == 2:
                torch.cuda.synchronize()
                while lm.frames_in_flight():
                    outs.append(lm.frame_collect())
                    ids.append(lm.track_ids())
        torch.cuda.synchronize()
        while lm.frames_in_flight():
            outs.append(lm.frame_collect())
            ids.append(lm.track_ids())
        dumps.append(lm.tracker_dump())
    finally:
        lm.close()
    return outs, ids, dumps


def test_predicting_changes_no_step(pkg, synth):
    """the ordering hazard: a context that predicts after every step, and one that predicts between pipelined submissions, give
    every step output, ID and the final dump bit-identical to a twin that never predicts"""
    frames = list(synth.frames(synth.SceneConfig(seed=4, n_objects=60), 24))
    base = _frames_arm(pkg, frames, None)
    for arm in ("after", "between"):
        got = _frames_arm(pkg, frames, arm)
        assert len(got[0]) == len(base[0]) == len(frames), arm
        for f, (a, b) in enumerate(zip(base[0], got[0])):
            for k in ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb", "boxes"):
                assert np.array_equal(_bits(a[k]), _bits(b[k])), (arm, f, k)
        for a, b in zip(base[1], got[1]):
            assert np.array_equal(a, b), arm
        assert np.array_equal(_bits(base[2][0]), _bits(got[2][0])), arm


def _seq_arm(pkg, seqs, predict, n_ticks):
    ctx = pkg.Lmot(_params(pkg))
    S = len(seqs)
    try:
        ctx.seq_open(S, ring=4)
        for k in range(S):
            ctx.seq_set_tracker_params(k, std_a=[1.5 + 0.1 * k, 2.0, 3.0])
        outs, preds = [], []
        for f in range(n_ticks):
            ts = [s.ts(f) for s in seqs]
            ctx.seq_track_submit([s.lists[f] for s in seqs], ts, [s.ego(f)[0] for s in seqs], [s.ego(f)[1] for s in seqs])
            if predict:
                devs = [_Dev(pkg, 2, 2048) for _ in range(S)]
                ctx.seq_predict_tracks_dev([[t + 1e5, t + 2e5] for t in ts], [d.out for d in devs])
                preds.append(devs)
            if f % 3 == 2:
                for _ in range(3):
                    outs.append(ctx.seq_collect())
        dumps = [ctx.seq_tracker_dump(k) for k in range(S)]
    finally:
        ctx.close()
    return outs, dumps


def test_predicting_changes_no_sequence_tick(pkg):
    seqs = [_ListSeq(k, n_ticks=12) for k in range(8)]
    a = _seq_arm(pkg, seqs, False, 12)
    b = _seq_arm(pkg, seqs, True, 12)
    for ta, tb in zip(a[0], b[0]):
        for k in range(8):
            for key in ("targets", "vandyaw", "track_manage", "is_vis", "vis_bb"):
                assert np.array_equal(_bits(ta[k][key]), _bits(tb[k][key])), (k, key)
    for da, db in zip(a[1], b[1]):
        assert np.array_equal(_bits(da), _bits(db))


# ------------------------------------------------------------------------------------------------ regimes
def test_regimes(pkg, ref):
    """one loaded table with every row kind: dead rows, rows that trip the P guard, rows whose S trips the S guard, trackManage 1, yaw
    at +-pi, |yawd| on both sides of CTRV's 0.001 switch, a model covariance whose P_aug Cholesky stops early; n_t = 1 and 32, a cap
    below the row count"""
    ts = _run_ref(ref, bench_scene(40))
    base = ref.tracker_dump()
    live = np.nonzero(base[:, 0] >= 5)[0]
    assert len(live) >= 12
    rows = []
    for j, mod in enumerate(("dead", "guard_p", "guard_s", "tm1", "yaw+pi", "yaw-pi", "yawd_lo", "yawd_hi", "chol", "plain")):
        d = base[live[j % len(live)]].copy()
        P = lambda m: d[24 + 25 * m: 49 + 25 * m].reshape(5, 5)
        if mod == "dead":
            d[0] = 0
        elif mod == "guard_p":
            P(0)[4, 4] = 2000.0
        elif mod == "guard_s":
            for m in range(1, 4):
                P(m)[0, 0] += 3.0; P(m)[1, 1] += 3.0
        elif mod == "tm1":
            d[0] = 1
        elif mod in ("yaw+pi", "yaw-pi"):
            for m in range(4):
                d[4 + 5 * m + 3] = np.pi if mod == "yaw+pi" else -np.pi
        elif mod in ("yawd_lo", "yawd_hi"):
            for m in range(4):
                d[4 + 5 * m + 4] = 0.00099 if mod == "yawd_lo" else 0.00101
        elif mod == "chol":
            for m in range(1, 4):
                P(m)[2, 2] = -1.0
        rows.append(d)
    dumps = np.concatenate([base, np.array(rows)])
    lm = pkg.Lmot(_params(pkg))
    try:
        _load_both(lm, ref, dumps, ts)
        for times in ([ts + 1e5], [ts + 2e4 * j for j in range(32)]):
            got, want = lm.predict_tracks(times), ref.tracker_predict(times)
            _vs_oracle(got, want, f"regimes n_t={len(times)}")
            fl = want["flags"][:, len(base):]
            assert np.all(fl[:, 0] == 2) and np.all(fl[:, 1] == 4) and np.all(fl[:, 2] & 8) and np.all(fl[:, 3:] & 1)
        # cap below the row count: the host form reports LMOT_ERR_CAPACITY with the count, the rows that fit are right
        o, bufs = _host_out(pkg, 3, 5)
        st = lm.lib.lmot_predict_tracks(lm.h, np.array([ts + 1e5, ts + 2e5, ts + 3e5]).ctypes.data_as(C.c_void_p), 3, C.byref(o))
        assert st == pkg.ERR_CAPACITY and o.n_rows == len(dumps)
        want = ref.tracker_predict([ts + 1e5, ts + 2e5, ts + 3e5], cap=5)
        assert np.array_equal(bufs["flags"], want["flags"]) and np.array_equal(bufs["track_manage"], want["track_manage"])
        np.testing.assert_allclose(bufs["x"], want["x"], rtol=TOL)
        d = _Dev(pkg, 1, 4)
        lm.predict_tracks_dev([ts], d.out, d.n.data_ptr())
        h = d.host()
        assert int(d.n.cpu()[0]) == len(dumps) and h["ids"].tolist() == [0, 1, 2, 3]
        # an empty table; never stepped; after load
        lm.tracker_load(np.zeros((0, 236)), 1, ts, 0.0, OFF, OFF, -np.pi / 2)
        e = lm.predict_tracks([ts])
        assert e["ids"].shape == (0,) and e["x"].shape == (1, 0, 5)
        lm.tracker_reset()
        with pytest.raises(pkg.LmotError) as ex:
            lm.predict_tracks([ts])
        assert ex.value.status == pkg.ERR_STATE
    finally:
        lm.close()


def _host_out(pkg, n_t, cap):
    bufs = {"ids": np.zeros(cap, np.int64), "track_manage": np.zeros(cap, np.int32), "flags": np.zeros((n_t, cap), np.uint8),
            "x": np.zeros((n_t, cap, 5)), "P": np.zeros((n_t, cap, 5, 5)), "mode_prob": np.zeros((n_t, cap, 3))}
    return pkg.pred_out(cap, {k: a.ctypes.data for k, a in bufs.items()}), bufs


def test_append_only_8192_rows(pkg, ref):
    """an append-only table of 8,192 rows, almost all dead: the bench scene's first spawns, then dead padding"""
    ts = _run_ref(ref, bench_scene(30))
    base = ref.tracker_dump()
    dead = np.repeat(base[:1], 8192 - len(base), 0)
    dead[:, 0] = 0
    dumps = np.concatenate([base, dead])
    lm = pkg.Lmot(_params(pkg, max_tracks=8192))
    try:
        _load_both(lm, ref, dumps, ts)
        times = [ts + 1e5, ts + 1e6]
        got = lm.predict_tracks(times, cap=8192)
        assert len(got["ids"]) == 8192
        _vs_oracle(got, ref.tracker_predict(times), "append-only 8192")
    finally:
        lm.close()


def test_retiring_table_ids(pkg, ref):
    """a retiring table: the rows are the retained ones, their IDs the _Ids bookkeeping, the values the oracle's on the erasing reference"""
    from oracle import ref_retire
    if not ref_retire.have_retire("intended"):
        pytest.skip("oracle/_ref not built")
    retire = ref_retire.retirer(ref)
    scene = bench_scene(40)
    lm = pkg.Lmot(_params(pkg))
    lm.set_track_retirement(True)
    try:
        ref.tracker_reset()
        ids = _Ids()
        for f, (ts, b, v, y) in enumerate(scene):
            out = lm.track_step(b, ts, v, y)
            ref.tracker_step(b, ts, v, y)
            retire()
            ids.step(out["track_manage"])
            if f in (10, 25, 39):
                times = [ts + 1e5, ts + 5e5]
                got = lm.predict_tracks(times)
                assert np.array_equal(got["ids"], np.asarray(ids.ids, np.int64)), f
                _vs_oracle(got, ref.tracker_predict(times), f"retiring step {f}", rows=_pd_tracks(ref.tracker_dump()))
        assert ids.next > len(ids.ids)
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ sequences
def test_sequences_one_launch_equals_per_sequence_and_twins(pkg):
    """S = 8 with eight parameter sets: one lmot_seq_predict_tracks_dev equals, bit for bit, every lmot_seq_predict_tracks(k) and every
    twin context's own-table prediction"""
    seqs = [_ListSeq(k, n_ticks=15) for k in range(8)]
    prms = [dict(std_a=[1.5 + 0.2 * k, 2.0 + 0.1 * k, 3.0], std_las_x=0.15 + 0.01 * k, trans=[[0.9 - 0.01 * k, 0.05 + 0.01 * k, 0.05],
                 [0.05, 0.9, 0.05], [0.05, 0.05, 0.9]]) for k in range(8)]
    ctx = pkg.Lmot(_params(pkg))
    twins = [pkg.Lmot(_params(pkg)) for _ in range(8)]
    try:
        ctx.seq_open(8, ring=4)
        for k in range(8):
            ctx.seq_set_tracker_params(k, **prms[k])
            twins[k].set_tracker_params(**prms[k])
        for f in range(15):
            ts = [s.ts(f) for s in seqs]
            v, y = [s.ego(f)[0] for s in seqs], [s.ego(f)[1] for s in seqs]
            ctx.seq_track([s.lists[f] for s in seqs], ts, v, y)
            for k in range(8):
                twins[k].track_step(seqs[k].lists[f], ts[k], v[k], y[k])
        t_us = np.array([[t + 1e5 * j for j in range(6)] for t in ts])
        import torch
        devs = [_Dev(pkg, 6, 512) for _ in range(8)]
        d_n = torch.zeros(8, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.seq_predict_tracks_dev(t_us, [d.out for d in devs], d_n.data_ptr())
        torch.cuda.synchronize()
        n = d_n.cpu().numpy()
        for k in range(8):
            devs[k].n.copy_(d_n[k:k + 1])
            one = devs[k].host()
            assert len(one["ids"]) == n[k] > 0
            _same(one, ctx.seq_predict_tracks(k, t_us[k]), ("seq", k))
            _same(one, twins[k].predict_tracks(t_us[k]), ("twin", k))
    finally:
        ctx.close()
        for t in twins:
            t.close()


# ------------------------------------------------------------------------------------------------ validation
def test_validation(pkg):
    lm = pkg.Lmot(_params(pkg))
    try:
        f = lambda *a: lm.lib.lmot_predict_tracks(lm.h, *a)
        o, _ = _host_out(pkg, 1, 4)
        t = lambda *v: np.array(v, np.float64).ctypes.data_as(C.c_void_p)
        assert f(t(1e6), 1, C.byref(o)) == pkg.ERR_STATE                      # never stepped
        lm.track_step(boxes_at([[10.0, 0.0]]), 1e6)
        assert f(t(1e6), 1, C.byref(o)) == pkg.OK                             # dt = 0
        for bad in ([np.nan], [np.inf], [1e6 - 1]):
            assert f(t(*bad), 1, C.byref(o)) == pkg.ERR_INVALID, bad
        assert f(t(*([2e6] * 33)), 33, C.byref(o)) == pkg.ERR_INVALID
        assert f(t(2e6), 0, C.byref(o)) == pkg.ERR_INVALID
        o2, _ = _host_out(pkg, 1, 4)
        o2.x = None
        assert f(t(2e6), 1, C.byref(o2)) == pkg.ERR_INVALID
        o3, _ = _host_out(pkg, 1, 4)
        o3.cap = -1
        assert f(t(2e6), 1, C.byref(o3)) == pkg.ERR_INVALID
        assert lm.lib.lmot_seq_predict_tracks(lm.h, 0, t(2e6), 1, C.byref(o)) == pkg.ERR_INVALID          # no open set
        lm.seq_open(2)
        assert lm.lib.lmot_seq_predict_tracks(lm.h, 0, t(2e6), 1, C.byref(o)) == pkg.ERR_STATE            # never stepped
        lm.seq_track([boxes_at([[10.0, 0.0]]), boxes_at([[5.0, 0.0]])], [1e6, 1e6])
        assert lm.lib.lmot_seq_predict_tracks(lm.h, 2, t(2e6), 1, C.byref(o)) == pkg.ERR_INVALID
        assert lm.lib.lmot_seq_predict_tracks(lm.h, 1, t(2e6), 1, C.byref(o)) == pkg.OK
        lm.enable_timing(True)
        assert lm.lib.lmot_seq_predict_tracks(lm.h, 1, t(2e6), 1, C.byref(o)) == pkg.ERR_STATE
        lm.track_step(boxes_at([[10.0, 0.0]]), 1.1e6)
        assert f(t(2e6), 1, C.byref(o)) == pkg.OK                             # timing mode: allowed for the own table
    finally:
        lm.close()


# ------------------------------------------------------------------------------------------------ kernel names
_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
from test_track_retire_gpu import bench_scene
scene = bench_scene(14)
names = {}
for arm in ("never", "predict"):
    c = pkg.Lmot()
    for ts, b, v, y in scene[:10]:
        c.track_step(b, ts, v, y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for ts, b, v, y in scene[10:]:
            c.track_step(b, ts, v, y)
            if arm == "predict":
                c.predict_tracks([ts + 1e5, ts + 2e5])
        torch.cuda.synchronize()
    names[arm] = sorted(e.name for e in prof.events() if e.device_type.name == "CUDA" and "kernel" in e.name.lower())
    c.close()
print("NAMES " + json.dumps(names))
"""


def test_kernel_names():
    """a context that never predicts launches exactly today's kernels; one that predicts shows one predict_tracks_kernel per call"""
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, ROOT, os.path.join(ROOT, "tests")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    import json
    names = json.loads([l for l in r.stdout.splitlines() if l.startswith("NAMES ")][-1][6:])
    never, pred = names["never"], names["predict"]
    assert not any("predict_tracks" in n for n in never)
    assert sum("predict_tracks_kernel" in n for n in pred) == 4
    assert sorted(n for n in pred if "predict_tracks" not in n) == never
