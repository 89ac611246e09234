"""Per-step accuracy of the CUDA tracker against an extended-precision evaluation of the reference (tests/tracker_accuracy.py).

Every case is teacher-forced: before each step the CUDA table, the reference (oracle/_ref) and its restatement in long double
(oracle/liboracle_port_hp.so, `hp`) are loaded with the reference's table, all three step the same boxes, and each block of every
live track -- x and P per model, the mode probabilities, zPred, S and K per model, (v, yaw) -- must satisfy
    e_cuda <= max(C * e_ref, F),  e_cuda <= 1e-9
where e is the block's distance from hp relative to its largest entry (C = 16, F = 2^-40: see tracker_accuracy.py).  Each test
prints the distributions of e_cuda and e_cuda / e_ref per block kind, the excluded counts and the worst block: the accuracy
headroom a change of tracker.cu has left.  The 1e-4 bars of test_tracker_gpu and friends stay as they are for free-running runs.

  a. synth scenes (seeds 1, 2, 5; seed 5 again with a moving ego) through lmot_track_step
  b. the benchmark's scene, 100 frames
  c. every size regime of test_tracker_regimes_gpu (its scene builders)
  d. the 1024-track x 256-detection stress step
  e. lmot_seq_track with 8 tables in one tick, each forced from its own reference table
  f. lmot_predict_tracks (predict_tracks_kernel) against port_tracker_predict at test_track_predict_gpu's horizons
"""
import numpy as np
import pytest

import tracker_accuracy as ta
from test_tracker_regimes_gpu import (STEP_US, _churn_scene, _crowd_scene, _long_table, _mature, _overlap_frames,
                                      _second_init_scene, boxes_at, lattice)

pytestmark = pytest.mark.gpu

OFF = -0.63035 - np.pi / 2          # firstEgoYawOffset_, imm_ukf_jpda.cpp:70
STILL = (0.0, OFF, OFF, -np.pi / 2)  # (ego_velo, ego_yaw, ego_pre_yaw, ego_point_yaw) of a load with a still ego
AFTER = (0.0, 1.0, 5e4, 1e5, 5e5, 1e6, 3e6, 1e7)   # test_track_predict_gpu's horizons (us after the last step)


@pytest.fixture(scope="module")
def hp():
    from oracle import ref as oracle
    if not oracle.have_port_hp():
        pytest.skip("oracle/liboracle_port_hp.so not built (make -C oracle port)")
    return oracle.PortOracleHP("intended")


def _ego_load(v, yaw):
    """what the reference's table holds after a step with ego (v, yaw): the next step's diffYaw is measured from it"""
    return (v, yaw + OFF, yaw + OFF, -np.pi / 2)


class _Cuda:
    """the context's own CUDA track table"""

    def __init__(self, ctx):
        self.ctx = ctx

    def reset(self):
        self.ctx.tracker_reset()

    def load(self, state, ts, ego):
        self.ctx.tracker_load(state, 1, ts, *ego)

    def step(self, boxes, ts, v, yaw):
        return self.ctx.track_step(boxes, ts, v, yaw)

    def dump(self):
        return self.ctx.tracker_dump()


def forced_run(ref, hp, cuda, acc, frames, start=None, ego=None, label=""):
    """frames: [(ts, boxes)]; start: (table, ts) loaded before the first step (default: the first step follows a reset);
    ego: f -> (v_gps, yaw_gps).  Every step starts from the reference's table.  -> the reference's last table"""
    ego = ego or (lambda f: (0.0, 0.0))
    if start is None:
        ref.tracker_reset(); hp.tracker_reset(); cuda.reset()
        state, prev, load = None, None, None
    else:
        (state, prev), load = start, STILL
    for f, (ts, boxes) in enumerate(frames):
        if state is not None:
            for o in (ref, hp):
                o.tracker_load(state, 1, prev, *load)
            cuda.load(state, prev, load)
        v, yaw = ego(f)
        a = ref.tracker_step(boxes, ts, v, yaw); da = ref.tracker_dump()
        h = hp.tracker_step(boxes, ts, v, yaw); dh = hp.tracker_dump()
        b = cuda.step(boxes, ts, v, yaw); db = cuda.dump()
        acc.step((a, da), (h, dh), (b, db), (label, f))
        state, prev, load = da, ts, _ego_load(v, yaw)
    return state


def _stamped(frames, t0=0.0):
    return [(t0 + (f + 1) * STEP_US, b) for f, b in enumerate(frames)]


def _detections(ref, synth, cfg, n_frames):
    out = []
    for ts, pts in synth.frames(cfg, n_frames):
        e, _ = ref.ground_remove(pts)
        g, k = ref.component_clustering(e)
        b, _ = ref.box_fitting(e, g, k)
        out.append((ts, b))
    return out


# ------------------------------------------------------------------------------------------------ a. synth scenes
@pytest.mark.parametrize("seed,moving", [(1, False), (2, False), (5, False), (5, True)], ids=["seed1", "seed2", "seed5", "seed5_ego"])
def test_synth_scenes(lm, ref_intended, hp, synth, seed, moving):
    acc = ta.Accuracy(f"synth seed {seed}{' moving ego' if moving else ''}, 30 frames")
    frames = _detections(ref_intended, synth, synth.SceneConfig(seed=seed, n_objects=72), 30)
    ego = (lambda f: (3.0 + 0.1 * f, 0.02 * f)) if moving else None
    forced_run(ref_intended, hp, _Cuda(lm), acc, frames, ego=ego, label=f"seed{seed}")
    acc.check()


# ------------------------------------------------------------------------------------------------ b. bench scene
def test_bench_scene_100_frames(lm, ref_intended, hp, synth):
    """One step is excluded: at frame 42 the secondInit track 177 (trackNum 1) dies in the reference and advances to 2 in the
    extended evaluation.  The double restatement (oracle/port) decides as the reference does, so the decision turns on double
    rounding; the CUDA step is held to the reference's integers on it like on every other step (test_tracker_gpu)."""
    acc = ta.Accuracy("bench scene (150 objects, 3.8 m lattice, 65 % pedestrians), 100 frames")
    cfg = synth.SceneConfig(n_objects=150, lattice_pitch=3.8, ped_fraction=0.65, seed=1)
    last = forced_run(ref_intended, hp, _Cuda(lm), acc, _detections(ref_intended, synth, cfg, 100), label="bench")
    assert (last[:, 0] > 0).sum() >= 40
    acc.check(max_excluded_steps=1)


# ------------------------------------------------------------------------------------------------ c. size regimes
@pytest.mark.parametrize("big", [False, True], ids=["M<=512", "M>512"])
def test_regime_crowded_gates(lm, ref_intended, hp, big):
    """more than 32 gated boxes per track; with big, more than 512 boxes per step"""
    acc = ta.Accuracy(f"crowded gates, M {'>' if big else '<='} 512")
    mature, steps = _crowd_scene(3, 12 if big else 6, (1024, 800, 1024, 700) if big else (0, 0, 0, 0), 4)
    forced_run(ref_intended, hp, _Cuda(lm), acc, _stamped(mature + steps), label="crowd")
    acc.check()


def test_regime_second_init_crowd(lm, ref_intended, hp):
    acc = ta.Accuracy("secondInit crowds")
    forced_run(ref_intended, hp, _Cuda(lm), acc, _stamped(_second_init_scene(5)), label="second_init")
    acc.check()


@pytest.mark.parametrize("n", [256, 257, 512, 513])
def test_regime_tc_width(lm, ref_intended, hp, n):
    """256 / 257 / 512 / 513 active tracks: both sides of spawn_output_kernel's one-track-per-thread widths"""
    acc = ta.Accuracy(f"{n} active tracks")
    rng = np.random.default_rng(n)
    last = forced_run(ref_intended, hp, _Cuda(lm), acc, _stamped(_mature(rng, lattice(23, 23, 8.0)[:n], 9)), label=f"tc{n}")
    assert (last[:, 0] > 0).sum() == n
    acc.check()


def test_regime_grid_stride(pkg, ref_intended, hp, monkeypatch):
    """8 CTAs for the per-track kernels: every CTA walks dozens of tracks of mixed kinds"""
    monkeypatch.setenv("LMOT_TRK_CTAS", "8")
    acc = ta.Accuracy("grid stride, 8 CTAs")
    ctx = pkg.Lmot()
    try:
        mature, steps = _crowd_scene(4, 12, (1024, 800, 1024, 700), 4)
        forced_run(ref_intended, hp, _Cuda(ctx), acc, _stamped(mature + steps), label="crowd")
        last = forced_run(ref_intended, hp, _Cuda(ctx), acc, _stamped(_churn_scene(6, 16)), label="churn")
        assert (last[:, 0] > 0).sum() >= 160
    finally:
        ctx.close()
    acc.check()


def test_regime_long_table_moving_ego(pkg, ref_intended, hp):
    """> 4600 rows, nearly all dead, beyond the unrolled 1024..4096-row copies, with a moving ego"""
    acc = ta.Accuracy("long table, moving ego")
    table, pos, ts = _long_table(ref_intended)
    assert len(table) > 4096
    rng = np.random.default_rng(9)
    p = pkg.default_params()
    p.max_tracks = 8192
    ctx = pkg.Lmot(p)
    try:
        frames = [(ts + (f + 1) * STEP_US, boxes_at(pos + rng.normal(0, 0.02, pos.shape))) for f in range(12)]
        forced_run(ref_intended, hp, _Cuda(ctx), acc, frames, start=(table, ts), ego=lambda f: (3.0 + 0.1 * f, 0.02 * (f + 1)),
                   label="long")
    finally:
        ctx.close()
    acc.check()


@pytest.mark.parametrize("nx", [16, 20])
def test_regime_overlapping_visible_boxes(lm, ref_intended, hp, nx):
    acc = ta.Accuracy(f"overlapping visible boxes, {nx} x {nx} tracks")
    forced_run(ref_intended, hp, _Cuda(lm), acc, _stamped(_overlap_frames(nx, 10)), label=f"overlap{nx}")
    acc.check()


# ------------------------------------------------------------------------------------------------ d. stress step
def test_stress_1024_tracks_256_detections(lm, ref_intended, hp):
    acc = ta.Accuracy("1024 tracks x 256 detections")
    rng = np.random.default_rng(0)
    pos = lattice(32, 32, 8.0, origin=(-124.0, -124.0))
    ref_intended.tracker_reset()
    ts = 0.0
    for _ in range(8):
        ts += STEP_US
        ref_intended.tracker_step(boxes_at(pos + rng.normal(0, 0.02, pos.shape)), ts)
    state = ref_intended.tracker_dump()
    assert (state[:, 0] == 5).sum() >= 1000
    sel = np.sort(rng.choice(len(pos), 256, replace=False))
    det = boxes_at(pos[sel] + rng.normal(0, 0.15, (256, 2)))
    forced_run(ref_intended, hp, _Cuda(lm), acc, [(ts + STEP_US, det)], start=(state, ts), label="stress")
    acc.check()


# ------------------------------------------------------------------------------------------------ e. sequence tables
def test_seq_track_eight_tables(pkg, ref_intended, hp):
    """one lmot_seq_track tick steps 8 tables; each is loaded from its own reference table (lmot_seq_tracker_load) before the tick
    and compared with the reference and hp stepped from that table alone"""
    from test_seq_track_gpu import _ListSeq, _params
    S, n_ticks = 8, 12
    ref = ref_intended
    acc = ta.Accuracy("lmot_seq_track, 8 tables")
    seqs = [_ListSeq(k, n_ticks=n_ticks, seed=700, n_obj=12 + 4 * k) for k in range(S)]
    tables = [None] * S
    ctx = pkg.Lmot(_params(pkg, 0, max_tracks=4096))
    try:
        ctx.seq_open(S, ring=2)
        for f in range(n_ticks):
            want = []
            for k, sq in enumerate(seqs):
                v, yaw = sq.ego(f)
                if tables[k] is None:
                    for o in (ref, hp):
                        o.tracker_reset()
                else:
                    ego = _ego_load(*sq.ego(f - 1))
                    for o in (ref, hp):
                        o.tracker_load(tables[k], 1, sq.ts(f - 1), *ego)
                    ctx.seq_tracker_load(k, tables[k], 1, sq.ts(f - 1), *ego)
                a = ref.tracker_step(sq.lists[f], sq.ts(f), v, yaw); da = ref.tracker_dump()
                h = hp.tracker_step(sq.lists[f], sq.ts(f), v, yaw); dh = hp.tracker_dump()
                want.append(((a, da), (h, dh)))
            got = ctx.seq_track([sq.lists[f] for sq in seqs], [sq.ts(f) for sq in seqs], [sq.ego(f)[0] for sq in seqs],
                                [sq.ego(f)[1] for sq in seqs])
            for k in range(S):
                acc.step(want[k][0], want[k][1], (got[k], ctx.seq_tracker_dump(k)), (f"seq{k}", f))
                tables[k] = want[k][0][1]
        assert all((t[:, 0] > 0).sum() >= 5 for t in tables), [int((t[:, 0] > 0).sum()) for t in tables]
    finally:
        ctx.close()
    acc.check()


# ------------------------------------------------------------------------------------------------ f. prediction
@pytest.mark.parametrize("table", ["bench20", "bench60", "stress1024"])
def test_predict_tracks(pkg, ref_intended, hp, table):
    """x, P, mode_prob, gate_z and gate_S of every valid row at ts_last + 0 .. 10 s"""
    from oracle import ref_predict
    from test_seq_track_gpu import _params
    from test_track_predict_gpu import _lattice_table, _run_ref
    from test_track_retire_gpu import bench_scene
    if not ref_predict.have_predict("intended"):
        pytest.skip("oracle/_ref/libref_predict_intended.so not built")
    ref = ref_intended
    predict = ref_predict.predictor(ref)
    if table == "stress1024":
        dumps, ts = _lattice_table(ref)
    else:
        ts = _run_ref(ref, bench_scene(int(table[5:])))
        dumps = ref.tracker_dump()
    acc = ta.Accuracy(f"predict_tracks, {table}")
    lm = pkg.Lmot(_params(pkg, max_tracks=4096))
    try:
        for o in (ref, hp, lm):
            o.tracker_load(dumps, 1, ts, *STILL)
        times = [ts + d for d in AFTER]
        got = lm.predict_tracks(times, cap=len(dumps))
        acc.predict(predict(times), hp.tracker_predict(times), got, table)
    finally:
        lm.close()
    acc.check()
