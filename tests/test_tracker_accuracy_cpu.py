"""CPU tests of the per-step accuracy metric (tests/tracker_accuracy.py) and of the extended-precision oracle behind it.

  1. the reference's own double evaluation against the extended-precision restatement (oracle/liboracle_port_hp.so), teacher-forced
     on synth seeds 1, 2 and 5: identical decisions on every step, every float output within 1 ulp, and the reference's error
     distribution pinned (median ~1e-16..1e-15, p99 <= ~1e-13, max ~1e-12 per block) -- the scale the bar is set against;
  2. the yaw-wrap and NaN rules of the block error;
  3. mutations of the reference's output arrays that the bar must catch (one P entry scaled by 1 + 1e-9, K rounded through float,
     the mode probabilities renormalised in float, zPred with 20 mantissa bits cleared) and one it must not (a 2 pi yaw shift).
"""
import numpy as np
import pytest

import tracker_accuracy as ta
from oracle import ref as oracle

OFF = -0.63035 - np.pi / 2          # firstEgoYawOffset_, imm_ukf_jpda.cpp:70
SEEDS = (1, 2, 5)


@pytest.fixture(scope="module")
def hp():
    if not oracle.have_port_hp():
        pytest.skip("oracle/liboracle_port_hp.so not built (make -C oracle port)")
    return oracle.PortOracleHP("intended")


def _boxes_sequence(ref, synth, seed, n_frames=30, n_objects=72):
    seq = []
    for ts, pts in synth.frames(synth.SceneConfig(seed=seed, n_objects=n_objects), n_frames):
        e, _ = ref.ground_remove(pts)
        g, k = ref.component_clustering(e)
        b, _ = ref.box_fitting(e, g, k)
        seq.append((ts, b))
    return seq


def _forced_run(ref, hp, seq, on_step):
    """teacher-forced: before every step after the first, both oracles are loaded from the reference's table"""
    ref.tracker_reset(); hp.tracker_reset()
    prev = None
    for f, (ts, boxes) in enumerate(seq):
        if f > 0:
            state = ref.tracker_dump()
            for o in (ref, hp):
                o.tracker_load(state, 1, prev, 0.0, OFF, OFF, -np.pi / 2)
        a = ref.tracker_step(boxes, ts); da = ref.tracker_dump()
        h = hp.tracker_step(boxes, ts); dh = hp.tracker_dump()
        on_step(f, (a, da), (h, dh))
        prev = ts


@pytest.fixture(scope="module")
def scenes(ref_intended, hp, synth):
    """every teacher-forced step of the three scenes: [(seed, frame, (ref result, ref dump), (hp result, hp dump))]"""
    out = []
    for seed in SEEDS:
        _forced_run(ref_intended, hp, _boxes_sequence(ref_intended, synth, seed),
                    lambda f, r, h, seed=seed: out.append((seed, f, r, h)))
    return out


def test_hp_oracle_is_extended_and_marshalled_as_such(hp):
    assert np.finfo(np.longdouble).nmant == 63
    assert hp.lib.port_real_digits() == 64 and oracle.PortOracle().lib.port_real_digits() == 53
    hp.tracker_reset()
    hp.tracker_step(np.zeros((0, 8, 3), np.float32), 1e5)
    assert hp.tracker_dump().dtype == np.longdouble


def test_reference_error_against_extended_precision(scenes):
    """The reference is the 'evaluation under test' here: its decisions equal hp's on every step, its float outputs are within
    1 ulp, and its blockwise error has the distribution the bar is built on."""
    acc = ta.Accuracy("reference vs extended precision, seeds 1 2 5")
    for seed, f, r, h in scenes:
        acc.step(r, h, r, (seed, f))
    acc.report(label="e_ref")
    kind, e, _ = acc.arrays()
    assert acc.excluded_steps == 0 and acc.steps == 3 * 30
    assert acc.float_worst_ulp <= 1
    assert float((e > ta.CEIL).mean()) <= ta.EXCLUDED_SHARE
    ok = e <= ta.CEIL
    for k in ta.KINDS:
        s = e[(kind == k) & ok]
        assert len(s) > 100, k
        assert np.median(s) < 2e-14 and np.quantile(s, 0.99) < 1e-12 and s.max() < 1e-10, (k, np.median(s), np.quantile(s, 0.99), s.max())
    # hp is not the double port in disguise: most blocks of the filter differ from the reference in the last bits
    for k in ("P", "S", "K"):
        s = e[(kind == k) & ok]
        assert (s > 0).mean() > 0.5, (k, (s > 0).mean())


def test_block_error_wrap_and_nan_rules():
    hpb = np.array([[10.0, 5.0, 1.0, np.pi - 1e-12, 0.1]], np.longdouble)
    got = hpb.astype(np.float64).copy()
    got[0, 3] = (np.pi - 1e-12) - 2 * np.pi                     # the same angle on the other side of +-pi
    assert ta.block_error(got, hpb, yaw=3)[0] < 1e-15
    assert ta.block_error(got, hpb)[0] > 0.5                    # without the wrap rule: a 2 pi error
    got[0, 3] = hpb[0, 3] + 4 * np.pi
    assert ta.block_error(got, hpb, yaw=3)[0] < 1e-15
    nan = np.full((1, 5), np.nan)
    assert ta.block_error(nan, nan.astype(np.longdouble))[0] == 0          # NaN on both sides agrees
    part = hpb.astype(np.float64).copy(); part[0, 1] = np.nan
    assert ta.block_error(part, hpb)[0] == np.inf                          # NaN on one side fails
    assert ta.block_error(hpb.astype(np.float64), part.astype(np.longdouble))[0] == np.inf
    assert not ta.passes(np.array([np.inf]), np.array([0.0]))[0]
    assert ta.block_error(np.zeros((1, 3)), np.zeros((1, 3), np.longdouble))[0] == 0
    assert ta.block_error(np.array([[0.0, 1e-300, 0.0]]), np.zeros((1, 3), np.longdouble))[0] == np.inf
    assert ta.ulp_distance(np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(2.0))) == 1
    assert ta.ulp_distance(np.float32(-0.0), np.float32(0.0)) == 0


def _mutated(scenes, mutate):
    """the reference's arrays, mutated, as the evaluation under test on every step of seed 1 from frame 10 on"""
    acc = ta.Accuracy("mutation")
    for seed, f, (a, da), h in scenes:
        if seed != 1 or f < 10:
            continue
        db = da.copy()
        b = {k: v.copy() for k, v in a.items()}
        mutate(db, b, np.nonzero(da[:, 0] > 0)[0])
        acc.step((a, da), h, (b, db), (seed, f))
    return acc


def _failing_kinds(acc):
    return {f[0] for f in acc.failures()}


def test_mutation_p_entry_scaled(scenes):
    def mutate(db, b, live):
        i = live[len(live) // 2]
        blk = db[i, ta.D_P + 25:ta.D_P + 50]                     # P of the cv model
        blk[np.argmax(np.abs(blk))] *= 1 + 1e-9
    acc = _mutated(scenes, mutate)
    assert _failing_kinds(acc) == {"P"} and len(acc.failures()) == acc.steps


def test_mutation_k_through_float(scenes):
    def mutate(db, b, live):
        db[live, ta.D_K:ta.D_K + 30] = db[live, ta.D_K:ta.D_K + 30].astype(np.float32).astype(np.float64)
    acc = _mutated(scenes, mutate)
    assert _failing_kinds(acc) == {"K"}
    assert len(acc.failures()) >= acc.steps


def test_mutation_mode_prob_renormalised_in_float(scenes):
    def mutate(db, b, live):
        mp = db[live, ta.D_MODE:ta.D_MODE + 3].astype(np.float32)
        db[live, ta.D_MODE:ta.D_MODE + 3] = mp / mp.sum(1, keepdims=True, dtype=np.float32)
    acc = _mutated(scenes, mutate)
    assert _failing_kinds(acc) == {"modeProb"} and len(acc.failures()) >= acc.steps


def test_mutation_zpred_mantissa_cleared(scenes):
    def mutate(db, b, live):
        z = np.ascontiguousarray(db[live, ta.D_ZPRED:ta.D_ZPRED + 6])
        db[live, ta.D_ZPRED:ta.D_ZPRED + 6] = (z.view(np.uint64) & ~np.uint64((1 << 20) - 1)).view(np.float64)
    acc = _mutated(scenes, mutate)
    assert _failing_kinds(acc) == {"zPred"} and len(acc.failures()) >= acc.steps


def test_mutation_yaw_shifted_by_two_pi_passes(scenes):
    def mutate(db, b, live):
        for m in range(4):
            db[live, ta.D_X + 5 * m + 3] += 2 * np.pi
        b["vandyaw"][live, 1] -= 2 * np.pi
    acc = _mutated(scenes, mutate)
    assert acc.steps >= 20 and not acc.failures()
