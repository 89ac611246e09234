"""Track prediction (lmot_predict_tracks) oracle against the reference, without a GPU.

The oracle of prediction is ref_tracker_predict (oracle/ref_predict.cpp, bound by oracle/ref_predict.py): every row of the reference's
own table, copied, through the reference's ProcessIMMUKF(dt), findMaxZandS and PostProcessIMMUKF({1, 1, 1}).  These tests check that
oracle: it leaves the reference's table alone, it agrees with the reference's own step where a step brings no information, and its
tunable build reads the tracker constants a test sets.
"""
import numpy as np
import pytest

from test_track_retire_cpu import bench_scene

D_X = 4
TIMES_AFTER = (0.0, 1.0, 5e4, 1e5, 5e5, 1e6, 3e6, 1e7)


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


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


def _run(r, scene):
    r.tracker_reset()
    for ts, b, v, y in scene:
        r.tracker_step(b, ts, v, y)
    return scene[-1][0]


def test_predict_leaves_the_reference_table_untouched(ref):
    """the helper works on copies: a dump before equals a dump after, bit for bit"""
    ts = _run(ref, bench_scene(30))
    before = ref.tracker_dump()
    p = ref.tracker_predict([ts + d for d in TIMES_AFTER])
    assert p["flags"].shape == (len(TIMES_AFTER), len(before))
    assert np.array_equal(_bits(before), _bits(ref.tracker_dump()))
    assert (p["flags"] == 1).any() and (p["flags"] == 2).any()


@pytest.mark.parametrize("n_steps", [20, 60])
def test_oracle_equals_an_empty_step(ref, n_steps):
    """tracks at trackManage 5..9 that survive an empty-list step at t: their x_merge_ equals the oracle's merged mean at t (to 1e-12
    relative).  Without measurements filterPDA leaves the model means untouched and gives the three models equal likelihoods."""
    scene = bench_scene(n_steps)
    ts = _run(ref, scene)
    before = ref.tracker_dump()
    t = ts + 1e5
    p = ref.tracker_predict([t])
    sel = (before[:, 0] >= 5) & (before[:, 0] <= 9)
    ref.tracker_step(np.zeros((0, 8, 3), np.float32), t, scene[-1][2], scene[-1][3])
    after = ref.tracker_dump()
    keep = sel & (after[: len(before), 0] != 0)
    assert keep.sum() >= 5, int(keep.sum())
    want = after[: len(before)][keep][:, D_X:D_X + 5]
    got = p["x"][0][keep]
    scale = np.maximum(np.abs(want), 1e-9)
    err = np.abs(got - want) / scale
    print(f"{int(keep.sum())} surviving tracks, worst relative x error {err.max():.3g}")
    assert err.max() <= 1e-12
    assert np.all(p["flags"][0][keep] & 1)


def test_tunable_at_defaults_equals_intended_and_follows_its_globals(ref, ref_tunable):
    scene = bench_scene(30)
    times = [scene[-1][0] + d for d in TIMES_AFTER]
    _run(ref, scene)
    want = ref.tracker_predict(times)
    ref_tunable.set_tracker_params(None)
    _run(ref_tunable, scene)
    got = ref_tunable.tracker_predict(times)
    for k in want:
        assert np.array_equal(_bits(want[k]), _bits(got[k])), k
    # the same rows, loaded into UKFs constructed with moved constants (ref_tracker_load builds every row anew)
    dumps = ref_tunable.tracker_dump()
    for change in (dict(std_a=[1.0, 1.5, 4.0]), dict(trans=[[0.8, 0.1, 0.1], [0.1, 0.8, 0.1], [0.1, 0.1, 0.8]])):
        ref_tunable.set_tracker_params(change)
        ref_tunable.tracker_load(dumps, 1, scene[-1][0])
        moved = ref_tunable.tracker_predict(times)
        valid = ((want["flags"] & 1) & (moved["flags"] & 1)).astype(bool)
        assert valid.any()
        assert not np.array_equal(want["P"][valid], moved["P"][valid]), change
    ref_tunable.set_tracker_params(None)
