"""lmot_tracker_params against the reference, without a GPU.

oracle/_ref/libref_tunable.so is libref_intended.so with the tracker's constants read from globals (oracle/tunable.mk).  These tests
check that oracle itself: at its defaults it must be the reference bit for bit, each global must reach the arithmetic it stands for,
and lmot_default_tracker_params must be the reference's values.
"""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hotpath_golden.npz")
OFF = -0.63035 - np.pi / 2           # firstEgoYawOffset_, imm_ukf_jpda.cpp:70

# every field moved alone: to one of the reference's commented alternatives where it keeps one, else to a value the scene reaches
ALTERNATIVES = {
    "gamma_g": 5.99,                                    # imm_ukf_jpda.cpp:31
    "p_g": 0.95,                                        # :32
    "p_d": 0.7,
    "distance_thres": 0.25,                             # :37
    "lifetime_thres": 8,                                # :42
    "bb_yaw_change_thres": 0.01,
    "second_init_v": 1.0,                               # :909 (targetV = 1.)
    "static_lifetime": 3,
    "static_dist": 30.0,
    "std_a": [0.8, 0.8, 5.0],                           # ukf.cpp:53-55
    "std_yawdd": [0.8, 0.8, 3.0],                       # :56-58
    "std_las_x": 0.3,                                   # :92
    "std_las_y": 0.3,                                   # :95
    "trans": [[0.8, 0.1, 0.1], [0.8, 0.1, 0.1], [0.1, 0.1, 0.8]],   # :156-166
    "mode_prob0": [0.6, 0.2, 0.2],
    "p0_diag": [0.5, 0.5, 1.0, 1.0, 1.0],               # :263-267
}


@pytest.fixture(scope="module")
def tunable():
    from oracle import ref_tunable
    if not ref_tunable.have_ref("tunable"):
        pytest.skip("oracle/_ref/libref_tunable.so not built (needs the reference checkout; `make -C oracle -f tunable.mk`)")
    r = ref_tunable.RefTunable()
    yield r
    r.set_tracker_params(None)


@pytest.fixture(scope="module")
def intended():
    from oracle import ref
    if not ref.have_ref("intended"):
        pytest.skip("oracle/_ref not built")
    return ref.RefOracle("intended")


def _golden_scene():
    z = np.load(GOLD)
    return [(float(z[f"ts{i}"]), z[f"boxes_intended{i}"], 0.0, 0.0) for i in range(int(z["n_frames"]))]


_SYNTH = []


def _synth_scene(ref):
    """40 frames of a synthetic scene, boxes from the reference's own detection, with ego motion"""
    if not _SYNTH:
        import importlib
        synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
        for f, (ts, pts) in enumerate(synth.frames(synth.SceneConfig(seed=7, n_objects=48), 40)):
            e, _ = ref.ground_remove(pts)
            g, k = ref.component_clustering(e)
            b, _ = ref.box_fitting(e, g, k)
            _SYNTH.append((ts, b, 2.0 + 0.05 * f, 0.3 + 0.01 * f))
    return _SYNTH


def _run(ref, scene):
    """free-running: per frame the outputs and the table dump"""
    ref.tracker_reset()
    out = []
    for ts, boxes, v, yaw in scene:
        r = ref.tracker_step(boxes, ts, v, yaw)
        out.append((r, ref.tracker_dump()))
    return out


# dump columns compared: all but initMeas_ (180, 181), which the reference leaves uninitialised until a track's second
# initialisation, and distFromInit_ (178), computed from it (two runs of the same library differ there)
DUMP_COLS = np.r_[0:178, 179, 182:236]


def _first_difference(a, b):
    """(frame, what) of the first output or dump row that is not bit-identical, or None"""
    for f, ((ra, da), (rb, db)) in enumerate(zip(a, b)):
        for k in ra:
            if ra[k].shape != rb[k].shape or ra[k].tobytes() != rb[k].tobytes():
                return f, k
        if da.shape != db.shape or da[:, DUMP_COLS].tobytes() != db[:, DUMP_COLS].tobytes():
            return f, "dump"
    return None


def test_tunable_at_defaults_is_the_reference(tunable, intended):
    """Catches a sed patch that changed arithmetic (an operand or an evaluation order) rather than only where a value comes from."""
    tunable.set_tracker_params(None)
    for name, scene in (("golden", _golden_scene()), ("synth", _synth_scene(intended))):
        d = _first_difference(_run(intended, scene), _run(tunable, scene))
        assert d is None, (name, d)


def test_each_global_reaches_the_reference(tunable, intended):
    """Catches a global the patch does not reach (moving it changes nothing), and a test scene that cannot tell a field apart."""
    scene = _synth_scene(intended)
    tunable.set_tracker_params(None)
    base = _run(tunable, scene)
    try:
        for field, val in ALTERNATIVES.items():
            tunable.set_tracker_params({field: val})
            d = _first_difference(base, _run(tunable, scene))
            print(f"{field} = {val}: first difference at frame, output {d}")
            assert d is not None, field
    finally:
        tunable.set_tracker_params(None)


def test_library_defaults_are_the_reference_values(pkg, tunable):
    """Catches a default of lmot_default_tracker_params that drifted from the reference (needs no device)."""
    tunable.set_tracker_params(None)
    lib = pkg.default_tracker_params()
    ref = tunable.get_tracker_params()
    assert set(lib) == set(ref)
    for k in ref:
        assert np.array_equal(np.asarray(lib[k], np.float64), np.asarray(ref[k], np.float64)), (k, lib[k], ref[k])


def test_tracker_params_layout(pkg):
    """Catches a Python structure that disagrees with include/lmot.h's field order (no device, no reference needed)."""
    d = pkg.default_tracker_params()
    assert d["gamma_g"] == 9.22 and d["lifetime_thres"] == 3 and d["static_lifetime"] == 8
    assert d["p0_diag"] == [0.5, 0.5, 3.0, 10.0, 1.0] and d["trans"][0] == [0.9, 0.05, 0.05]
    assert d["std_a"] == [2.0, 2.0, 3.0] and d["std_las_y"] == 0.15 and d["mode_prob0"] == [0.33] * 3
