"""Per-sequence detection parameters (lmot_detect_params), the parts that need no device: the defaults, the reference values they stand
for, the rejections that come before any sequence set exists, and the oracle with the reference's two detection literals as globals.

oracle/_ref/libref_detect_tunable.so (oracle/detect_tunable.mk) is libref_intended.so with `hGround + 0.25` (ground_removal.cpp:239)
and `numPoints < 30` (box_fitting.cpp:100) read from globals.  At its defaults it must be the reference bit for bit, and each of the
two globals must reach an output.
"""
import ctypes as C
import os

import numpy as np
import pytest

f32 = np.float32

# lmot_detect_params field -> the reference's mutable global of the same role (groundremove/ground_removal.cpp,
# cluster/component_clustering.cpp, cluster/box_fitting.cpp); ground_tolerance and min_cluster_points are literals there
REF_GLOBALS = dict(r_min="rMin", r_max="rMax", t_hmin="tHmin", t_hmax="tHmax", t_hdiff="tHDiff", h_sensor="hSeonsor", roi_m="roiM",
                   ram_points="ramPoints", l_slope_dist="lSlopeDist", l_num_points="lnumPoints", sensor_height="sensorHeight",
                   t_height_min="tHeightMin", t_height_max="tHeightMax", t_width_min="tWidthMin", t_width_max="tWidthMax",
                   t_len_min="tLenMin", t_len_max="tLenMax", t_area_max="tAreaMax", t_ratio_min="tRatioMin", t_ratio_max="tRatioMax",
                   min_len_ratio="minLenRatio", t_pt_per_m3="tPtPerM3")
INT_FIELDS = {"ram_points", "l_slope_dist", "l_num_points"}


def test_defaults_are_lmot_params_detection_fields(pkg):
    d = pkg.default_detect_params()
    p = pkg.default_params()
    for name, _ in pkg.DetectParams._fields_:
        assert d[name] == getattr(p, name), name
    # a context's parameters: its own detection fields, whatever they are
    p.r_max = 60.0; p.roi_m = 30.0; p.ram_points = 300; p.min_cluster_points = 12; p.rule_filter = pkg.RULE_GCC13_O2_COMPAT
    d = pkg.default_detect_params(p)
    assert (d["r_max"], d["roi_m"], d["ram_points"], d["min_cluster_points"], d["rule_filter"]) == (60.0, 30.0, 300, 12, 1)
    assert d["ground_tolerance"] == 0.25


def test_defaults_equal_the_reference_globals(pkg, ref_intended):
    d = pkg.default_detect_params()
    for field, name in REF_GLOBALS.items():
        typ = C.c_int if field in INT_FIELDS else C.c_float
        assert typ.in_dll(ref_intended.lib, name).value == d[field], (field, name)
    # picScale is a dynamic initialiser of roiM (box_fitting.cpp:18): the library evaluates 900 / roi_m in float as well
    assert C.c_float.in_dll(ref_intended.lib, "picScale").value == float(f32(900) / f32(d["roi_m"]))
    assert d["ground_tolerance"] == 0.25 and d["min_cluster_points"] == 30      # the literals of ground_removal.cpp:239, box_fitting.cpp:100


def test_validation_without_a_device(pkg):
    lib = pkg.load_library()
    d = pkg.DetectParams()
    assert lib.lmot_default_detect_params(None, C.byref(d)) == pkg.OK
    assert lib.lmot_default_detect_params(None, None) == pkg.ERR_INVALID
    assert lib.lmot_seq_set_detect_params(None, 0, C.byref(d)) == pkg.ERR_INVALID
    assert lib.lmot_seq_set_detect_params(None, 0, None) == pkg.ERR_INVALID
    assert lib.lmot_seq_get_detect_params(None, 0, C.byref(d)) == pkg.ERR_INVALID
    with pytest.raises(ValueError):
        pkg._detect_params(pkg.default_detect_params(), {"no_such_field": 1})


def test_header_declares_the_new_calls(pkg):
    src = open(os.path.join(os.path.dirname(pkg.__file__), "..", "include", "lmot.h")).read()
    for name in ("lmot_default_detect_params", "lmot_seq_set_detect_params", "lmot_seq_get_detect_params"):
        assert name + "(" in src and name in pkg.ABI_SYMBOLS
    assert f"#define LMOT_MAX_RAM_POINTS {pkg.MAX_RAM_POINTS}" in src


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hotpath_golden.npz")


@pytest.fixture(scope="module")
def detect_tunable():
    from oracle import ref_detect_tunable
    if not ref_detect_tunable.have_ref("detect_tunable"):
        pytest.skip("oracle/_ref/libref_detect_tunable.so not built (needs the reference checkout; `make -C oracle -f detect_tunable.mk`)")
    return ref_detect_tunable.RefDetectTunable()


def _golden_frames():
    z = np.load(GOLD)
    return [(float(z[f"ts{i}"]), z[f"pts{i}"]) for i in range(int(z["n_frames"]))]


def _detect(ref, pts):
    e, g = ref.ground_remove(pts)
    grid, k = ref.component_clustering(e)
    boxes, markers = ref.box_fitting(e, grid, k)
    return e, g, grid, k, boxes, markers


def _u(a):
    a = np.ascontiguousarray(a)
    return a.view(f"u{a.dtype.itemsize}")


def test_detect_tunable_defaults_are_the_reference(pkg, detect_tunable, ref_intended):
    """At its defaults the patched build is libref_intended bit for bit on the golden scene: clouds, label grid, boxes, markers and
    the tracker on those boxes -- and its two globals hold the literals, which are lmot_default_detect_params' values."""
    d = pkg.default_detect_params()
    assert detect_tunable.var("ground_tolerance").value == 0.25 == d["ground_tolerance"]
    assert detect_tunable.var("min_cluster_points").value == 30 == d["min_cluster_points"]
    detect_tunable.tracker_reset(); ref_intended.tracker_reset()
    for f, (ts, pts) in enumerate(_golden_frames()):
        a, b = _detect(detect_tunable, pts), _detect(ref_intended, pts)
        for x, y in zip(a, b):
            if isinstance(x, np.ndarray):
                assert x.shape == y.shape and np.array_equal(_u(x), _u(y)), f
            else:
                assert x == y, f
        ta, tb = detect_tunable.tracker_step(a[4], ts), ref_intended.tracker_step(b[4], ts)
        for key in ("targets", "vandyaw", "track_manage", "vis_bb"):
            assert np.array_equal(_u(ta[key]), _u(tb[key])), (f, key)


def test_each_detect_global_reaches_an_output(detect_tunable):
    """Each global, moved alone, changes an output of the golden scene; back at its default, the output is the default one again
    (catches a pattern that patched something else, or a global the code never reads)."""
    frames = _golden_frames()
    base = [_detect(detect_tunable, pts) for _, pts in frames]
    with detect_tunable.detect_params(dict(ground_tolerance=0.6)):
        moved = [_detect(detect_tunable, pts) for _, pts in frames]
    assert any(len(m[1]) > len(b[1]) for m, b in zip(moved, base)), "ground_tolerance 0.6 labelled no further point ground"
    with detect_tunable.detect_params(dict(min_cluster_points=200)):
        moved = [_detect(detect_tunable, pts) for _, pts in frames]
    assert any(len(m[4]) < len(b[4]) for m, b in zip(moved, base)), "min_cluster_points 200 removed no box"
    with detect_tunable.detect_params(dict(min_cluster_points=5)):
        moved = [_detect(detect_tunable, pts) for _, pts in frames]
    assert any(len(m[4]) > len(b[4]) for m, b in zip(moved, base)), "min_cluster_points 5 added no box"
    again = [_detect(detect_tunable, pts) for _, pts in frames]
    for a, b in zip(again, base):
        assert len(a[1]) == len(b[1]) and np.array_equal(_u(a[4]), _u(b[4]))
