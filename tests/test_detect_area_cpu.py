"""Detection areas without a device: lmot_detect_area_mask against the NumPy restatement of the definition, the validation of areas, and
the reference's own clustering and box fitting on E_area of a cluttered roadside scene."""
import math

import numpy as np
import pytest

from detect_area_scenes import CORRIDOR, area_filter, cluttered_frames, mask_ref, near_clutter, rect

f32 = np.float32


def _pose(yaw, tx, ty):
    c, s = math.cos(yaw), math.sin(yaw)
    if yaw in (0.0, math.pi / 2, -math.pi / 2, math.pi):    # the exact quarter turns
        c, s = round(c), round(s)
    return np.array([[c, -s, 0, tx], [s, c, 0, ty], [0, 0, 1, 1.5]], f32)


# centre abscissae of roi 50 are -24.9 + 0.2 k: vertices placed on them exercise the half-open straddle test; vertical edges never straddle
CENTRE = -24.9 + 0.2 * 40
POLYGONS = {
    "convex": [np.array([[-12.0, -3.0], [4.0, -9.5], [14.5, 2.0], [3.3, 11.7], [-9.9, 8.0]])],
    "concave": [np.array([[-15.0, -15.0], [15.0, -15.0], [15.0, 15.0], [0.1, 0.3], [-15.0, 15.0]])],
    "holed": [rect(-20.0, -20.0, 20.0, 20.0), rect(-5.0, -5.0, 5.0, 5.0), rect(-2.0, -2.0, 2.0, 2.0)],
    "self_intersecting": [np.array([[-10.0, -10.0], [10.0, 10.0], [10.0, -10.0], [-10.0, 10.0]])],
    "raster": [rect(x, y, x + 2.0, y + 2.0) for x in range(-24, 24, 6) for y in range(-24, 24, 8)],
    "on_centres": [np.array([[CENTRE, -7.0], [CENTRE + 3.0, -7.0], [CENTRE + 3.0, 6.0], [CENTRE, 6.0], [CENTRE, 1.3]])],
    "beyond_grid": [rect(-40.0, -3.0, 60.0, 3.0)],
}
POSES = {"identity": None, "yaw0_offset": _pose(0.0, 1.2, -0.7), "yaw+90": _pose(math.pi / 2, -2.0, 0.5),
         "yaw-90": _pose(-math.pi / 2, 0.3, 3.1), "yaw180": _pose(math.pi, 4.0, -1.0), "yaw30": _pose(math.pi / 6, -1.1, 2.2)}


@pytest.mark.parametrize("poly", sorted(POLYGONS))
@pytest.mark.parametrize("pose", sorted(POSES))
@pytest.mark.parametrize("roi", [50.0, 30.0])
@pytest.mark.parametrize("keep_outside", [False, True])
def test_host_mask_equals_definition(pkg, poly, pose, roi, keep_outside):
    got = pkg.detect_area_mask(POLYGONS[poly], keep_outside, POSES[pose], roi)
    want = mask_ref(POLYGONS[poly], keep_outside, POSES[pose], roi)
    assert np.array_equal(got, want)
    assert not (got[:, 7] >> np.uint32(26)).any()           # bits above 250 are 0


def test_host_mask_shapes(pkg):
    """the identity pose keeps the vertices exactly: a rectangle on cell edges is exactly its cells; keep_outside is the complement"""
    m = pkg.detect_area_mask([rect(-10.0, -4.0, 10.0, 4.0)])
    bits = np.unpackbits(m.view(np.uint8), bitorder="little").reshape(250, 256)[:, :250]
    assert bits.sum() == 100 * 40 and bits[75:175, 105:145].all()
    o = pkg.detect_area_mask([rect(-10.0, -4.0, 10.0, 4.0)], keep_outside=True)
    ob = np.unpackbits(o.view(np.uint8), bitorder="little").reshape(250, 256)[:, :250]
    assert np.array_equal(ob, 1 - bits)


@pytest.mark.parametrize("case", ["rings_neg", "rings_65", "short_ring", "too_many", "nan", "inf", "keep_2", "null_xy", "null_len"])
def test_validation(pkg, case):
    import ctypes as C
    lib = pkg.load_library()
    sq = rect(-1.0, -1.0, 1.0, 1.0)
    rings, ko = [sq], 0
    if case == "short_ring":
        rings = [sq, sq[:2]]
    elif case == "too_many":
        rings = [np.zeros((513, 2)), np.ones((512, 2))]
    elif case == "nan":
        rings = [np.where(np.arange(8).reshape(4, 2) == 5, np.nan, sq)]
    elif case == "inf":
        rings = [np.where(np.arange(8).reshape(4, 2) == 2, -np.inf, sq)]
    elif case == "keep_2":
        ko = 2
    a, keep = pkg._area(rings, ko)
    if case == "rings_neg":
        a.n_rings = -1
    elif case == "rings_65":
        rr = [sq] * 65
        a, keep = pkg._area(rr)
    elif case == "null_xy":
        a.xy = None
    elif case == "null_len":
        a.ring_len = None
    fn = lib.lmot_detect_area_mask
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    out = np.zeros((250, 8), np.uint32)
    assert fn(C.cast(C.byref(a), C.c_void_p), None, 50.0, out.ctypes.data) == pkg.ERR_INVALID


def test_validation_limits_are_inclusive(pkg):
    """64 rings and 1024 vertices are allowed; a bad roi or mount is not; the setters need a context (NULL: invalid)"""
    assert pkg.detect_area_mask([rect(-1.0, -1.0, 1.0, 1.0)] * 64).any() is not None
    pkg.detect_area_mask([np.stack([np.cos(t), np.sin(t)], 1) * 10 for t in [np.linspace(0, 6.2, 1024)]])
    for roi in (0.0, -5.0, float("nan")):
        with pytest.raises(pkg.LmotError):
            pkg.detect_area_mask([rect(-1.0, -1.0, 1.0, 1.0)], roi_m=roi)
    with pytest.raises(pkg.LmotError):
        pkg.detect_area_mask([rect(-1.0, -1.0, 1.0, 1.0)], mount=np.array([[2, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], f32))
    lib = pkg.load_library()
    assert lib.lmot_set_detect_area(None, None) == pkg.ERR_INVALID
    assert lib.lmot_seq_set_detect_area(None, 0, None) == pkg.ERR_INVALID


def test_clutter_dropped_by_the_reference_on_e_area(ref_intended, synth, pkg):
    """roadside poles and hedges outside the road corridor give boxes on the whole elevated cloud and none on E_area"""
    ref = ref_intended
    mask = pkg.detect_area_mask(CORRIDOR)
    boxed_clutter = kept = 0
    for ts, pts in cluttered_frames(synth, 3):
        e, _ = ref.ground_remove(pts)
        grid, k = ref.component_clustering(e)
        b, _ = ref.box_fitting(e, grid, k)
        boxed_clutter += int(near_clutter(b).sum())
        ea = area_filter(e, mask)
        grid, k = ref.component_clustering(ea)
        ba, _ = ref.box_fitting(ea, grid, k)
        assert not near_clutter(ba).any()
        assert (np.abs(ba.reshape(-1, 8, 3)[:, :4, 1].mean(1)) < 8.0).all()
        kept += len(ba)
    assert boxed_clutter >= 10, boxed_clutter
    assert kept > 0
