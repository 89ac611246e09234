"""Background subtraction of DESIGN.md §6n without a device: the NumPy restatement of the cell map, the freeze rule and the filter
(tests/background_scenes.py) on hand-built cases and against a brute-force freeze, and the reference's chain on the stationary-sensor
scene with the proposed defaults, pinned for seed 5."""
import math

import numpy as np
import pytest

import background_scenes as bs

f32 = np.float32


def _cell(x, y, z, **cfg):
    c, r = bs.cells(np.array([[x, y, z]], f32), **dict(bs.DEFAULTS, **cfg))
    return int(c[0]), r[0]


def test_cells_of_hand_built_points():
    # straight ahead, level: az = 0 -> column cols / 2; el = 0 -> row floor(25 / 28 * 64) = 57
    c, r = _cell(10.0, 0.0, 0.0)
    assert c == 57 * 1800 + 900 and r == f32(10.0)
    # r is the 3-D range, (x * x + y * y) + z * z in float
    _, r = _cell(3.0, 4.0, 12.0, elev_max_deg=80.0)
    assert r == f32(13.0)
    # az = +pi (y = +0, x < 0) lands on cols and is clamped to the last column; y = -0 gives -pi, the first column
    assert _cell(-5.0, 0.0, -0.5)[0] % 1800 == 1799
    assert _cell(-5.0, -0.0, -0.5)[0] % 1800 == 0
    # above and below the window: no cell; the window's lower edge is in, its upper edge is out
    assert _cell(10.0, 0.0, 5.0)[0] == -1 and _cell(10.0, 0.0, -10.0)[0] == -1
    lo = math.radians(-25.0)
    assert _cell(math.cos(lo) * 10, 0.0, math.sin(lo) * 9.99)[0] // 1800 == 0
    assert _cell(math.cos(lo) * 10, 0.0, math.sin(lo) * 10.01)[0] == -1
    hi = math.radians(3.0)
    assert _cell(math.cos(hi) * 10, 0.0, math.sin(hi) * 9.99)[0] // 1800 == 63
    assert _cell(math.cos(hi) * 10, 0.0, math.sin(hi) * 10.01)[0] == -1
    # zero range: az = atan2f(0, 0) = 0, el = 0, a cell of range 0
    c, r = _cell(0.0, 0.0, 0.0)
    assert c == 57 * 1800 + 900 and r == 0.0


def test_cells_step_by_step_in_float():
    # the restatement equals a scalar evaluation of every step in float32 on random clouds
    rng = np.random.default_rng(3)
    p = rng.uniform(-40, 40, (3000, 3)).astype(f32)
    p[:, 2] = rng.uniform(-12, 3, 3000).astype(f32)
    for cfg in [{}, dict(rows=128, cols=4096, elev_min_deg=-30.0, elev_max_deg=11.0), dict(rows=1, cols=1)]:
        c = dict(bs.DEFAULTS, **cfg)
        got, r = bs.cells(p, **c)
        lo, hi, span = bs.window(**c)
        for i in range(0, 3000, 7):
            x, y, z = (f32(v) for v in p[i])
            s = f32(x * x) + f32(y * y)
            rxy = np.sqrt(f32(s))
            az, el = np.arctan2(y, x), np.arctan2(z, rxy)
            col = min(int(np.floor(f32(f32(f32(az + bs.PI) / bs.TWO_PI) * f32(c["cols"])))), c["cols"] - 1)
            rowf = np.floor(f32(f32(f32(el - lo) / span) * f32(c["rows"])))
            want = int(rowf) * c["cols"] + col if 0 <= rowf < c["rows"] else -1
            assert got[i] == want
            assert r[i] == np.sqrt(f32(s + f32(z * z)))


def test_points_on_bin_boundaries():
    # points whose azimuth is the float nearest a column edge, both sides: the column is the floor of the float expression
    cols = 1800
    for j in (1, 450, 899, 900, 1350, 1799):
        a = f32(j / cols * (2 * math.pi) - math.pi)
        for az in (np.nextafter(a, f32(-4)), a, np.nextafter(a, f32(4))):
            x, y = f32(20 * math.cos(az)), f32(20 * math.sin(az))
            c, _ = _cell(x, y, -1.0)
            want = min(int(np.floor(f32(f32(np.arctan2(y, x) + bs.PI) / bs.TWO_PI) * f32(cols))), cols - 1)
            assert c % cols == want and abs(c % cols - j) <= 1


def test_learning_counts_frames_not_points():
    lrn = bs.Learner(rows=4, cols=8, elev_min_deg=-10.0, elev_max_deg=10.0)
    p = np.array([[10.0, 0.0, 0.0], [12.0, 0.0, 0.0], [11.0, 0.0, 0.01]], f32)    # one cell, three points
    lrn.learn(p)
    lrn.learn(p[:1])
    c, _ = bs.cells(p[:1], **lrn.c)
    assert lrn.hits[c[0]] == 2 and lrn.B[c[0]] == f32(12.0) and lrn.hits.sum() == 2


@pytest.mark.parametrize("cfg", [dict(nbr_cols=0, nbr_rows=0), dict(nbr_cols=1, nbr_rows=0), dict(nbr_cols=2, nbr_rows=1),
                                 dict(nbr_cols=3, nbr_rows=2, min_hit_frac=0.0), dict(nbr_cols=1, nbr_rows=1, min_hit_frac=1.0)])
def test_freeze_equals_brute_force(cfg):
    rng = np.random.default_rng(len(str(cfg)))
    rows, cols, frames = 6, 11, 7
    hits = rng.integers(0, frames + 1, rows * cols)
    B = rng.uniform(1, 60, rows * cols).astype(f32)
    c = dict(dict(rows=rows, cols=cols, min_hit_frac=0.5), **cfg)
    got = bs.freeze(hits, B, frames, **c)
    assert np.array_equal(got, bs.freeze_brute(hits, B, frames, **c))


def test_freeze_threshold_and_column_wrap():
    rows, cols, L = 2, 5, 4
    hits = np.full(rows * cols, 4)
    B = np.full(rows * cols, 30.0, f32)
    B[0] = 5.0                                           # row 0, column 0
    hits[6] = 1                                          # row 1, column 1: 1 < ceil(0.5 * 4) -> no background
    t = bs.freeze(hits, B, L, rows, cols, 0.5, 1, 0)
    assert list(t[0]) == [5.0, 5.0, 30.0, 30.0, 5.0]     # column 0's value reaches column 4 across the wrap
    t = bs.freeze(hits, B, L, rows, cols, 0.5, 0, 0)
    assert t[1, 1] == np.inf and t[0, 0] == 5.0
    assert bs.freeze(hits, B, L, rows, cols, 0.25, 0, 0)[1, 1] == 30.0   # ceil(0.25 * 4) = 1
    t = bs.freeze(hits, B, L, rows, cols, 0.5, 0, 1)
    assert t[1, 0] == 5.0 and t[1, 1] == 30.0            # rows reach across, but do not wrap


def test_filter_keeps_points_in_front_and_without_a_cell():
    rows, cols = 4, 8
    cfg = dict(rows=rows, cols=cols, elev_min_deg=-10.0, elev_max_deg=10.0)
    Bn = np.full((rows, cols), 20.0, f32)
    e = np.array([[19.7, 0.0, 0.0], [19.69, 0.0, 0.0], [25.0, 0.0, 0.0], [10.0, 0.0, 8.0]], f32)
    keep = bs.keep_flags(e, Bn, margin_m=0.3, **cfg)
    # 19.7 < 20 - 0.3 is false in float (20 - 0.3 = 19.7 as float); 19.69 is in front; 25 is behind; the last has no cell
    assert list(keep) == [bool(f32(19.7) < f32(20.0) - f32(0.3)), True, False, True]
    assert np.array_equal(bs.foreground(e, Bn, margin_m=0.3, **cfg), e[keep])
    assert list(bs.keep_flags(e, np.full((rows, cols), np.inf, f32), **cfg)) == [True] * 4


def test_default_values_and_validation():
    assert bs.DEFAULTS == dict(rows=64, elev_min_deg=-25.0, elev_max_deg=3.0, cols=1800, learn_frames=50, min_hit_frac=0.5,
                               margin_m=0.3, nbr_cols=1, nbr_rows=0)
    bs.validate(**bs.DEFAULTS)
    bs.validate(**dict(bs.DEFAULTS, rows=128, cols=4096, learn_frames=1, min_hit_frac=0.0, margin_m=0.0))
    bs.validate(**dict(bs.DEFAULTS, min_hit_frac=1.0))
    for bad in [dict(rows=0), dict(rows=129), dict(cols=0), dict(cols=4097), dict(elev_min_deg=3.0), dict(elev_max_deg=-30.0),
                dict(elev_min_deg=float("nan")), dict(learn_frames=0), dict(min_hit_frac=-0.01), dict(min_hit_frac=1.01),
                dict(margin_m=-0.1), dict(margin_m=float("inf")), dict(nbr_cols=1800), dict(nbr_rows=64)]:
        with pytest.raises(ValueError):
            bs.validate(**dict(bs.DEFAULTS, **bad))


# The reference's chain on the stationary-sensor scene (seed 5, 50 learning frames, 20 scored frames) with the proposed defaults:
# (object instances, of them standing where they stood through all of learning, found on E, ghosts on E, found on E_fg, ghosts on
# E_fg, found only on E_fg, lost on E_fg, lost and learned).  E_fg removes most ghost boxes, but it also loses objects that E finds and
# that stood nowhere near their learning-time place, so the filter is not built (DESIGN.md §6n).
PREMISE = {
    ("64", "moving"): (520, 65, 122, 459, 117, 97, 9, 14, 1),
    ("32", "moving"): (520, 65, 27, 225, 26, 67, 9, 10, 0),
}


@pytest.mark.parametrize("sensor,mode", list(PREMISE))
def test_premise_numbers(synth, ref_intended, sensor, mode):
    lrn = bs.Learner()
    Bn = None
    tot = np.zeros(9, np.int64)
    for pts, obj, learned, learning in bs.stationary_frames(synth, sensor, mode, 50, 20, seed=5):
        e, g = ref_intended.ground_remove(pts)
        if learning:
            lrn.learn(np.concatenate([e, g]))
            continue
        Bn = lrn.freeze() if Bn is None else Bn
        fe, ge = bs.matched(bs.ref_boxes(ref_intended, e), obj)
        fk, gk = bs.matched(bs.ref_boxes(ref_intended, bs.foreground(e, Bn)), obj)
        tot += [len(obj), learned.sum(), fe.sum(), ge, fk.sum(), gk, (fk & ~fe).sum(), (fe & ~fk).sum(), (fe & ~fk & learned).sum()]
    got = tuple(int(v) for v in tot)
    assert got == PREMISE[(sensor, mode)]
    assert got[5] < got[3] / 2                                     # most ghost boxes go
    assert got[7] > got[8]                                         # some objects are lost that learning does not explain

