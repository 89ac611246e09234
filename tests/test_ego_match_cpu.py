"""Scan-matched ego motion without a device: the restatement of tests/ego_match_scenes.py against a per-hypothesis brute force, and
its field, sample and validation rules."""
import math

import numpy as np
import pytest

import ego_match_scenes as em

f32 = np.float32
SMALL = dict(grid=32, cell_m=0.25, r_min=0.5, r_max=5.0, sub_m=0.5, max_points=64, yaw_step=0.02, yaw_half=3, shift_half=3,
             refine=2, min_points=1, z_min=-1.0, z_max=1.0)


def small(**kw):
    return dict(em.defaults(), **dict(SMALL, **kw))


def cloud(rng, n, half=4.0, nan=0):
    p = np.zeros((n, 4), f32)
    p[:, 0:2] = rng.uniform(-half, half, (n, 2))
    p[:, 2] = rng.uniform(-1.5, 1.5, n)
    p[:nan, rng.integers(0, 3)] = np.nan
    return p


def moved(p, dx, dy, dth):
    """the cloud seen from a frame at (dx, dy, dth) in p's frame"""
    c, s = math.cos(dth), math.sin(dth)
    q = p.copy()
    x, y = p[:, 0].astype(np.float64) - dx, p[:, 1].astype(np.float64) - dy
    q[:, 0], q[:, 1] = c * x + s * y, -s * x + c * y
    return q


def ref_field(p, s):
    x, y, ok, win, ix, iy = em.band(p, s)
    return em.field(ix, iy, win, s["grid"])[0], x, y, win


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("refine", [1, 3])
def test_restatement_equals_brute_force(seed, refine):
    rng = np.random.default_rng(seed)
    s = small(refine=refine)
    p0 = cloud(rng, 60, nan=3)
    p0[:4, 0] = [7.0, -7.0, 4.9, -4.9]          # outside the window (H = 4) and on its edge
    p1 = moved(p0, *rng.uniform(-0.3, 0.3, 2), rng.uniform(-0.05, 0.05))
    L, *_ = ref_field(p0, s)
    _, x, y, win = ref_field(p1, s)
    xs, ys = em.sample(x, y, win, s)
    prior = (0.0, 0.0, 0.0) if seed % 2 else tuple(rng.uniform(-0.4, 0.4, 2)) + (0.03,)
    assert em.match(L, xs, ys, s, prior) == em.brute_match(L, xs, ys, s, prior)


def test_ties_go_to_the_first_hypothesis():
    s = small(refine=2)
    L = np.zeros((32, 32), np.uint8)          # an empty reference: every hypothesis scores 0
    xs, ys = np.array([0.1, 1.0], f32), np.array([0.2, -1.0], f32)
    got = em.match(L, xs, ys, s, (0.0, 0.0, 0.0))
    assert got == em.brute_match(L, xs, ys, s, (0.0, 0.0, 0.0))
    R = 2
    # coarse: j = -3, kx = ky = -3; fine: u = ax = ay = -R around it
    assert got == (0, (R * -3 - R) * s["cell_m"] / R, (R * -3 - R) * s["cell_m"] / R, float(R * -3 - R) * s["yaw_step"] / R)


def test_grid_edges_and_outside_cells_score_zero():
    s = small(refine=1, yaw_half=0, shift_half=3)
    L = np.zeros((32, 32), np.uint8)
    L[0, :] = 3
    L[:, 31] = 3
    H = float(em.half_width(s))
    xs = np.array([-H + 0.1, H - 0.1], f32)
    ys = np.array([-H + 0.1, H - 0.1], f32)
    sc = em.coarse_scores(L, xs, ys, s, 0, 0, 0)
    bf = np.zeros_like(sc)
    for ix in range(7):
        for iy in range(7):
            for x, y in zip(xs, ys):
                cx = int(np.floor((x + f32(H)) / f32(s["cell_m"]))) + ix - 3
                cy = int(np.floor((y + f32(H)) / f32(s["cell_m"]))) + iy - 3
                bf[0, ix, iy] += int(L[cy, cx]) if 0 <= cx < 32 and 0 <= cy < 32 else 0
    assert np.array_equal(sc, bf)


def test_empty_band_and_nan_frames():
    s = small()
    p = np.full((10, 4), np.nan, f32)
    x, y, ok, win, ix, iy = em.band(p, s)
    assert not ok.any()
    m = em.Matcher(s)
    o1 = m.estimate(p, 100_000.0)
    o2 = m.estimate(p, 200_000.0)
    assert (o1["ok"], o1["n_used"], o2["ok"], o2["n_used"], o2["score"], o2["v"]) == (0, 0, 0, 0, 0, 0.0)


def test_band_rules():
    s = small()
    p = np.array([[1.0, 0.0, 0.0, 0], [0.4, 0.0, 0.0, 0], [5.0, 0.0, 0.0, 0], [5.01, 0.0, 0.0, 0], [1.0, 0.0, 1.0, 0],
                  [1.0, 0.0, 1.01, 0], [1.0, 0.0, -1.0, 0], [np.inf, 0.0, 0.0, 0], [3.0, 4.0, 0.0, 0]], f32)
    _, _, ok, win, ix, iy = em.band(p, s)
    assert ok.tolist() == [True, False, True, False, True, False, True, False, True]
    # (5, 0): cell floor((5 + 4) / 0.25) = 36 is outside the 32-cell window; (3, 4) likewise
    assert win.tolist() == [True, False, False, False, True, False, True, False, False]


def test_field_is_three_minus_chebyshev_distance():
    rng = np.random.default_rng(4)
    g = 32
    ix, iy = rng.integers(0, g, 12), rng.integers(0, g, 12)
    L, n = em.field(ix, iy, np.ones(12, bool), g)
    occ = set(zip(iy.tolist(), ix.tolist()))
    assert n == len(occ)
    for cy in range(g):
        for cx in range(g):
            d = min(max(abs(cy - a), abs(cx - b)) for a, b in occ)
            assert L[cy, cx] == 3 - min(3, d)


def test_sample_rule():
    s = small(max_points=3)
    # sub-cells of 0.5 m from -4: points 0 and 2 share one, 1 is alone, 3 and 4 are further up
    x = np.array([0.1, 1.1, 0.2, -2.0, 2.0], f32)
    y = np.array([0.1, 0.1, 0.3, 2.0, 3.0], f32)
    win = np.ones(5, bool)
    xs, ys = em.sample(x, y, win, dict(s, max_points=8))
    assert xs.tolist() == [x[0], x[1], x[3], x[4]]
    xs, ys = em.sample(x, y, win, s)          # 4 > 3: every 2nd
    assert xs.tolist() == [x[0], x[3]]


def test_validation():
    d = em.defaults()
    assert em.valid(d)
    bad = [dict(grid=16), dict(grid=1056), dict(grid=100), dict(cell_m=0.0), dict(cell_m=float("nan")), dict(grid=1024, cell_m=0.5),
           dict(z_min=1.0, z_max=1.0), dict(r_min=40.0), dict(r_min=-1.0), dict(r_max=2000.0), dict(sub_m=0.01), dict(max_points=0),
           dict(max_points=9000), dict(yaw_step=0.0), dict(yaw_step=0.2), dict(yaw_half=181), dict(shift_half=128), dict(refine=0),
           dict(refine=16), dict(min_points=0), dict(min_score_frac=1.5), dict(min_score_frac=float("inf")), dict(sensor=-2),
           dict(sensor=8)]
    for b in bad:
        assert not em.valid(dict(d, **b)), b
    for g in (dict(grid=1024, cell_m=0.39), dict(refine=1), dict(yaw_half=0, shift_half=0), dict(sensor=7)):
        assert em.valid(dict(d, **g)), g


def test_state_rules():
    rng = np.random.default_rng(9)
    s = small(min_points=5)
    p0 = cloud(rng, 80)
    m = em.Matcher(s)
    o = m.estimate(p0, 1_000_000.0)
    assert (o["ok"], o["v"], o["dtheta"], o["yaw"]) == (0, 0.0, 0.0, 0.0)          # first call
    o = m.estimate(moved(p0, 0.25, 0.0, 0.02), 1_100_000.0)
    assert o["ok"] == 1 and o["dx"] == pytest.approx(0.25, abs=0.13) and o["yaw"] == o["dtheta"]
    y1 = o["yaw"]
    o = m.estimate(p0, 1_100_000.0)                                                     # dt = 0: nothing matched, yaw kept
    assert (o["ok"], o["v"], o["dtheta"], o["yaw"]) == (0, 0.0, 0.0, y1)
    o = m.estimate(p0[:3], 1_200_000.0)                                                 # below min_points: the prior (0 after dt = 0)
    assert (o["ok"], o["score"], o["dx"]) == (0, 0, 0.0)
    m.reset()
    o = m.estimate(p0, 1_300_000.0)
    assert (o["ok"], o["yaw"]) == (0, 0.0)


def test_constant_velocity_fallback_uses_the_scaled_prior():
    rng = np.random.default_rng(2)
    s = small(min_points=5)
    p0 = cloud(rng, 80)
    m = em.Matcher(s)
    m.estimate(p0, 0.0)
    o1 = m.estimate(moved(p0, 0.25, 0.0, 0.0), 100_000.0)
    assert o1["ok"] == 1
    o2 = m.estimate(np.zeros((0, 4), f32), 300_000.0)                                  # empty: prior = delta * 2
    assert o2["ok"] == 0 and o2["dx"] == o1["dx"] * 2.0 and o2["v"] == pytest.approx(o1["v"])
