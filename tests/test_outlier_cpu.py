"""The outlier filter of DESIGN.md §6m without a device: the NumPy restatement of steps 1-4
(tests/weather_scenes.py) equals the pairwise evaluation on small clouds, and the reference's chain on snowy frames of synth.py's scene
gives the counts pinned below on E and on E_kept."""
import numpy as np
import pytest

import weather_scenes as ws

f32 = np.float32


def _both(p, **cfg):
    got, want = ws.keep_flags(p, **cfg), ws.keep_brute(p, **cfg)
    assert np.array_equal(got, want)
    return got


def test_neighbour_exactly_at_the_radius():
    # R = min_radius = 0.5 for both points; d^2 = 0.25 = R^2 exactly: a neighbour.  One float further: not.
    p = np.array([[0.25, 0.0, 0.0], [0.75, 0.0, 0.0]], f32)
    assert list(_both(p, min_radius=0.5, min_neighbors=1)) == [True, True]
    q = p.copy()
    q[1, 0] = np.nextafter(f32(0.75), f32(1.0))
    assert list(_both(q, min_radius=0.5, min_neighbors=1)) == [False, False]


def test_duplicates_are_neighbours():
    p = np.array([[5.0, 1.0, -1.0]] * 3 + [[9.0, 9.0, 0.0]], f32)
    assert list(_both(p, min_neighbors=2)) == [True, True, True, False]
    assert list(_both(p, min_neighbors=3)) == [False] * 4


def test_k_minus_one_and_k_neighbours():
    # a centre with exactly k neighbours is kept, with k - 1 it is not
    k = 4
    centre = np.array([[10.0, 0.0, 0.0]], f32)
    ring = np.array([[10.0 + 0.02 * np.cos(a), 0.02 * np.sin(a), 0.0] for a in np.linspace(0, 2 * np.pi, k, endpoint=False)], f32)
    full = np.concatenate([centre, ring])
    assert _both(full, min_neighbors=k)[0]
    assert not _both(full[:-1], min_neighbors=k)[0]


def test_clamping_at_both_radii():
    # near the sensor beta * alpha * r is below min_radius: R = min_radius
    near = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.039], [1.0, 0.0, -0.041]], f32)
    assert list(_both(near, min_neighbors=1)) == [True, True, False]
    # at r = 100 m beta * alpha * r = 1.05 m: clamped to max_radius = 1 m
    far = np.array([[100.0, 0.0, 0.0], [100.0, 0.0, 1.0], [100.0, 0.0, -1.02]], f32)
    assert list(_both(far, min_neighbors=1)) == [True, True, False]
    assert list(_both(far, min_neighbors=1, max_radius=2.0)) == [True, True, True]


def test_relation_is_not_symmetric():
    # 0.3165 m apart at 30 m: R = 0.315 m for the nearer point, 0.3183 m for the farther, which alone has a neighbour
    p = np.array([[30.0, 0.0, 0.0], [30.3165, 0.0, 0.0]], f32)
    assert list(_both(p, min_neighbors=1)) == [False, True]


def test_lone_point_and_k_zero():
    lone = np.array([[3.0, 4.0, 0.0]], f32)
    assert list(_both(lone, min_neighbors=1)) == [False]
    assert list(_both(lone, min_neighbors=0)) == [True]
    assert ws.keep_flags(np.zeros((0, 4), f32)).shape == (0,)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_clouds(seed):
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.normal([8.0, 3.0, -1.0], 0.15, (120, 3)), rng.uniform(-30, 30, (60, 3))]).astype(f32)
    p[5] = p[6]
    for cfg in [{}, dict(min_neighbors=1), dict(min_neighbors=6, beta=5.0), dict(alpha_rad=0.01, max_radius=0.3)]:
        _both(p, **cfg)


def test_snow_replaces_returns_in_front_of_the_hit(synth):
    pts, _ = ws.scene_frames(synth, "32", 1)[0]
    s = ws.snow(pts, 0.03, seed=4)
    moved = (s != pts).any(1)
    assert 0.02 < moved.mean() < 0.04
    r0 = np.linalg.norm(pts[moved, :3].astype(np.float64), axis=1)
    r1 = np.linalg.norm(s[moved, :3].astype(np.float64), axis=1)
    assert (r1 < r0).all()


# the reference's chain on synth.py's scene (seed 5, 60 objects, 3 frames) with the filter's defaults, per sensor and snow level:
# (objects found on E, ghost boxes on E, objects found on E_kept, ghost boxes on E_kept).  Snow costs objects, and the defaults lose more
# on clean and snowy frames alike than they win back, so the filter is not built (DESIGN.md §6m).
PREMISE = {
    "64": {None: (84, 31, 71, 30), "light": (85, 30, 72, 30), "moderate": (81, 31, 71, 23), "heavy": (79, 31, 71, 27)},
    "32": {None: (56, 25, 31, 21), "light": (54, 22, 31, 21), "moderate": (43, 23, 29, 21), "heavy": (39, 22, 29, 22)},
}


@pytest.mark.parametrize("sensor", ["64", "32"])
def test_premise_numbers(synth, ref_intended, sensor):
    got = {}
    for level in PREMISE[sensor]:
        tot = np.zeros(4, np.int64)
        for pts, obj in ws.scene_frames(synth, sensor, 3, level=level):
            _, b, _ = ws.ref_detect(ref_intended, pts)
            _, bk, _ = ws.ref_detect(ref_intended, pts, ws.DEFAULTS)
            tot += ws.score(b, obj) + ws.score(bk, obj)
        got[level] = tuple(int(x) for x in tot)
    assert got == PREMISE[sensor]
    assert got["heavy"][0] < got[None][0]                          # snow costs the reference objects
    assert all(v[2] < v[0] for v in got.values())                  # the defaults find fewer objects than no filter, clean or snowy
