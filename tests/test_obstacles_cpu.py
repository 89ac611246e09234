"""Obstacle footprints restated in NumPy (tests/obstacle_scenes.py): the monotone-chain hull over column extremes equals the hull by
definition on random and hand-built cell sets, its vertex order, start and metres conversion are the documented ones, the 140-vertex bound
is tight, and on existing scenes the reference chain leaves structures without a box that an obstacle footprint covers."""
import importlib

import numpy as np
import pytest

import detect_area_scenes as da
import layer_scenes as ls
import obstacle_scenes as os_

f32 = np.float32


def _check_polygon(cells, h):
    """strictly convex, counter-clockwise, starting at the smallest (u, v), every cell corner inside or on it"""
    m = len(h)
    assert m >= 4
    assert tuple(h[0]) == min(map(tuple, h))
    for i in range(m):
        assert os_._cross(h[i], h[(i + 1) % m], h[(i + 2) % m]) > 0, "three consecutive vertices collinear or turning right"
    C = os_.corners(cells)
    for i in range(m):
        a, b = h[i], h[(i + 1) % m]
        assert np.all((b[0] - a[0]) * (C[:, 1] - a[1]) - (b[1] - a[1]) * (C[:, 0] - a[0]) >= 0)


def _same_as_brute(cells):
    h = os_.hull(cells)
    assert set(map(tuple, h)) == os_.brute_vertices(cells)
    _check_polygon(cells, h)
    return h


@pytest.mark.parametrize("seed", range(12))
def test_hull_equals_brute_force_random(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 25))
    span = int(rng.integers(1, 12))
    u0, v0 = rng.integers(0, 250 - span, 2)
    cells = {(int(u0 + a), int(v0 + b)) for a, b in rng.integers(0, span, (n, 2))}
    _same_as_brute(cells)


def test_hand_built_cases():
    # a single cell: its four corners
    assert os_.hull([(5, 7)]).tolist() == [[5, 7], [6, 7], [6, 8], [5, 8]]
    # 1 x k strips in u and in v: still four vertices (the long sides' corners are collinear)
    for k in (2, 3, 9):
        assert os_.hull([(3 + i, 4) for i in range(k)]).tolist() == [[3, 4], [3 + k, 4], [3 + k, 5], [3, 5]]
        assert os_.hull([(3, 4 + i) for i in range(k)]).tolist() == [[3, 4], [4, 4], [4, 4 + k], [3, 4 + k]]
    # an L: the inner corner is not a vertex, the diagonal cuts it
    L = [(0, 0), (1, 0), (2, 0), (0, 1), (0, 2)]
    assert _same_as_brute(L).tolist() == [[0, 0], [3, 0], [3, 1], [1, 3], [0, 3]]
    # a diagonal chain: a hexagon
    D = [(10 + i, 20 + i) for i in range(5)]
    assert _same_as_brute(D).tolist() == [[10, 20], [11, 20], [15, 24], [15, 25], [14, 25], [10, 21]]
    # collinear boundary corners of a block with a bump: only the bump's corners and the block's are kept
    B = [(u, v) for u in range(4) for v in range(3)] + [(1, 3), (2, 3)]
    _same_as_brute(B)
    assert [1, 3] not in os_.hull(B).tolist() and [0, 3] in os_.hull(B).tolist()
    # cells on the grid edges 0 and 249: corners 0 and 250
    E = [(0, 0), (249, 249), (0, 249), (249, 0)]
    assert _same_as_brute(E).tolist() == [[0, 0], [250, 0], [250, 250], [0, 250]]
    _same_as_brute([(249, 3), (249, 4), (248, 9)])
    # gaps between columns (dilation joins cells three apart) and an empty set
    _same_as_brute([(5, 5), (8, 9), (8, 2)])
    assert len(os_.hull([])) == 0


def test_vertex_count_bound_is_tight():
    """no convex lattice polygon in [0, 250]^2 has more than 140 vertices (cheapest distinct primitive edge vectors under the 4 x 250
    L1 budget), and the cells inside the constructed polygon reach it"""
    assert os_.bound_from_l1() == os_.MAX_HULL
    P = os_.max_hull_polygon()
    assert len(P) == os_.MAX_HULL and P.min() == 0 and P.max() == 250
    cells = os_.max_hull_cells()
    h = os_.hull(cells)
    assert len(h) == os_.MAX_HULL
    assert set(map(tuple, h)) == set(map(tuple, P))
    _check_polygon(cells, h)


@pytest.mark.parametrize("roi", [50.0, 30.0])
def test_metres_and_cells_inside(roi):
    """vertex (u, v) in metres with the unit's roi, computed in double and rounded once; every point of a cluster lies inside or on its
    polygon"""
    assert os_.to_metres([[0, 0]], roi).tolist() == [[-roi / 2, -roi / 2]]
    assert os_.to_metres([[250, 125]], roi).tolist() == [[roi / 2, 0.0]]
    u = np.arange(251)
    want = np.array([f32(float(x) * float(f32(roi)) / 250.0 - float(f32(roi)) / 2.0) for x in u], f32)
    assert np.array_equal(os_.to_metres(np.stack([u, u], 1), roi)[:, 0].view(np.uint32), want.view(np.uint32))
    rng = np.random.default_rng(3)
    pts = np.concatenate([rng.normal([3.0, -2.0, -1.0], [1.5, 0.7, 0.4], (400, 3)),
                          rng.normal([-8.0, 6.0, -0.5], [0.3, 2.0, 0.6], (300, 3))]).astype(f32)
    ids = np.r_[np.ones(400, np.int32), np.full(300, 2, np.int32)]
    obs = os_.obstacles(pts, ids, 2, roi)
    for o in obs:
        sel = pts[ids == o["cluster"]]
        assert os_.inside(o["xy"], sel[:, :2]).all()
        assert o["z_min"] == sel[:, 2].min() and o["z_max"] == sel[:, 2].max()
        xi, yi, _ = ls.columns(sel, roi)
        assert o["n_cells"] == len(set(zip(xi.tolist(), yi.tolist())))


def _uncovered_structures(ref, pts, items):
    """the reference chain on one frame -> how many of the structures (each a boolean mask over E) lie wholly inside one obstacle footprint
    whose cluster got no box, and how many clusters of the frame got no box"""
    e, _ = ref.ground_remove(pts)
    grid, k = ref.component_clustering(e)
    ids = os_.label_ids(e, grid)
    flags, boxes = os_.ref_box_flags(ref, e, ids, k)
    want, _ = ref.box_fitting(e, grid, k)
    assert np.array_equal(boxes.view(np.uint32), np.asarray(want, f32).reshape(-1, 8, 3).view(np.uint32))   # per cluster == whole frame
    obs = os_.obstacles(e, ids, k, box_ok=flags)
    covered = 0
    for sel in items(e):
        if not sel.any():
            continue
        for o in obs:
            if o["box"] < 0 and os_.inside(o["xy"], e[sel, :2]).all():
                covered += 1
                break
    return covered, int((~flags).sum()), k


def test_structures_without_boxes_have_footprints(ref_intended):
    """seed 7: the 3.5 m truck of the canopy scene and the roadside poles and hedges of the detection-area scene get no box from the
    reference chain; the truck and 10 of the 18 roadside items each lie wholly inside the footprint of an obstacle without a box"""
    synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
    pts, objects = ls.render("64", seed=7)
    (tx, ty), = [(x, y) for x, y, kind in objects if kind == "truck"]
    truck = lambda e: (np.hypot(e[:, 0] - tx, e[:, 1] - ty) < 4.5) & (e[:, 2] > synth.SENSOR_Z_GROUND + 0.3)
    got = _uncovered_structures(ref_intended, pts, lambda e: [truck(e)])
    assert got[0] == 1, got
    _, frame = next(iter(da.cluttered_frames(synth, 1, seed=7)))

    def clutter(e):
        return [(np.abs(e[:, 0] - x) <= L / 2 + 0.05) & (np.abs(e[:, 1] - y) <= W / 2 + 0.05) for x, y, L, W, _ in da.CLUTTER]
    got = _uncovered_structures(ref_intended, frame, clutter)
    assert got[0] == PINNED_CLUTTER, got


PINNED_CLUTTER = 10            # of the 18 poles and hedges (the others get a box, or too few returns to cluster)
