"""Track retirement (lmot_set_track_retirement) against the reference, without a GPU.

The oracle of retirement is the reference with one extra operation after every immUkfJpdaf: ref_tracker_retire (oracle/ref_retire.cpp,
bound by oracle/ref_retire.py) stably erases the tracks with trackNumVec_[i] == 0 from targets_ / trackNumVec_ and touches nothing
else.  These tests check that oracle, and the one
claim the contract rests on: the erasing reference equals the unbounded one (rows matched by track ID) up to the first frame in which
a dead track's frozen x_merge_ lies inside a visible track's box -- mergeOverSegmentation (imm_ukf_jpda.cpp:682-695) tests every
track, dead ones included, and nothing else of the reference reads a dead row.
"""
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "hotpath_golden.npz")
D_X = 4
KEYS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis")


@pytest.fixture(scope="module")
def ref():
    from oracle import ref, ref_retire
    if not ref.have_ref("intended") or not ref_retire.have_retire("intended"):
        pytest.skip("oracle/_ref not built")
    r = ref.RefOracle("intended")
    r.tracker_retire = ref_retire.retirer(r)
    return r


def bench_scene(n):
    """the tracking-only bench workload (scripts/seq_track_measure.py): ~64 tracks, clutter boxes that spawn and die, with a moving ego"""
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    try:
        stm = importlib.import_module("seq_track_measure")
    finally:
        sys.path.pop(0)
    lists = stm.bench_lists(0, n)
    return [(1e5 * (f + 1), lists[f], 2.0 + 0.5 * np.sin(0.03 * f), 0.4 + 0.004 * f) for f in range(n)]


def golden_scene():
    z = np.load(GOLD)
    return [(float(z[f"ts{i}"]), z[f"boxes_intended{i}"], 0.0, 0.0) for i in range(int(z["n_frames"]))]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def test_retire_without_dead_rows_is_a_noop(ref):
    scene = golden_scene()
    ref.tracker_reset()
    plain = [ref.tracker_step(b, ts, v, y) for ts, b, v, y in scene]
    f0 = next(f for f, o in enumerate(plain) if len(o["track_manage"]) and np.all(o["track_manage"] != 0))
    ref.tracker_reset()
    for f, (ts, b, v, y) in enumerate(scene):
        o = ref.tracker_step(b, ts, v, y)
        if f == f0:
            n = ref.tracker_num_tracks()
            ref.tracker_retire()
            assert ref.tracker_num_tracks() == n
        for k in KEYS + ("vis_bb",):
            assert _same(o[k], plain[f][k]), (f, k)


def test_retire_removes_exactly_the_dead_rows(ref):
    ref.tracker_reset()
    checked = 0
    for ts, b, v, y in bench_scene(60):
        ref.tracker_step(b, ts, v, y)
        before = ref.tracker_dump()
        ref.tracker_retire()
        after = ref.tracker_dump()
        want = before[before[:, 0] != 0]
        assert after.shape == want.shape and np.array_equal(after.view(np.uint64), want.view(np.uint64))
        checked += int(np.sum(before[:, 0] == 0))
    assert checked > 0, "the scene never killed a track"


def _contains(c, px, py):
    """mergeOverSegmentation's test (imm_ukf_jpda.cpp:670-692): which of the positions (px, py) (arrays) does the box with corners c
    (4 x (x, y), float) contain?"""
    v = c.astype(np.float64)
    (v1x, v1y), (v2x, v2y), (v3x, v3y), (v4x, v4y) = v
    cp1x, cp1y = (v1x + v2x + v3x) / 3, (v1y + v2y + v3y) / 3
    cp2x, cp2y = (v1x + v4x + v3x) / 3, (v1y + v4y + v3y) / 3

    def k(ax, ay, bx, by, cx, cy):
        return ((ax - bx) * (py - ay) + (ay - by) * (ax - px)) * ((ax - bx) * (cy - ay) + (ay - by) * (ax - cx))
    c1, c2, c3 = k(v1x, v1y, v2x, v2y, cp1x, cp1y), k(v1x, v1y, v3x, v3y, cp1x, cp1y), k(v3x, v3y, v2x, v2y, cp1x, cp1y)
    c4, c5, c6 = k(v1x, v1y, v4x, v4y, cp2x, cp2y), k(v1x, v1y, v3x, v3y, cp2x, cp2y), k(v3x, v3y, v4x, v4y, cp2x, cp2y)
    return ((c1 > 0) & (c2 > 0) & (c3 > 0)) | ((c4 > 0) & (c5 > 0) & (c6 > 0))


def test_erasing_reference_equals_unbounded_until_a_ghost_containment(ref):
    scene = bench_scene(320)
    # unbounded: row index = track ID; x_merge_ of every dead track, frozen from the step it died in
    ref.tracker_reset()
    full, ghost_frames, n_ghost = [], [], 0
    dead_pos = {}
    row = np.zeros(236, np.float64)
    for f, (ts, b, v, y) in enumerate(scene):
        o = ref.tracker_step(b, ts, v, y)
        vis_rows = np.nonzero(o["is_vis"])[0]
        hits = 0
        if dead_pos:
            dj = np.fromiter(dead_pos.keys(), np.int64)
            dp = np.array(list(dead_pos.values()), np.float64)
            for slot, i in enumerate(vis_rows):
                hits += int(np.sum(_contains(o["vis_bb"][slot, :4, :2], dp[:, 0], dp[:, 1]) & (dj != i)))
        if hits:
            ghost_frames.append(f)
            n_ghost += hits
        for j in np.nonzero(o["track_manage"] == 0)[0]:
            if int(j) not in dead_pos:
                ref._td(int(j), row)
                dead_pos[int(j)] = (row[D_X], row[D_X + 1])
        full.append(o)
    # erasing reference, IDs by bookkeeping: the rows retained after the previous step, then this step's spawns
    ref.tracker_reset()
    ids, nxt, first_diff = [], 0, None
    for f, (ts, b, v, y) in enumerate(scene):
        o = ref.tracker_step(b, ts, v, y)
        n = len(o["track_manage"])
        n_new = n - len(ids)
        ids += list(range(nxt, nxt + n_new))
        nxt += n_new
        sel = np.asarray(ids, np.int64)
        same = all(_same(o[k], full[f][k][sel]) for k in KEYS) and _same(o["vis_bb"], full[f]["vis_bb"])
        if not same and first_diff is None:
            first_diff = f
        ref.tracker_retire()
        ids = [i for i, tm in zip(ids, o["track_manage"]) if tm != 0]
        assert ref.tracker_num_tracks() == len(ids)
    first_ghost = ghost_frames[0] if ghost_frames else None
    print(f"\nbench scene, {len(scene)} frames: unbounded table {len(full[-1]['track_manage'])} rows, erasing table {len(ids)} rows; "
          f"first ghost containment at frame {first_ghost}, {n_ghost} ghost containments in {len(ghost_frames)} frames; "
          f"first difference at frame {first_diff}")
    if first_diff is not None:
        assert first_ghost is not None and first_diff >= first_ghost, "the erasing reference differs before any ghost containment"
