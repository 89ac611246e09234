"""Obstacle footprints on the device (include/lmot.h, lmot_set_obstacles): off is today's path, the footprints, z ranges and box indices equal
the NumPy restatement (tests/obstacle_scenes.py) on the reference's clusters and per-cluster box verdicts bit for bit, through every
frame submission path, next to the other front-end settings, in batched and sequence ticks, and in the size regimes where they matter."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import layer_scenes as ls
import obstacle_scenes as os_

pytestmark = pytest.mark.gpu
f32 = np.float32


def _params(pkg, gf=0, rule=0, max_points=1 << 17, **kw):
    p = pkg.default_params()
    p.max_points = max_points
    p.global_frame = gf
    p.rule_filter = rule
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _frames(synth, n, seed=5, rings=32, azimuths=900, n_objects=30):
    return [(ts, p) for ts, p in synth.frames(synth.SceneConfig(seed=seed, rings=rings, azimuths=azimuths, n_objects=n_objects), n)]


def _bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _want(ref, elev, ids, k, roi=50.0, max_boxes=1024):
    flags, boxes = os_.ref_box_flags(ref, elev, ids, k, roi)
    return os_.obstacles(elev, ids, k, roi, box_ok=flags, max_boxes=max_boxes), boxes


def _assert_equal(res, want, boxes=None, want_boxes=None):
    """device result of one unit == restatement: every header field, every vertex bit for bit, and box i of the unit's list is the
    reference's box of the cluster that names it"""
    got = res["obstacles"]
    assert res["status"] == 0
    assert len(got) == len(want)
    polys = []
    for row, w in zip(got, want):
        assert (row["cluster"], row["n_points"], row["n_cells"], row["box"]) == (w["cluster"], w["n_points"], w["n_cells"], w["box"]), (row, w)
        assert _bits([row["z_min"], row["z_max"]]).tolist() == _bits([w["z_min"], w["z_max"]]).tolist()
        assert row["vertex_count"] == len(w["hull"])
        polys.append(w["xy"])
    assert res["n_vertices"] == sum(len(p) for p in polys)
    got_xy = np.concatenate([res["vertices"][o: o + c] for o, c in zip(got["vertex_offset"], got["vertex_count"])]) if len(got) else np.zeros((0, 2), f32)
    want_xy = np.concatenate(polys) if polys else np.zeros((0, 2), f32)
    assert np.array_equal(_bits(got_xy), _bits(want_xy))
    if boxes is not None:
        b = np.asarray(boxes, f32).reshape(-1, 8, 3)
        named = sorted(int(x) for x in got["box"] if x >= 0)
        assert named == list(range(len(b)))
        if want_boxes is not None:
            assert np.array_equal(_bits(b), _bits(want_boxes))


def _ref(mode):
    from oracle import ref
    if not ref.have_ref(mode):
        pytest.skip("oracle/_ref not built")
    return ref.RefOracle(mode)


def _oracle_frame(ref, pts, max_boxes=1024):
    e, _ = ref.ground_remove(pts)
    grid, k = ref.component_clustering(e)
    ids = os_.label_ids(e, grid)
    want, wb = _want(ref, e, ids, k, max_boxes=max_boxes)
    return want, wb


# ------------------------------------------------------------------------------------------------ today's path
_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
P = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)][0]
out = {}
for arm in ("off", "on_then_off", "on"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p)
    ctx.seq_open(4, ring=4)
    if arm in ("on_then_off", "on"):
        ctx.set_obstacles(on=1); ctx.seq_set_obstacles(1, on=1, max_vertices=1000)
    if arm == "on_then_off":
        ctx.set_obstacles(); ctx.seq_set_obstacles(1)
    d = torch.from_numpy(P).cuda(); torch.cuda.synchronize()
    def run(t):
        ctx.frame(P, t)
        ctx.frame_dev(d.data_ptr(), len(P), t + 1e5); ctx.frame_fetch()
        ctx.batch([P, P], t + 2e5)
        ctx.seq([P] * 4, [t] * 4)
        torch.cuda.synchronize()
    for w in range(4):                 # every frame slot of the ring and both banks once: first-use allocations stay out of the trace
        run(1e6 + w * 1e6)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(9e6)
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    ctx.close()
print(json.dumps(out))
"""


def test_off_is_todays_path(pkg, synth):
    """obstacles set and cleared again leave the same kernels, copies and memsets; on, every submission adds obstacles_kernel and nothing
    else; results of a context that had them on and off again are bit-identical"""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    assert n["off"] and not any("obstacles_kernel" in x for x in n["off"]), n["off"]
    assert sorted(n["off"]) == sorted(n["on_then_off"])
    assert sum("obstacles_kernel" in x for x in n["on"]) == 4                    # frame, frame_dev, batch, one tick
    assert sorted(x for x in n["on"] if "obstacles_kernel" not in x) == sorted(n["off"])
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_obstacles(on=1, max_vertices=500)
        b.set_obstacles()
        assert b.get_obstacles() == {"on": 0, "max_vertices": 65536}
        c = pkg.Lmot(_params(pkg))
        c.set_obstacles(on=1)
        for ts, p in _frames(synth, 4):
            ra, rb, rc = a.frame(p, ts), b.frame(p, ts), c.frame(p, ts)
            for x in (rb, rc):
                assert np.array_equal(_bits(ra["boxes"]), _bits(x["boxes"]))
                assert np.array_equal(np.asarray(ra["track_manage"]), np.asarray(x["track_manage"]))
        with pytest.raises(pkg.LmotError):
            b.obstacles_result(0)                                              # a result submitted with obstacles off: STATE
        c.close()
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("rule", [0, 1])
def test_against_oracle(pkg, synth, gf, rule):
    """lmot_frame, pipelined _submit / _collect at strides 2 and 3, and lmot_frame_dev + _fetch: footprints == the restatement on the
    reference's label grid, box indices == the per-cluster reference verdicts, and box i of the frame is the reference's"""
    import torch
    ref = _ref("intended" if rule == 0 else "o2")
    frames = _frames(synth, 5, seed=9, rings=64, azimuths=1800, n_objects=40)
    want = [_oracle_frame(ref, p) for _, p in frames]
    ctx = pkg.Lmot(_params(pkg, gf, rule, pipeline_depth=4))
    try:
        ctx.set_obstacles(on=1)
        for (ts, p), (w, wb) in zip(frames, want):
            r = ctx.frame(p, ts)
            res = ctx.obstacles_result(0)
            assert res["n_units"] == 1 and len(res["obstacles"]) == r["num_cluster"]
            _assert_equal(res, w, r["boxes"], None if gf else wb)
        for stride in (2, 3):
            ctx.tracker_reset()
            pending = []
            for i, (ts, p) in enumerate(frames):
                ctx.frame_submit(p, ts)
                pending.append(i)
                if len(pending) == stride or i == len(frames) - 1:
                    for j in pending:
                        r = ctx.frame_collect()
                        _assert_equal(ctx.obstacles_result(0), want[j][0], r["boxes"])
                    pending = []
        ctx.tracker_reset()
        for (ts, p), (w, wb) in zip(frames, want):
            d = torch.from_numpy(np.ascontiguousarray(p)).cuda()
            torch.cuda.synchronize()
            ctx.frame_dev(d.data_ptr(), len(p), ts)
            r = ctx.frame_fetch()
            _assert_equal(ctx.obstacles_result(0), w, r["boxes"])
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ with the other settings
def test_with_layers_area_search_lines(pkg, synth, ref_intended):
    """layers on: footprints == the restatement on the device's point clusters; box search changes the box list, not the footprints, and
    `box` follows the new list; ground lines change the elevated cloud, and every cluster still has its obstacle with `box` following the
    list; a detection area restricts the clusters to the area's points"""
    pts, _ = ls.render("64", seed=7)
    e, _ = ref_intended.ground_remove(pts)
    base = pkg.Lmot(_params(pkg, max_points=1 << 18))
    try:
        base.set_obstacles(on=1)
        r0 = base.frame(pts, 1e6)
        res0 = base.obstacles_result(0)
        base.set_layers(on=1)
        r = base.frame(pts, 2e6)
        ids = base.debug_point_clusters()[0]
        want = os_.obstacles(e, ids, r["num_cluster"], box_ok=np.zeros(r["num_cluster"], bool))
        res = base.obstacles_result(0)
        got = res["obstacles"]
        for row, w in zip(got, want):
            assert (row["n_points"], row["n_cells"]) == (w["n_points"], w["n_cells"])
        assert np.array_equal(_bits(res["vertices"]), _bits(np.concatenate([w["xy"] for w in want])))
        assert sorted(int(x) for x in got["box"] if x >= 0) == list(range(len(r["boxes"])))
        base.set_layers()
        base.set_box_search(on=1)
        r = base.frame(pts, 3e6)
        res = base.obstacles_result(0)
        for f in ("cluster", "n_points", "n_cells", "vertex_offset", "vertex_count", "z_min", "z_max"):
            assert np.array_equal(res["obstacles"][f], res0["obstacles"][f]), f
        assert np.array_equal(_bits(res["vertices"]), _bits(res0["vertices"]))
        assert sorted(int(x) for x in res["obstacles"]["box"] if x >= 0) == list(range(len(r["boxes"])))
        base.set_box_search()
        base.set_ground_lines(on=1)
        r = base.frame(pts, 3.5e6)
        res = base.obstacles_result(0)
        assert len(res["obstacles"]) == r["num_cluster"] and res["obstacles"]["n_points"].sum() <= r["n_elevated"]
        assert sorted(int(x) for x in res["obstacles"]["box"] if x >= 0) == list(range(len(r["boxes"])))
        base.set_ground_lines()
        base.set_detect_area([np.array([[-15.0, -15.0], [15.0, -15.0], [15.0, 15.0], [-15.0, 15.0]])])
        r = base.frame(pts, 4e6)
        res = base.obstacles_result(0)
        assert len(res["obstacles"]) == r["num_cluster"]
        assert np.all(np.abs(res["vertices"]) <= 16.0)
    finally:
        base.close()


def test_accumulate_and_rigs(pkg, synth):
    """accumulation (E_acc), rigs separate and merged via lmot_batch / lmot_batch_dev: one unit per frame (merged: one), n_obstacles the
    unit's num_cluster, box indices name the unit's boxes exactly once, every footprint holds its cluster's cells"""
    import torch
    frames = _frames(synth, 3, seed=4)
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_obstacles(on=1)
        ctx.set_accumulate(sweeps=3)
        for ts, p in frames:
            r = ctx.frame(p, ts)
            res = ctx.obstacles_result(0)
            assert len(res["obstacles"]) == r["num_cluster"]
            assert sorted(int(x) for x in res["obstacles"]["box"] if x >= 0) == list(range(len(r["boxes"])))
        ctx.set_accumulate()
        ctx.set_sensors([np.eye(4, dtype=np.float32)[:3], np.eye(4, dtype=np.float32)[:3]])
        for merge in (0, 1):
            ctx.set_rig_merge(merge)
            for dev in (False, True):
                ts, p = frames[0]
                if dev:
                    d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for _ in range(2)]
                    torch.cuda.synchronize()
                    ctx.batch_dev([(x.data_ptr(), len(p)) for x in d], ts + 1e6)
                    out = ctx.batch_fetch()
                else:
                    out = ctx.batch([p, p], ts + 1e6)
                units = 1 if merge else 2
                assert ctx.obstacles_result(0)["n_units"] == units
                for u in range(units):
                    res = ctx.obstacles_result(u)
                    assert len(res["obstacles"]) == out["num_cluster"][u]
                    assert sorted(int(x) for x in res["obstacles"]["box"] if x >= 0) == list(range(out["n_boxes"][u]))
                if not merge:
                    a, b = ctx.obstacles_result(0), ctx.obstacles_result(1)
                    assert np.array_equal(_bits(a["vertices"]), _bits(b["vertices"]))
                with pytest.raises(pkg.LmotError):
                    ctx.obstacles_result(units)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ sequences
def test_sequences_equal_twins(pkg, synth):
    """S = 8 with mixed settings and FRAMES, LISTS, SKIP and RESTART entries: each FRAMES sequence with obstacles on equals a twin context
    with only its own settings; LISTS, skipped and off sequences have no result"""
    frames = _frames(synth, 3, seed=6)
    S = 8
    ctx = pkg.Lmot(_params(pkg))
    twins = []
    try:
        ctx.seq_open(S, ring=4)
        cfg = {0: dict(on=1), 1: dict(on=1, max_vertices=200), 2: None, 3: dict(on=1), 4: dict(on=1), 5: dict(on=1), 6: dict(on=1), 7: dict(on=1)}
        for k, o in cfg.items():
            t = pkg.Lmot(_params(pkg))
            if o:
                ctx.seq_set_obstacles(k, **o)
                t.set_obstacles(**o)
            if k == 5:
                ctx.seq_set_layers(k, on=1); t.set_layers(on=1)
            if k == 6:
                ctx.seq_set_box_search(k, on=1); t.set_box_search(on=1)
            twins.append(t)
        assert ctx.seq_get_obstacles(1) == {"on": 1, "max_vertices": 200}
        for i, (ts, p) in enumerate(frames):
            entries = []
            for k in range(S):
                if k == 3 and i == 1:
                    entries.append(None)                                             # SKIP
                elif k == 4:
                    entries.append(dict(lists=np.zeros((0, 8, 3), f32), timestamp=ts))     # LISTS
                else:
                    entries.append(dict(frames=p, timestamp=ts, restart=(k == 7 and i == 2)))
            out = ctx.seq_tick(entries)
            for k in range(S):
                if entries[k] is None or k == 4 or cfg[k] is None:
                    with pytest.raises(pkg.LmotError):
                        ctx.seq_obstacles_result(k, 0)
                    continue
                if k == 7 and i == 2:
                    twins[k].tracker_reset()
                want_r = twins[k].frame(p, ts)
                got, want = ctx.seq_obstacles_result(k, 0), twins[k].obstacles_result(0)
                assert got["status"] == want["status"] and got["n_vertices"] == want["n_vertices"]
                assert np.array_equal(got["obstacles"], want["obstacles"])
                assert np.array_equal(_bits(got["vertices"]), _bits(want["vertices"]))
                assert np.array_equal(_bits(out[k]["boxes"]), _bits(want_r["boxes"]))
        ctx.seq_open(2, ring=2)
        assert ctx.seq_get_obstacles(0) == {"on": 0, "max_vertices": 65536}
    finally:
        ctx.close()
        for t in twins:
            t.close()


# ------------------------------------------------------------------------------------------------ regimes
def test_regimes(pkg, synth, ref_intended):
    """an empty frame; max_clusters clusters; one cluster of about 110 k points; a pool that overflows; settings changed in flight;
    validation and timing mode"""
    ctx = pkg.Lmot(_params(pkg, max_points=1 << 18, max_clusters=64, pipeline_depth=4))
    try:
        ctx.set_obstacles(on=1)
        # empty frame
        ctx.frame(np.zeros((0, 4), f32), 1e6)
        res = ctx.obstacles_result(0)
        assert res["n_units"] == 1 and len(res["obstacles"]) == 0 and res["n_vertices"] == 0
        # more clusters than max_clusters: the first 64 are reported
        ts, p = _frames(synth, 1, seed=9, rings=64, azimuths=1800, n_objects=60)[0]
        e, _ = ref_intended.ground_remove(p)
        grid, k = ref_intended.component_clustering(e)
        assert k > 64
        try:
            ctx.frame(p, 2e6)
        except pkg.LmotError:
            pass                                                                   # LMOT_ERR_CAPACITY: the clusters were cut
        res = ctx.obstacles_result(0)
        ids = os_.label_ids(e, grid)
        ids[ids > 64] = 0
        want, _ = _want(ref_intended, e, ids, 64)
        got = res["obstacles"]
        assert len(got) == 64
        assert [(r["n_points"], r["n_cells"], r["vertex_count"]) for r in got] == [(w["n_points"], w["n_cells"], len(w["hull"])) for w in want]
    finally:
        ctx.close()
    # one cluster of ~110 k points: a dense 6 x 6 m block
    rng = np.random.default_rng(1)
    blk = np.concatenate([rng.uniform([4.0, 4.0, -1.2], [10.0, 10.0, 0.5], (110_000, 3)), np.ones((110_000, 1))], 1).astype(f32)
    gnd = np.concatenate([rng.uniform([-20, -20, -1.73], [20, 20, -1.72], (20_000, 3)), np.ones((20_000, 1))], 1).astype(f32)
    pts = np.concatenate([blk, gnd])
    ctx = pkg.Lmot(_params(pkg, max_points=1 << 18))
    try:
        ctx.set_obstacles(on=1)
        ctx.frame(pts, 1e6)
        e, _ = ref_intended.ground_remove(pts)
        grid, k = ref_intended.component_clustering(e)
        _assert_equal(ctx.obstacles_result(0), _want(ref_intended, e, os_.label_ids(e, grid), k)[0])
        assert ctx.obstacles_result(0)["obstacles"]["n_points"].max() > 100_000
        # pool overflow: headers intact, hulls beyond the pool get count 0, the needed total is reported
        ts, p = _frames(synth, 1, seed=9, rings=64, azimuths=1800, n_objects=40)[0]
        ctx.set_obstacles(on=1, max_vertices=140)
        ctx.frame(p, 2e6)
        small = ctx.obstacles_result(0)
        assert small["status"] == pkg.ERR_CAPACITY
        ctx.set_obstacles(on=1)
        ctx.frame(p, 2e6)
        full = ctx.obstacles_result(0)
        assert small["n_vertices"] == full["n_vertices"] > 140
        for f in ("cluster", "n_points", "n_cells", "box", "vertex_offset", "z_min", "z_max"):
            assert np.array_equal(small["obstacles"][f], full["obstacles"][f]), f
        fits = full["obstacles"]["vertex_offset"] + full["obstacles"]["vertex_count"] <= 140
        assert np.array_equal(small["obstacles"]["vertex_count"], np.where(fits, full["obstacles"]["vertex_count"], 0))
        assert np.array_equal(_bits(small["vertices"]), _bits(full["vertices"][: len(small["vertices"])]))
        # settings changed while steps are in flight: each step keeps the setting it was submitted with
        ctx.tracker_reset()
        ctx.set_obstacles(on=1)
        ctx.frame_submit(p, 3e6)
        ctx.set_obstacles()
        ctx.frame_submit(p, 3.1e6)
        ctx.set_obstacles(on=1, max_vertices=140)
        ctx.frame_submit(p, 3.2e6)
        ctx.frame_collect()
        assert ctx.obstacles_result(0)["n_vertices"] == full["n_vertices"] and ctx.obstacles_result(0)["status"] == 0
        ctx.frame_collect()
        with pytest.raises(pkg.LmotError):
            ctx.obstacles_result(0)
        ctx.frame_collect()
        assert ctx.obstacles_result(0)["status"] == pkg.ERR_CAPACITY
        # validation
        for bad in (dict(on=2), dict(on=1, max_vertices=139), dict(on=1, max_vertices=(1 << 24) + 1)):
            with pytest.raises(pkg.LmotError):
                ctx.set_obstacles(**bad)
        assert ctx.get_obstacles() == {"on": 1, "max_vertices": 140}
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_obstacles(0, on=1)                                         # no open set
        with pytest.raises(pkg.LmotError):
            ctx.obstacles_result(-1)
        # timing mode: an obstacle submission is refused, nothing submitted
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError):
            ctx.frame(p, 4e6)
        ctx.enable_timing(False)
    finally:
        ctx.close()
