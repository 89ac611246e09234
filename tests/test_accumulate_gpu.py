"""Sweep accumulation on the device (include/lmot.h, lmot_set_accumulate): an accumulating context equals, bit for bit, a plain twin context
that builds E_acc in NumPy from its own ground removal and lmot_accumulate_pose, clusters and boxes it through the stage entry points and
steps its tracker on those boxes.  Plus the cuts, the reset rules, the reference's detection on E_acc, the untouched off path and the
value on a sparse 16-beam scene."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from accumulate_scenes import e_acc, hits, sparse_frames

pytestmark = pytest.mark.gpu
f32 = np.float32


def _params(pkg, gf=0, depth=None, max_points=1 << 17):
    p = pkg.default_params()
    p.max_points = max_points
    p.global_frame = gf
    if depth:
        p.pipeline_depth = depth
    return p


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _same_tracks(a, b):
    for k in ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb"):
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k


class Twin:
    """the definition through the stage entry points of a plain context"""

    def __init__(self, pkg, params, sweeps, max_age_s):
        self.ctx = pkg.Lmot(params)
        self.K, self.age, self.cap = sweeps, max_age_s, int(params.max_points)
        self.hist = []

    def step(self, pts, ts, v, yaw, ref=None):
        c = self.ctx
        e_t = c.ground_remove(pts)["elevated"]
        fold_t = c.origin_points(ts, v, yaw)[:3].copy()
        acc, used = e_acc(e_t, ts, fold_t, self.hist, self.age, self.cap)
        grid, k = c.component_cluster(acc)
        outs = c.cluster_outputs()
        boxes, _ = c.box_fit(acc, grid, k)
        if ref is not None:
            g2, k2 = ref.component_clustering(acc)
            b2, _ = ref.box_fitting(acc, g2, k2)
            assert k2 == k and np.array_equal(_bits(b2), _bits(boxes)), "reference detection on E_acc"
        tr = c.track_step(boxes, ts, v, yaw)
        self.record(e_t, ts, fold_t)
        return dict(n_elevated=len(e_t), num_cluster=k, boxes=boxes, n_points=len(acc), used=used, outs=outs, **tr)

    def record(self, e_t, ts, fold_t):
        """E_t joins the history with the fold read after the step (ego8[5..7]); lmot_origin_points peeked the same before it, except on
        a table's first step (no history to move then)"""
        f = self.ctx.tracker_get_ego()[5:8].copy()
        assert not self.hist or np.array_equal(f, fold_t)
        self.hist = ([(e_t, ts, f)] + self.hist)[: self.K - 1]

    def close(self):
        self.ctx.close()


def _check(got, want, info):
    assert got["n_elevated"] == want["n_elevated"] and got["num_cluster"] == want["num_cluster"]
    assert np.array_equal(_bits(got["boxes"]), _bits(want["boxes"]))
    _same_tracks(got, want)
    assert len(info) == 1
    u = info[0]
    assert u["n_points"] == want["n_points"] and u["sweeps_used"] == len(want["used"])
    for j, (ts_s, D) in enumerate(want["used"]):
        assert u["stamp_us"][j] == ts_s
        assert np.array_equal(u["pose"][j].view(np.uint32), D.view(np.uint32))


SCHEDULES = {
    # name: (sweeps, max_age_s, max_points, stamp step of each frame in units of 0.1 s (0: the same stamp again, -1: back in time))
    "turn_k4": (4, 0.5, 1 << 17, [1] * 12),
    "age_cut": (6, 0.25, 1 << 17, [1, 1, 3, 1, 1, 1, 2, 1, 1, 1]),
    "stamp_back": (4, 0.5, 1 << 17, [1, 1, 1, 0, 1, -1, 1, 1, 1]),
    "points_cut": (8, 1.0, 20000, [1] * 12),
}


@pytest.mark.parametrize("name", sorted(SCHEDULES))
def test_frame_equals_twin(pkg, synth, name, ref_intended):
    """lmot_frame frame by frame, with cluster outputs and the reference's detection on E_acc"""
    K, age, cap, steps = SCHEDULES[name]
    frames = sparse_frames(pkg, synth, "turn", len(steps))
    p = _params(pkg, max_points=cap)
    a, b = pkg.Lmot(p), Twin(pkg, _params(pkg, max_points=cap), K, age)
    try:
        a.set_accumulate(sweeps=K, max_age_s=age)
        assert a.get_accumulate() == dict(sweeps=K, max_age_s=age)
        ts = 0.0
        used = []
        for (_, v, yaw, pts, _, _), s in zip(frames, steps):
            ts += s * 1e5
            got = a.frame(pts, ts, v, yaw)
            want = b.step(pts, ts, v, yaw, ref_intended)
            _check(got, want, a.accumulate_info())
            cl, ob, cm = a.cluster_outputs()
            for x, y in zip((cl, ob, cm), want["outs"]):
                assert np.array_equal(_bits(x), _bits(y)), "cluster outputs of E_acc"
            used.append(len(want["used"]))
        assert np.array_equal(a.tracker_dump(), b.ctx.tracker_dump())
        assert max(used) > 0
        if name == "points_cut":
            assert max(used) < K - 1
    finally:
        a.close(); b.close()


AREA = [np.array([[-20.0, -20.0], [20.0, -20.0], [20.0, 20.0], [-20.0, 20.0]])]


def _twin_masked(pkg, b, pts, ts, v, yaw):
    """the twin step with a detection area: E_acc filtered by the unit's mask before clustering (step 4)"""
    from detect_area_scenes import area_filter
    c = b.ctx
    e_t = c.ground_remove(pts)["elevated"]
    fold_t = c.origin_points(ts, v, yaw)[:3].copy()
    acc, used = e_acc(e_t, ts, fold_t, b.hist, b.age, b.cap)
    kept = area_filter(acc, pkg.detect_area_mask(AREA))
    grid, k = c.component_cluster(kept)
    boxes, _ = c.box_fit(kept, grid, k)
    tr = c.track_step(boxes, ts, v, yaw)
    b.record(e_t, ts, fold_t)
    return dict(n_elevated=len(e_t), num_cluster=k, boxes=boxes, n_points=len(acc), used=used, **tr)


@pytest.mark.parametrize("mode", ["submit_depth4_k8", "dev_global_frame", "area_retire"])
def test_pipelined_equals_twin(pkg, synth, mode):
    """lmot_frame_submit at pipeline_depth 4 with K = 8 (sweeps cross slot reuse), lmot_frame_dev with global_frame 1, and accumulation
    with a detection area and retirement on one stream"""
    import torch
    frames = sparse_frames(pkg, synth, "turn", 14)
    K = 8 if mode.startswith("submit") else 4
    gf = 1 if mode == "dev_global_frame" else 0
    a = pkg.Lmot(_params(pkg, gf, depth=4))
    b = Twin(pkg, _params(pkg, gf), K, 1.0)
    try:
        a.set_accumulate(sweeps=K, max_age_s=1.0)
        if mode == "area_retire":
            a.set_detect_area(AREA)
            a.set_track_retirement(True)
            b.ctx.set_track_retirement(True)
        want, got, infos, dev = [], [], [], []
        for ts, v, yaw, pts, _, _ in frames:
            if mode == "dev_global_frame":
                d = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
                dev.append(d)
                torch.cuda.synchronize()
                a.frame_dev(d.data_ptr(), len(pts), ts, v, yaw)
                got.append(a.frame_fetch())
                infos.append(a.accumulate_info())
            else:
                a.frame_submit(pts, ts, v, yaw)
                if a.frames_in_flight() >= 4:
                    got.append(a.frame_collect())
                    infos.append(a.accumulate_info())
            want.append(_twin_masked(pkg, b, pts, ts, v, yaw) if mode == "area_retire" else b.step(pts, ts, v, yaw))
        while a.frames_in_flight() > 0:
            got.append(a.frame_collect())
            infos.append(a.accumulate_info())
        assert len(got) == len(want)
        for g, w, inf in zip(got, want, infos):
            _check(g, w, inf)
        if mode == "area_retire":
            assert np.array_equal(a.track_ids(), b.ctx.track_ids())
        assert np.array_equal(a.tracker_dump(), b.ctx.tracker_dump())
    finally:
        a.close(); b.close()


def test_reset_rules_and_errors(pkg, synth):
    frames = sparse_frames(pkg, synth, "straight", 8)
    a = pkg.Lmot(_params(pkg))
    try:
        for bad in (dict(sweeps=0), dict(sweeps=9), dict(max_age_s=0.0), dict(max_age_s=float("nan")), dict(max_age_s=-1.0)):
            with pytest.raises(pkg.LmotError):
                a.set_accumulate(**bad)
        assert a.get_accumulate() == dict(sweeps=1, max_age_s=0.5)
        a.set_accumulate(sweeps=3)
        used = lambda: a.accumulate_info()[0]["sweeps_used"]
        seq = iter(frames)

        def step():
            ts, v, yaw, pts, _, _ = next(seq)
            a.frame(pts, ts, v, yaw)
            return used()

        assert step() == 0 and step() == 1 and step() == 2
        a.tracker_reset()
        assert step() == 0 and step() == 1
        a.set_sensors(None)
        assert step() == 0
        a.set_accumulate(sweeps=3)
        assert step() == 0
        ts, v, yaw, pts, _, _ = frames[0]
        a.enable_timing(True)
        for call in (lambda: a.frame(pts, ts + 2e7, v, yaw), lambda: a.batch([pts, pts], ts + 2e7, v, yaw)):
            with pytest.raises(pkg.LmotError) as e:
                call()
            assert e.value.status == pkg.ERR_STATE
        a.enable_timing(False)
        a.set_accumulate()
        a.frame(pts, ts + 3e7, v, yaw)
        assert a.accumulate_info() == []
    finally:
        a.close()


_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
P = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)][0]
out = {}
for arm in ("never", "one", "four"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p)
    if arm == "one": ctx.set_accumulate(sweeps=1)
    if arm == "four": ctx.set_accumulate(sweeps=4)
    d = torch.from_numpy(P).cuda(); torch.cuda.synchronize()
    res = []
    def run(t):
        res.append(ctx.frame(P, t))
        ctx.frame_dev(d.data_ptr(), len(P), t + 1e5); res.append(ctx.frame_fetch())
        torch.cuda.synchronize()
    run(1e6)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(1.2e6)
    out[arm] = dict(names=[e.name for e in prof.events() if str(e.device_type).endswith("CUDA")],
                    boxes=[r["boxes"].tobytes().hex() for r in res], tm=[r["track_manage"].tolist() for r in res])
    ctx.close()
print(json.dumps(out))
"""


def test_off_is_todays_path(pkg):
    """sweeps = 1 gives a context that never set the option: the same results and the same kernels, copies and memsets; K = 4 adds
    accumulate_kernel"""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    assert n["never"]["names"] and not any("accumulate" in x for x in n["never"]["names"])
    assert sorted(n["never"]["names"]) == sorted(n["one"]["names"])
    assert n["never"]["boxes"] == n["one"]["boxes"] and n["never"]["tm"] == n["one"]["tm"]
    assert any("accumulate_kernel" in x for x in n["four"]["names"])


def test_sparse_value(pkg, synth, capsys):
    """(frame, static object) pairs with a box centre within 1 m, K = 4 against K = 1, straight driving and a turn"""
    tot = {}
    for K in (1, 4):
        tot[K] = 0
        for kind in ("straight", "turn"):
            frames = sparse_frames(pkg, synth, kind, 16)
            a = pkg.Lmot(_params(pkg))
            try:
                a.set_accumulate(sweeps=K)
                for ts, v, yaw, pts, _, objs in frames:
                    tot[K] += hits(a.frame(pts, ts, v, yaw)["boxes"], objs)
            finally:
                a.close()
    with capsys.disabled():
        print(f"\nsparse 16-beam scene, (frame, static object) pairs with a box within 1 m: K=1 {tot[1]}, K=4 {tot[4]}")
    assert tot[4] > tot[1], tot
