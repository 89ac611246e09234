"""Scan-matched ego motion on the GPU (lmot_ego_estimate*, lmot_seq_ego_estimate*): every lmot_ego_out field bit-identical to the
restatement of tests/ego_match_scenes.py, the sequence form against own-stream contexts, the state rules, the frame pipeline untouched, and
the matched ego fed back into lmot_frame."""
import functools
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import accumulate_scenes as acs
import ego_match_scenes as em

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
f32 = np.float32
STEPS = 40


@functools.lru_cache(maxsize=None)
def _drive(kind, beams=16, movers=0, seed=3, steps=STEPS):
    import importlib
    synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
    return em.drive_frames(synth, kind, steps, beams=beams, movers=movers, seed=seed)


@functools.lru_cache(maxsize=None)
def _want(kind, beams=16, movers=0, seed=3, steps=STEPS, sensor=-1):
    poses = [_mount(j) for j in range(3)] if sensor >= 0 else None
    m = em.Matcher(dict(sensor=sensor), poses)
    return [m.estimate(_in_sensor(f[3], poses[sensor]) if poses else f[3], f[0]) for f in _drive(kind, beams, movers, seed, steps)]


def _mount(j):
    """sensor j's pose (sensor -> vehicle): a yaw of 0.1 j and an offset"""
    c, s = math.cos(0.1 * j), math.sin(0.1 * j)
    return np.array([[c, -s, 0.0, 0.3 * j], [s, c, 0.0, -0.2 * j], [0.0, 0.0, 1.0, 0.1]], f32)


def _in_sensor(p, pose):
    """the cloud as sensor `pose` would see it (the vehicle-frame cloud moved by the pose's inverse, in double then float)"""
    P = pose.astype(np.float64)
    q = p.copy()
    d = p[:, :3].astype(np.float64) - P[:, 3]
    q[:, :3] = (d @ P[:, :3]).astype(f32)
    return q


def _same(got, want, where=""):
    for k, v in want.items():
        assert got[k] == v, (where, k, got[k], v)


def _stride(p, stride):
    q = np.zeros((len(p), stride), f32)
    q[:, : min(4, stride)] = p[:, : min(4, stride)]
    return q


@pytest.mark.parametrize("kind,stride", [("straight", 3), ("turn", 4), ("turn", 5)])
def test_host_frames_bit_exact(pkg, kind, stride):
    ctx = pkg.Lmot()
    try:
        for t, (f, w) in enumerate(zip(_drive(kind), _want(kind))):
            _same(ctx.ego_estimate(_stride(f[3], stride), f[0]), w, t)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind,beams", [("straight", 32), ("turn", 16)])
def test_device_frames_bit_exact(pkg, kind, beams):
    ctx = pkg.Lmot()
    try:
        for t, (f, w) in enumerate(zip(_drive(kind, beams), _want(kind, beams))):
            d = torch.from_numpy(np.ascontiguousarray(f[3])).cuda()
            torch.cuda.current_stream().synchronize()
            _same(ctx.ego_estimate_dev(d.data_ptr(), len(f[3]), f[0]), w, t)
    finally:
        ctx.close()


def test_sensor_table_stream(pkg):
    """sensor = 2: the caller passes sensor 2's frame; the matcher moves it into the vehicle frame by the table's pose"""
    ctx = pkg.Lmot()
    try:
        ctx.set_sensors([_mount(j) for j in range(3)])
        ctx.set_ego_match(sensor=2)
        pose = _mount(2)
        for t, (f, w) in enumerate(zip(_drive("turn"), _want("turn", sensor=2))):
            _same(ctx.ego_estimate(_in_sensor(f[3], pose), f[0]), w, t)
        ctx.set_ego_match(sensor=3)                                 # no fourth sensor
        with pytest.raises(pkg.LmotError):
            ctx.ego_estimate(_drive("turn")[0][3], 1e9)
    finally:
        ctx.close()


SEQ_DRIVES = [("straight", 16, 0, 3), ("turn", 16, 0, 3), ("straight", 32, 0, 4), ("turn", 32, 12, 5),
              ("turn", 16, 0, 6), ("straight", 16, 12, 7), ("turn", 32, 0, 3), ("straight", 32, 0, 8)]


def test_eight_sequences_equal_eight_contexts(pkg):
    """one lmot_seq_ego_estimate_dev over 8 sequences (some with their own settings) == 8 own-stream contexts; a NULL entry leaves its
    sequence untouched (its next frame still matches against the frame before the skip)"""
    n = 12
    frames = [_drive(k, b, m, s, n) for k, b, m, s in SEQ_DRIVES]
    cfg = [dict(), dict(refine=1), dict(yaw_half=10, shift_half=20), dict(max_points=300, min_points=100), dict(grid=512),
           dict(cell_m=0.15, sub_m=0.5), dict(refine=3, yaw_step=0.004), dict(min_score_frac=0.6)]
    skip = {(1, 3), (4, 5), (4, 6), (7, 0)}
    seq, own = pkg.Lmot(), [pkg.Lmot() for _ in range(8)]
    try:
        seq.seq_open(8, ring=2)
        for k in range(8):
            if cfg[k]:
                seq.seq_set_ego_match(k, **cfg[k])
                own[k].set_ego_match(**cfg[k])
                assert seq.seq_get_ego_match(k) == own[k].get_ego_match()
        for t in range(n):
            dev = [torch.from_numpy(np.ascontiguousarray(frames[k][t][3])).cuda() for k in range(8)]
            torch.cuda.synchronize()
            ptrs = [None if (k, t) in skip else dev[k].data_ptr() for k in range(8)]
            got = seq.seq_ego_estimate_dev(ptrs, [len(frames[k][t][3]) for k in range(8)], [frames[k][t][0] for k in range(8)])
            for k in range(8):
                if (k, t) in skip:
                    assert got[k] is None
                    continue
                _same(got[k], own[k].ego_estimate(frames[k][t][3], frames[k][t][0]), (k, t))
    finally:
        seq.close()
        for c in own:
            c.close()


def test_state_rules(pkg):
    fr = _drive("straight")
    ctx = pkg.Lmot()
    try:
        o = ctx.ego_estimate(fr[0][3], fr[0][0])
        assert (o["ok"], o["v"], o["dtheta"], o["yaw"], o["score"], o["n_ref"]) == (0, 0.0, 0.0, 0.0, 0, 0) and o["n_used"] > 0
        o = ctx.ego_estimate(fr[1][3], fr[1][0])
        assert o["ok"] == 1 and abs(o["v"] - 4.0) < 0.5 and o["n_ref"] > 0
        for ts in (fr[1][0], fr[1][0] - 1.0, float("nan")):                  # dt <= 0 or not finite: v = 0, nothing matched
            o = ctx.ego_estimate(fr[2][3], ts)
            assert (o["ok"], o["v"], o["dtheta"], o["score"]) == (0, 0.0, 0.0, 0)
        ctx.set_ego_match(min_points=8192)                                  # below min_points: the prior (constant velocity)
        m = em.Matcher(dict(min_points=8192))
        for f in fr[:4]:
            _same(ctx.ego_estimate(f[3], f[0]), m.estimate(f[3], f[0]))
        ctx.set_ego_match()                                                 # a setting resets: the next call is a first call
        o = ctx.ego_estimate(fr[5][3], fr[5][0])
        assert (o["ok"], o["v"], o["yaw"]) == (0, 0.0, 0.0)
        ctx.ego_estimate(fr[6][3], fr[6][0])
        ctx.ego_reset()
        o = ctx.ego_estimate(fr[7][3], fr[7][0])
        assert (o["ok"], o["v"], o["yaw"]) == (0, 0.0, 0.0)
        o = ctx.ego_estimate(np.zeros((0, 4), f32), fr[8][0])              # an empty frame: no match, the prior
        assert (o["n_used"], o["ok"]) == (0, 0)
        # validation agrees with the restatement, and a refused setting changes nothing
        ctx.set_ego_match(refine=3)
        d = em.defaults()
        for b in (dict(grid=16), dict(grid=100), dict(cell_m=float("nan")), dict(z_min=1.0, z_max=1.0), dict(r_min=40.0),
                  dict(sub_m=0.01), dict(max_points=9000), dict(yaw_step=0.2), dict(shift_half=128), dict(refine=0), dict(sensor=8)):
            assert not em.valid(dict(d, **b))
            with pytest.raises(pkg.LmotError):
                ctx.set_ego_match(**b)
            assert ctx.get_ego_match()["refine"] == 3
        ctx.seq_open(2, ring=2)
        ctx.seq_set_ego_match(1, grid=256)
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_ego_match(2, grid=256)
        ctx.seq_ego_estimate([fr[0][3], fr[0][3]], [fr[0][0]] * 2)
        ctx.seq_ego_reset(0)
        ctx.seq_open(2, ring=2)                                             # reopening: every sequence back to the defaults
        assert ctx.seq_get_ego_match(1) == pkg.default_ego_match()
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError):
            ctx.ego_estimate(fr[0][3], fr[0][0])
    finally:
        ctx.close()


_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
P = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)][0]
out = {}
for arm in ("never", "used"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p)
    ctx.seq_open(4, ring=4)
    d = torch.from_numpy(P).cuda(); torch.cuda.synchronize()
    if arm == "used":
        ctx.ego_estimate(P, 1.0); ctx.seq_ego_estimate([P, None, P, None], [1.0] * 4)
    def run(t):
        ctx.frame(P, t)
        ctx.frame_dev(d.data_ptr(), len(P), t + 1e5); ctx.frame_fetch()
        ctx.batch([P, P], t + 2e5)
        ctx.seq([P] * 4, [t] * 4)
        torch.cuda.synchronize()
    for w in range(4):
        run(1e6 + w * 1e6)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(9e6)
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    if arm == "used":
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.ego_estimate(P, 2e5)
        out["estimate"] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    ctx.close()
print(json.dumps(out))
"""


def test_frame_pipeline_launches_unchanged():
    """a context that never estimates issues no matcher work, and estimation leaves the frame path's launches as they were"""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    assert n["never"] and not any("ego_" in x for x in n["never"])
    assert sorted(n["never"]) == sorted(n["used"])
    ks = [x for x in n["estimate"] if "kernel" in x]
    for k in ("ego_clear_kernel", "ego_band_kernel", "ego_field_kernel", "ego_sample_kernel", "ego_coarse_kernel", "ego_fine_kernel"):
        assert sum(k in x for x in ks) == 1, ks


def test_interleaved_with_pipelined_frames(pkg, synth):
    """estimates between pipelined lmot_frame_dev calls leave every frame result bit-identical"""
    frames = [p for _, p in synth.frames(synth.SceneConfig(seed=2, rings=32, azimuths=900), 12)]
    res = {}
    for arm in ("plain", "interleaved"):
        ctx = pkg.Lmot()
        try:
            dev = [torch.from_numpy(p).cuda() for p in frames]
            torch.cuda.synchronize()
            got, est = [], []
            for t, d in enumerate(dev):
                ts = (t + 1) * 1e5
                ctx.frame_dev(d.data_ptr(), len(frames[t]), ts, 1.0, 0.01 * t)
                if arm == "interleaved":
                    est.append(ctx.ego_estimate_dev(d.data_ptr(), len(frames[t]), ts))
                if t >= 3:
                    got.append(ctx.frame_collect())
            while ctx.frames_in_flight():
                got.append(ctx.frame_collect())
            res[arm] = got
        finally:
            ctx.close()
    assert len(res["plain"]) == len(res["interleaved"]) == 12
    for a, b in zip(res["plain"], res["interleaved"]):
        for k in ("n_elevated", "n_ground", "num_cluster"):
            assert a[k] == b[k]
        for k in ("boxes", "targets", "vandyaw", "track_manage", "is_static"):
            assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def _end_to_end(pkg, kind, beams, ego, accumulate):
    frames = _drive(kind, beams)
    ctx = pkg.Lmot()
    try:
        if accumulate:
            ctx.set_accumulate(sweeps=4)
        static, hits = 0, 0
        for (ts, _, _, pts, _, objs), (v, yaw) in zip(frames, ego):
            r = ctx.frame(pts, ts, v, yaw)
            static += int(np.sum(np.asarray(r["is_static"]) == 1))
            hits += acs.hits(r["boxes"], objs)
        return static, hits, ctx.tracker_get_ego()[5:8].copy()
    finally:
        ctx.close()


@pytest.mark.parametrize("kind,beams", [("straight", 32), ("turn", 32)])
def test_matched_ego_through_the_pipeline(pkg, kind, beams):
    """lmot_frame fed the matched (v, yaw): the fold is the restatement's fold of those values and ends far closer to the GPS fold than
    v = 0 does (scripts/ego_match_premise.py: 0.40 / 0.37 m against 15.6 / 10.5 m after 40 steps); the static flags equal GPS ego's, as
    in the premise; with accumulation the static objects register about as often as with GPS ego"""
    frames = _drive(kind, beams)
    ctx = pkg.Lmot()
    try:
        matched = [(o["v"], o["yaw"]) for o in (ctx.ego_estimate(f[3], f[0]) for f in frames)]
    finally:
        ctx.close()
    assert matched == [(w["v"], w["yaw"]) for w in _want(kind, beams)]
    gps = [(f[1], f[2]) for f in frames]
    zero = [(0.0, 0.0)] * len(frames)
    runs = {name: _end_to_end(pkg, kind, beams, ego, False) for name, ego in (("gps", gps), ("matched", matched), ("v0", zero))}
    h = dict(init=False, ts=0.0, pre_yaw=0.0, fold=None)
    for f, (v, yaw) in zip(frames, matched):
        want_fold = em.fold_step(h, f[0], v, yaw)
    assert np.array_equal(runs["matched"][2], want_fold)
    fg = runs["gps"][2]
    err_m = math.hypot(*(runs["matched"][2][:2] - fg[:2]))
    err_0 = math.hypot(*(runs["v0"][2][:2] - fg[:2]))
    assert err_m < 0.1 * err_0 and err_m < 1.0, (err_m, err_0)
    assert runs["matched"][0] == runs["gps"][0]
    acc = {name: _end_to_end(pkg, kind, beams, ego, True)[1] for name, ego in (("gps", gps), ("matched", matched))}
    assert acc["matched"] >= 0.8 * acc["gps"], acc
    print(json.dumps(dict(kind=kind, beams=beams, static={k: v[0] for k, v in runs.items()}, fold_err_matched=err_m, fold_err_v0=err_0,
                          acc_hits=acc)))
