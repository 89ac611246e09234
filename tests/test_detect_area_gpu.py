"""Detection areas on the device (include/lmot.h, lmot_set_detect_area): every masked unit's cell mask equals lmot_detect_area_mask, and a
masked step equals the reference's groundRemove, the E_area filter, componentClustering and boxFitting, then the tracker on those boxes --
through lmot_frame / _submit / _dev, batched rigs (separate and merging) and sequence ticks.  Unmasked submissions run today's kernels."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from detect_area_scenes import CORRIDOR, area_filter, cluttered_frames, mask_ref, near_clutter, rect, ref_detect_area
from test_sensor_rig_gpu import rig_apply, yaw_pose

pytestmark = pytest.mark.gpu
f32 = np.float32

AREA = [np.array([[-20.0, -6.0], [18.0, -9.0], [21.0, 7.5], [2.0, 3.0], [-17.0, 10.0]]), rect(-4.0, -2.0, 3.0, 1.5)]


def _params(pkg, gf=0):
    p = pkg.default_params()
    p.max_points = 1 << 17
    p.global_frame = gf
    return p


def _frames(synth, n, seed=5):
    return [(ts, p) for ts, p in synth.frames(synth.SceneConfig(seed=seed, rings=32, azimuths=900, n_objects=30), n)]


def _bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _same_frame(a, b):
    for k in ("n_elevated", "n_ground", "num_cluster"):
        assert a[k] == b[k], k
    assert np.array_equal(_bits(a["boxes"]), _bits(b["boxes"]))
    for k in ("targets", "track_manage", "is_static", "is_vis", "vis_bb"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


# ------------------------------------------------------------------------------------------------ today's path
_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
P = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)][0]
sq = [np.array([[-10.0, -5.0], [10.0, -5.0], [10.0, 5.0], [-10.0, 5.0]])]
out = {}
for arm in ("off", "on_then_off", "on"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p)
    ctx.seq_open(4, ring=4)
    if arm != "off":
        ctx.set_detect_area(sq); ctx.seq_set_detect_area(1, sq)
    if arm == "on_then_off":
        ctx.set_detect_area(None); ctx.seq_set_detect_area(1, None)
    d = torch.from_numpy(P).cuda(); torch.cuda.synchronize()
    def run(t):
        ctx.frame(P, t)
        ctx.frame_dev(d.data_ptr(), len(P), t + 1e5); ctx.frame_fetch()
        ctx.batch([P, P], t + 2e5)
        ctx.seq([P] * 4, [t] * 4)
        torch.cuda.synchronize()
    run(1e6)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(2e6)
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    ctx.close()
print(json.dumps(out))
"""


def test_off_is_todays_path(pkg, synth):
    """an area set and cleared again leaves the same results and the same kernels, copies and memsets; a masked context adds
    detect_area_kernel and the masking variants"""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    assert n["off"] and not any("area" in x for x in n["off"]), n["off"]
    assert sorted(n["off"]) == sorted(n["on_then_off"])
    for k in ("detect_area_kernel", "ccl_area_kernel", "tile_hist_area_kernel"):
        assert any(k in x for x in n["on"]), k
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_detect_area(AREA)
        b.set_detect_area([])
        assert b.get_detect_area()["rings"] == []
        for ts, p in _frames(synth, 4):
            _same_frame(a.frame(p, ts), b.frame(p, ts))
            assert len(b.debug_area_masks()) == 0
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ masks
def test_device_masks_equal_host(pkg, synth):
    """frame path (identity, roi 50 and 30) and a 4-sensor rig (each sensor's own pose) against lmot_detect_area_mask and the restatement"""
    P = _frames(synth, 1)[0][1]
    for roi, ko in ((50.0, False), (30.0, True)):
        p = _params(pkg)
        p.roi_m = roi
        ctx = pkg.Lmot(p)
        try:
            ctx.set_detect_area(AREA, ko)
            ctx.frame(P, 1e5)
            got = ctx.debug_area_masks()
            assert got.shape == (1, 250, 8)
            assert np.array_equal(got[0], pkg.detect_area_mask(AREA, ko, None, roi))
            assert np.array_equal(got[0], mask_ref(AREA, ko, None, roi))
        finally:
            ctx.close()
    rig = [yaw_pose(1, 0, 1.5, 0.2, 0), yaw_pose(0, 1, -0.5, 1.0, 0), yaw_pose(-1, 0, -2.0, -0.3, 0), yaw_pose(0, -1, 0.4, -1.2, 0)]
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_sensors(rig)
        ctx.set_detect_area(AREA)
        ctx.batch([P] * 4, 1e5)
        got = ctx.debug_area_masks()
        assert got.shape == (4, 250, 8)
        for j in range(4):
            assert np.array_equal(got[j], pkg.detect_area_mask(AREA, False, rig[j], 50.0)), j
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ frames against the reference
@pytest.mark.parametrize("keep_outside", [False, True])
@pytest.mark.parametrize("gf", [0, 1])
def test_frames_against_reference(pkg, synth, ref_intended, keep_outside, gf):
    """lmot_frame, pipelined lmot_frame_submit and lmot_frame_dev: counts, clouds, num_cluster and boxes against the reference on E_area;
    tracks against a twin context stepped with lmot_track_step on the reference's boxes, and (global_frame 0) the reference's tracker"""
    import torch
    ref = ref_intended
    mask = pkg.detect_area_mask(AREA, keep_outside)
    frames = _frames(synth, 6)
    exp = [ref_detect_area(ref, p, mask) for _, p in frames]
    ctxs = [pkg.Lmot(_params(pkg, gf)) for _ in range(4)]
    sync, piped, dev, twin = ctxs
    try:
        for c in (sync, piped, dev):
            c.set_detect_area(AREA, keep_outside)
        ref.tracker_reset()
        got_sync = []
        for (ts, p), (cnt, b, _, _) in zip(frames, exp):
            r = sync.frame(p, ts)
            assert (r["n_elevated"], r["n_ground"], r["num_cluster"], len(r["boxes"])) == cnt
            assert np.array_equal(_bits(r["boxes"]), _bits(b))
            t = twin.track_step(b, ts)
            for k in ("targets", "track_manage", "is_static", "is_vis", "vis_bb"):
                assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(t[k]).view(np.uint8)), k
            if gf == 0:
                w = ref.tracker_step(b, ts)
                assert np.array_equal(r["track_manage"], w["track_manage"])
                assert np.allclose(r["targets"], w["targets"], rtol=1e-4, atol=1e-4)
            got_sync.append(r)
        for ts, p in frames:
            piped.frame_submit(p, ts)
        for r in got_sync:
            _same_frame(piped.frame_collect(), r)
        d = [torch.from_numpy(p).cuda() for _, p in frames]
        torch.cuda.synchronize()
        for (ts, p), x in zip(frames, d):
            dev.frame_dev(x.data_ptr(), len(p), ts)
        _same_frame(dev.frame_fetch(), got_sync[-1])
    finally:
        for c in ctxs:
            c.close()


def test_full_area_equals_no_area(pkg, synth):
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_detect_area([rect(-1000.0, -1000.0, 1000.0, 1000.0)])
        for ts, p in _frames(synth, 5):
            _same_frame(a.frame(p, ts), b.frame(p, ts))
            assert b.debug_area_masks()[0][:, :7].min() == 0xFFFFFFFF
    finally:
        a.close(); b.close()


def test_cluster_outputs_after_masked_frame(pkg, synth, ref_intended):
    ref = ref_intended
    mask = pkg.detect_area_mask(AREA)
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_detect_area(AREA)
        for ts, p in _frames(synth, 3):
            ctx.frame(p, ts)
            _, _, ea, grid = ref_detect_area(ref, p, mask)
            cl_r, ob_r, cm_r = ref.cluster_outputs(ea, grid)
            cl, ob, cm = ctx.cluster_outputs()
            assert cl.shape[0] == cl_r.shape[0] and np.array_equal(cl[:, :3].view(np.uint32), cl_r.view(np.uint32))
            assert ob.shape[0] == ob_r.shape[0] and ob.shape[0] > 50
            assert np.array_equal(ob[:, :3].astype(np.float64), ob_r[:, :3]) and np.array_equal(ob[:, 3].astype(np.int64), ob_r[:, 3].astype(np.int64))
            assert np.array_equal(cm, cm_r)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ rigs
def _rig4():
    return [yaw_pose(1, 0, 1.0, 0.0, 0), yaw_pose(0, 1, 0.0, 0.8, 0), yaw_pose(-1, 0, -1.0, 0.0, 0), yaw_pose(0, -1, 0.0, -0.8, 0)]


def test_rigs(pkg, synth, ref_intended):
    """a non-merging 4-sensor rig (each sensor's mask in its own frame) and a merging one, through lmot_batch and pipelined lmot_batch_dev"""
    import torch
    ref = ref_intended
    rig = _rig4()
    ticks = [((i + 1) * 1e5, [_frames(synth, 1, seed=40 + 4 * i + j)[0][1] for j in range(4)]) for i in range(3)]
    for merge in (False, True):
        a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
        try:
            for c in (a, b):
                c.set_sensors(rig)
                c.set_rig_merge(merge)
                c.set_detect_area(AREA)
            want = []
            for ts, fr in ticks:
                if merge:
                    E = np.concatenate([rig_apply(rig[j], ref.ground_remove(fr[j])[0]) for j in range(4)]).astype(f32)
                    ea = area_filter(E, pkg.detect_area_mask(AREA))
                    grid, k = ref.component_clustering(ea)
                    bx, _ = ref.box_fitting(ea, grid, k)
                else:
                    bx = np.concatenate([rig_apply(rig[j], ref_detect_area(ref, fr[j], pkg.detect_area_mask(AREA, False, rig[j]))[1])
                                         for j in range(4)]).astype(f32).reshape(-1, 8, 3)
                r = a.batch(fr, ts)
                assert np.array_equal(_bits(r["boxes"]), _bits(bx)), (merge, ts)
                want.append(r)
            dev = [[torch.from_numpy(p).cuda() for p in fr] for _, fr in ticks]
            torch.cuda.synchronize()
            for (ts, fr), d in zip(ticks, dev):
                b.batch_dev([(x.data_ptr(), len(p)) for x, p in zip(d, fr)], ts)
            r = b.batch_fetch()
            assert np.array_equal(_bits(r["boxes"]), _bits(want[-1]["boxes"]))
            assert np.array_equal(r["track_manage"], want[-1]["track_manage"])
        finally:
            a.close(); b.close()


# ------------------------------------------------------------------------------------------------ sequences
def test_sequences_equal_twins(pkg, synth):
    """six sequences, eight frames a tick (the most one tick holds): areas on some, with and without tables, merge, own detection values
    and deskew; lmot_seq and lmot_seq_tick with SKIP, RESTART and LISTS -- every sequence identical to a twin context fed its steps"""
    rig2 = [yaw_pose(1, 0, 1.0, 0.0, 0), yaw_pose(-1, 0, -1.0, 0.0, 0)]
    area_b = [rect(-15.0, -5.0, 15.0, 5.0)]
    setup = [dict(), dict(area=AREA, deskew=True), dict(area=area_b, keep=True), dict(area=AREA, det=dict(roi_m=40.0)),
             dict(area=AREA, rig=rig2), dict(area=area_b, rig=rig2, merge=True)]
    S = len(setup)
    nf = [2 if "rig" in s else 1 for s in setup]
    ctx = pkg.Lmot(_params(pkg))
    twins = []
    try:
        ctx.seq_open(S, ring=4)
        for k, s in enumerate(setup):
            tp = _params(pkg)
            if "det" in s:
                tp.roi_m = s["det"]["roi_m"]
            t = pkg.Lmot(tp)
            if "rig" in s:
                ctx.seq_set_sensors(k, s["rig"]); t.set_sensors(s["rig"])
                ctx.seq_set_rig_merge(k, s.get("merge", False)); t.set_rig_merge(s.get("merge", False))
            if "det" in s:
                ctx.seq_set_detect_params(k, **s["det"])
            if "deskew" in s:
                ctx.seq_set_deskew(k, on=1, time_field=3, t_min=-0.1, t_max=0.0); t.set_deskew(on=1, time_field=3, t_min=-0.1, t_max=0.0)
            if "area" in s:
                ctx.seq_set_detect_area(k, s["area"], s.get("keep", False)); t.set_detect_area(s["area"], s.get("keep", False))
            twins.append(t)
        pool = [p for _, p in _frames(synth, 6, seed=9)]
        for tick in range(6):
            ts = (tick + 1) * 1e5
            fr = [[pool[(tick + k + j) % 6] for j in range(nf[k])] for k in range(S)]
            if tick < 2:
                out = ctx.seq([fr[k] if nf[k] > 1 else fr[k][0] for k in range(S)], [ts] * S)
                kinds = ["frames"] * S
            else:
                kinds = [("skip" if (k + tick) % 4 == 0 else "lists" if (k + tick) % 5 == 0 and nf[k] == 1 else "frames") for k in range(S)]
                ents = []
                for k in range(S):
                    if kinds[k] == "skip":
                        ents.append(None)
                    elif kinds[k] == "lists":
                        ents.append(dict(lists=[np.zeros((0, 8, 3), f32)] * nf[k], timestamp=ts))
                    else:
                        ents.append(dict(frames=fr[k] if nf[k] > 1 else fr[k][0], timestamp=ts, restart=(tick == 4 and k == 1)))
                out = ctx.seq_tick(ents)
            for k in range(S):
                if kinds[k] == "skip":
                    continue
                t = twins[k]
                if kinds[k] == "lists":
                    w = t.track_step(np.zeros((0, 8, 3), f32), ts)
                else:
                    if tick == 4 and k == 1:
                        t.tracker_reset()
                    w = t.batch(fr[k], ts) if nf[k] > 1 else t.frame(fr[k][0], ts)
                    assert np.array_equal(_bits(out[k]["boxes"]), _bits(w["boxes"])), (tick, k)
                assert np.array_equal(out[k]["track_manage"], w["track_manage"]), (tick, k)
                assert np.array_equal(_bits(out[k]["targets"]), _bits(w["targets"])), (tick, k)
        assert ctx.seq_get_detect_area(1)["rings"][0].shape == AREA[0].shape
        ctx.seq_open(S, ring=4)
        assert all(ctx.seq_get_detect_area(k)["rings"] == [] for k in range(S))
    finally:
        ctx.close()
        for t in twins:
            t.close()


def test_area_changes_every_tick_in_flight(pkg, synth):
    """a moving vehicle: the corridor moves every frame; pipelined submissions keep the area they were submitted with"""
    frames = _frames(synth, 8)
    areas = [[rect(-20.0 + 2 * f, -6.0 - 0.5 * f, 20.0 + f, 6.0)] for f in range(8)]
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        want = []
        for (ts, p), ar in zip(frames, areas):
            a.set_detect_area(ar)
            want.append(a.frame(p, ts))
        for (ts, p), ar in zip(frames, areas):
            b.set_detect_area(ar)
            b.frame_submit(p, ts)
        for w in want:
            _same_frame(b.frame_collect(), w)
    finally:
        a.close(); b.close()


def test_clutter_scene(pkg, synth):
    """roadside poles and hedges: boxes and tracks without the area; none of either once the road corridor is the area"""
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_detect_area(CORRIDOR)
        clutter_boxes = 0
        for ts, p in cluttered_frames(synth, 6):
            ra, rb = a.frame(p, ts), b.frame(p, ts)
            clutter_boxes += int(near_clutter(ra["boxes"]).sum())
            assert not near_clutter(rb["boxes"]).any()
            tg = np.asarray(rb["targets"]).reshape(-1, 3)
            assert (np.abs(tg[:, 1]) < 8.0).all(), tg
        assert clutter_boxes >= 10
        assert (np.abs(np.asarray(ra["targets"]).reshape(-1, 3)[:, 1]) > 10.0).any()
    finally:
        a.close(); b.close()


def test_validation(pkg, synth):
    P = _frames(synth, 1)[0][1]
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_detect_area(AREA)
        for bad in ([AREA[0][:2]], [np.full((4, 2), np.nan)], [rect(0, 0, 1, 1)] * 65, [np.zeros((1025, 2))]):
            with pytest.raises(pkg.LmotError):
                ctx.set_detect_area(bad)
        with pytest.raises(pkg.LmotError):
            ctx.set_detect_area(AREA, keep_outside=2)
        g = ctx.get_detect_area()
        assert len(g["rings"]) == 2 and np.array_equal(g["rings"][0], AREA[0]) and not g["keep_outside"]
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_detect_area(0, AREA)                 # no open set
        ctx.seq_open(2, ring=2)
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_detect_area(2, AREA)
        ctx.lib.lmot_enable_timing(ctx.h, 1)
        with pytest.raises(pkg.LmotError) as e:
            ctx.frame(P, 1e5)
        assert e.value.status == pkg.ERR_STATE
        with pytest.raises(pkg.LmotError):
            ctx.batch([P], 1e5)
        ctx.set_detect_area(None)
        ctx.frame(P, 1e5)                                    # unmasked: timing mode works as before
        ctx.lib.lmot_enable_timing(ctx.h, 0)
    finally:
        ctx.close()
