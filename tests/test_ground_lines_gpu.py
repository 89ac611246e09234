"""Ground lines on the device (include/lmot.h, lmot_set_ground_lines): the ground kernel's lines variant and box heights from the local
ground against the reference's own chain on the line-labelled cloud (tests/ground_lines_scenes.py), through every frame path, rigs,
sequences next to plain ones, setting changes in flight, and the objects found on sloped scenes."""
import numpy as np
import pytest

import ground_lines_scenes as gls

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


def _bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _same_frame(a, b, keys=("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")):
    for k in ("n_elevated", "n_ground", "num_cluster"):
        assert a[k] == b[k], k
    assert np.array_equal(_bits(a["boxes"]), _bits(b["boxes"]))
    for k in keys:
        if k in a:
            assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def _tunable():
    from oracle import ref_detect_tunable as rdt
    if not rdt.have_ref("detect_tunable"):
        pytest.skip("oracle/_ref/libref_detect_tunable.so not built")
    return rdt.RefDetectTunable()


_SCENES = {}


def _scene(name, rings=64, azimuths=1875):
    key = (name, rings, azimuths)
    if key not in _SCENES:
        _SCENES[key] = gls.render(name, rings=rings, azimuths=azimuths)
    return _SCENES[key]


def _moving(name, n, rings=32, azimuths=900):
    """n frames of a sloped scene: the sensor's own sweep moves the noise, the frame stamps advance"""
    pts, _ = _scene(name, rings, azimuths)
    rng = np.random.default_rng(len(name))
    out = []
    for f in range(n):
        p = pts.copy()
        p[:, :3] += rng.normal(0, 0.01, (len(p), 3)).astype(f32)
        out.append(((f + 1) * 100_000.0, p))
    return out


# ------------------------------------------------------------------------------------------------ today's path
# the trace runs in a process of its own, as every other kernel-name test of the suite: a profiler session leaves state behind in the
# process that later in-process profiling of other tests would see
_NAMES_SCRIPT = r"""
import importlib, json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
import ground_lines_scenes as gls
P = gls.render("grade8", rings=32, azimuths=900)[0]
out = {}
for arm in ("plain", "on_then_off", "on"):
    p = pkg.default_params(); p.max_points = 1 << 17
    ctx = pkg.Lmot(p)
    if arm != "plain":
        ctx.set_ground_lines(on=1)
    if arm == "on_then_off":
        ctx.set_ground_lines()
    ctx.frame(P, 1e5)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.frame(P, 2e5)
        torch.cuda.synchronize()
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    ctx.close()
print(json.dumps(out))
"""


def test_off_is_todays_path(pkg):
    """never set, and set then reset: the same kernels, copies and memsets and bit-identical results as a context that never had ground
    lines; on: the ground and box-fitting kernels are the lines variants, one for one"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    assert n["plain"] and sorted(n["plain"]) == sorted(n["on_then_off"])
    assert not any("lines" in k for k in n["plain"])
    assert sum("ground_fused_lines_kernel" in k for k in n["on"]) == 1 and sum("box_fit_lines_kernel" in k for k in n["on"]) == 1
    assert not any("ground_fused_kernel" in k or "box_fit_kernel" in k for k in n["on"])
    assert len(n["on"]) == len(n["plain"])
    frames = _moving("grade8", 3)
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_ground_lines(on=1)
        b.set_ground_lines()
        for ts, p in frames:
            _same_frame(a.frame(p, ts), b.frame(p, ts))
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ against the reference's chain
@pytest.mark.parametrize("name", ["flat", "grade8", "pitch3", "roll2"])
def test_frame_against_reference(pkg, name):
    """device gz equals the host function on the reference's minZ grid; counts equal the restated labels; boxes equal the reference's
    boxFitting per cluster with sensorHeight = -g, bit for bit"""
    rt = _tunable()
    pts, _ = _scene(name)
    want = gls.ref_lines_detect(rt, pts)
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_ground_lines(on=1)
        r = ctx.frame(pts, 100_000.0)
        gz = ctx.debug_ground_lines()
        assert gz.shape == (1, 80, 120)
        host = pkg.ground_lines_grid(rt.polar_grid(pts)["minz"], float(f32(3.4)), 120.0, 2.0)    # lmot_params' floats
        assert np.array_equal(_bits(gz[0]), _bits(host))
        assert np.array_equal(_bits(host), _bits(want["gz"]))
        assert (r["n_elevated"], r["n_ground"], r["num_cluster"]) == (len(want["elev"]), len(want["ground"]), want["k"])
        assert len(want["boxes"]) > 5
        assert np.array_equal(_bits(r["boxes"]), _bits(want["boxes"]))
        ctx.set_ground_lines()
        ctx.frame(pts, 200_000.0)
        assert ctx.debug_ground_lines().shape[0] == 0
    finally:
        ctx.close()


@pytest.mark.parametrize("search", [0, 90])
@pytest.mark.parametrize("rule", [0, 1])
def test_rule_modes_against_reference(pkg, rule, search):
    """both rule modes, boxFitting's fit and box search: boxes equal the reference's boxFitting (or box search's restated fit with the
    reference's ruleBasedFilter) per cluster with sensorHeight = -g, bit for bit; the tracker on them equals the reference's"""
    from box_search_scenes import RefSearch, have_ref_search
    from oracle import ref
    rt = _tunable()
    mode = "o2" if rule else "intended"
    if not ref.have_ref(mode) or not have_ref_search(mode):
        pytest.skip("oracle/_ref reference libraries not built")
    fitter = ref.RefOracle(mode)
    rs = RefSearch(mode) if search else None
    frames = _moving("grade8", 4, 64, 1875)
    ctx = pkg.Lmot(_params(pkg, 0, rule))
    try:
        ctx.set_ground_lines(on=1)
        if search:
            ctx.set_box_search(on=1, n_angles=search)
        fitter.tracker_reset()
        for ts, p in frames:
            want = gls.ref_lines_detect(rt, p, fitter=fitter, search=(rs, search) if search else None)
            r = ctx.frame(p, ts)
            assert (r["n_elevated"], r["n_ground"], r["num_cluster"]) == (len(want["elev"]), len(want["ground"]), want["k"])
            assert len(want["boxes"]) > 5
            assert np.array_equal(_bits(r["boxes"]), _bits(want["boxes"]))
            if rule == 0:
                w = fitter.tracker_step(want["boxes"], ts)
                assert np.array_equal(r["track_manage"], w["track_manage"])
                assert np.allclose(r["targets"], w["targets"], rtol=1e-4, atol=1e-4)
    finally:
        ctx.close()


@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("rule", [0, 1])
def test_frame_paths(pkg, gf, rule):
    """lmot_frame, pipelined lmot_frame_submit (stride 4 and 3), lmot_frame_dev and lmot_detect_dev agree bit for bit; the tracker on the
    boxes equals a twin stepped with lmot_track_step on them"""
    import torch
    frames = _moving("pitch3", 6)
    ctxs = [pkg.Lmot(_params(pkg, gf, rule, pipeline_depth=4)) for _ in range(5)]
    sync, piped4, piped3, dev, twin = ctxs
    try:
        for c in (sync, piped4, piped3, dev):
            c.set_ground_lines(on=1)
        got = []
        for ts, p in frames:
            r = sync.frame(p, ts)
            if gf == 0:
                t = twin.track_step(r["boxes"], ts)
                for k in ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb"):
                    assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(t[k]).view(np.uint8)), k
            got.append(r)
        assert sum(len(r["boxes"]) for r in got) > 10
        for c, stride in ((piped4, 4), (piped3, 3)):
            out = []
            for ts, p in frames:
                c.frame_submit(np.ascontiguousarray(p[:, :stride]), ts)
                if c.frames_in_flight() == 4:
                    out.append(c.frame_collect())
            while c.frames_in_flight():
                out.append(c.frame_collect())
            for x, y in zip(out, got):
                _same_frame(x, y)
        d = [torch.from_numpy(p).cuda() for _, p in frames]
        torch.cuda.synchronize()
        for (ts, p), x in zip(frames, d):
            dev.frame_dev(x.data_ptr(), len(p), ts)
        _same_frame(dev.frame_fetch(), got[-1])
        if gf == 0:
            det = pkg.Lmot(_params(pkg, gf, rule))
            try:
                det.set_ground_lines(on=1)
                det.detect_dev(d[0].data_ptr(), len(frames[0][1]))
                r = det.frame_fetch()
                assert np.array_equal(_bits(r["boxes"]), _bits(got[0]["boxes"]))
            finally:
                det.close()
    finally:
        for c in ctxs:
            c.close()


def test_box_search_with_lines(pkg):
    """box search measures each cluster from its local ground: the bottom corners of every box sit at a g of the grid (or the flat
    -sensor_height), and a sequence with both settings equals a context with both"""
    pts, _ = _scene("grade8", 32, 900)
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        a.set_ground_lines(on=1)
        a.set_box_search(on=1)
        r = a.frame(pts, 100_000.0)
        gz = a.debug_ground_lines()[0]
        bottoms = r["boxes"][:, 0, 2]
        assert len(bottoms) > 3
        allowed = set(_bits(gz).ravel().tolist()) | {int(_bits(np.array([-2.0], f32))[0])}
        assert set(_bits(bottoms).tolist()) <= allowed
        plain = pkg.Lmot(_params(pkg))
        try:
            plain.set_box_search(on=1)
            q = plain.frame(pts, 100_000.0)
            assert not np.array_equal(_bits(q["boxes"]), _bits(r["boxes"]))
        finally:
            plain.close()
        b.seq_open(2, ring=4)
        b.seq_set_ground_lines(1, on=1)
        b.seq_set_box_search(1, on=1)
        s = b.seq([pts, pts], [100_000.0, 100_000.0])
        _same_frame(s[1], r)
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ rigs
def _tilted_rig():
    """two sensors: one pitched down 3 degrees at the front, one level and turned around at the back (sensor -> vehicle [R | t])"""
    c, s = np.cos(np.radians(3.0)), np.sin(np.radians(3.0))
    front = np.array([[c, 0, s, 1.0], [0, 1, 0, 0], [-s, 0, c, 0]], f32)
    back = np.array([[-1, 0, 0, -1.0], [0, -1, 0, 0], [0, 0, 1, 0]], f32)
    return np.stack([front, back]), [1.9, 2.1]


@pytest.mark.parametrize("merge", [0, 1])
def test_rig(pkg, merge):
    """each rig frame's lines come from its own minZ grid and its sensor's sensor_height; separate units box from their grids, a merge
    unit from the flat height; a sequence with the same rig equals the context's batches"""
    rt = _tunable()
    pose, heights = _tilted_rig()
    fr = [_scene("pitch3", 32, 900)[0], _scene("grade4", 32, 900)[0]]
    ctx, seq = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        for c in (ctx,):
            c.set_sensors(pose, sensor_height=heights)
            c.set_rig_merge(merge)
            c.set_ground_lines(on=1)
        seq.seq_open(2, ring=4)
        seq.seq_set_sensors(0, pose, sensor_height=heights)
        seq.seq_set_rig_merge(0, merge)
        seq.seq_set_ground_lines(0, on=1)
        out = []
        for t in range(3):
            ts = (t + 1) * 100_000.0
            r = ctx.batch(fr, ts)
            gz = ctx.debug_ground_lines()
            assert gz.shape[0] == 2
            for i in range(2):
                host = pkg.ground_lines_grid(rt.polar_grid(fr[i])["minz"], float(f32(3.4)), 120.0, float(f32(heights[i])))
                assert np.array_equal(_bits(gz[i]), _bits(host))
            s = seq.seq([fr, fr[0]], [ts, ts])[0]
            for k in ("n_elevated", "n_ground", "num_cluster"):
                assert s[k] == sum(r[k]), k
            _same_frame(dict(s, n_elevated=0, n_ground=0, num_cluster=0), dict(r, n_elevated=0, n_ground=0, num_cluster=0))
            out.append(r)
        assert len(out[-1]["boxes"]) > 3
        if merge:                                        # the merge unit's boxes stand on the vehicle's flat ground
            assert np.all(out[-1]["boxes"][:, 0, 2] == f32(-2.0))
    finally:
        ctx.close(); seq.close()


# ------------------------------------------------------------------------------------------------ sequences next to plain ones
def test_sequences_mixed(pkg):
    """seven sequences (eight frames: one has a two-sensor rig) with mixed settings (lines on and off, box search, own detection values)
    in one tick, over several ticks, each equal to a twin context with only its settings"""
    names = ["grade8", "flat", "pitch3", "roll2", "grade4", "grade8", "pitch3"]
    frames = [_moving(n, 3) for n in names]
    pose, heights = _tilted_rig()
    cfg = [
        dict(lines=dict(on=1)), dict(), dict(lines=dict(on=1, max_slope=0.2)), dict(lines=dict(on=1), search=dict(on=1)),
        dict(lines=dict(on=1), det=dict(sensor_height=1.8, r_min=2.5)), dict(search=dict(on=1)),
        dict(lines=dict(on=1, max_step=0.2), rig=True),
    ]
    ctx = pkg.Lmot(_params(pkg))
    twins = [pkg.Lmot(_params(pkg)) for _ in range(len(cfg))]
    try:
        ctx.seq_open(len(cfg), ring=4)
        for k, c in enumerate(cfg):
            tw = twins[k]
            tw.seq_open(1, ring=2)
            if "lines" in c:
                ctx.seq_set_ground_lines(k, **c["lines"]); tw.seq_set_ground_lines(0, **c["lines"])
            if "search" in c:
                ctx.seq_set_box_search(k, **c["search"]); tw.seq_set_box_search(0, **c["search"])
            if "det" in c:
                ctx.seq_set_detect_params(k, **c["det"]); tw.seq_set_detect_params(0, **c["det"])
            if c.get("rig"):
                ctx.seq_set_sensors(k, pose, sensor_height=heights); tw.seq_set_sensors(0, pose, sensor_height=heights)
        for t in range(3):
            ent = [[f[t][1], f[t][1]] if c.get("rig") else f[t][1] for f, c in zip(frames, cfg)]
            ts = [f[t][0] for f in frames]
            got = ctx.seq(ent, ts)
            for k in range(len(cfg)):
                w = twins[k].seq([ent[k]], [ts[k]])[0]
                _same_frame(got[k], w)
        assert ctx.seq_get_ground_lines(2) == {"on": 1, "max_slope": 0.2, "max_rmse": 0.08, "max_step": 0.3}
        ctx.seq_tracker_reset(0)
        assert ctx.seq_get_ground_lines(0)["on"] == 1
        ctx.seq_open(8, ring=4)
        assert all(ctx.seq_get_ground_lines(k)["on"] == 0 for k in range(8))
    finally:
        ctx.close()
        for t in twins:
            t.close()


# ------------------------------------------------------------------------------------------------ lifecycle and validation
def test_changes_in_flight(pkg):
    """a change applies from the next submission: frames and ticks in flight keep theirs"""
    frames = _moving("grade8", 8)
    a, b = pkg.Lmot(_params(pkg, pipeline_depth=4)), pkg.Lmot(_params(pkg))
    try:
        settings = [dict(on=1), None, dict(on=1, max_slope=0.1), dict(on=1, max_step=0.5)]
        got, want = [], []
        for i, (ts, p) in enumerate(frames):
            if i % 2 == 0:
                s = settings[i // 2]
                for c in (a, b):
                    c.set_ground_lines(**s) if s else c.set_ground_lines()
            a.frame_submit(p, ts)
            want.append(b.frame(p, ts))
            if a.frames_in_flight() == 4:
                got.append(a.frame_collect())
        while a.frames_in_flight():
            got.append(a.frame_collect())
        for x, y in zip(got, want):
            _same_frame(x, y)
        assert want[0]["n_ground"] != want[2]["n_ground"]
        c, tw = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
        try:
            c.seq_open(2, ring=4); tw.seq_open(2, ring=4)
            res, ref_res = [], []
            for i, (ts, p) in enumerate(frames):
                on = [1, 0, 1, 1, 0, 1, 0, 1][i]
                for x in (c, tw):
                    x.seq_set_ground_lines(1, on=on, max_slope=0.3 if i % 3 else 0.15)
                c.seq_submit([p, p], [ts, ts])
                ref_res.append(tw.seq([p, p], [ts, ts]))
                if i >= 3:
                    res.append(c.seq_collect())
            while len(res) < len(frames):
                res.append(c.seq_collect())
            for r, w in zip(res, ref_res):
                for k in range(2):
                    _same_frame(r[k], w[k])
        finally:
            c.close(); tw.close()
    finally:
        a.close(); b.close()


def test_validation(pkg):
    p = _moving("flat", 1)[0][1]
    ctx = pkg.Lmot(_params(pkg))
    try:
        for bad in (dict(on=2), dict(on=-1), dict(on=1, max_slope=0.0), dict(on=1, max_rmse=-0.1), dict(on=1, max_step=0.0),
                    dict(on=1, max_slope=float("nan")), dict(on=1, max_step=float("inf"))):
            with pytest.raises(pkg.LmotError) as e:
                ctx.set_ground_lines(**bad)
            assert e.value.status == pkg.ERR_INVALID
            assert ctx.get_ground_lines()["on"] == 0
        for k in (-1, 0):
            with pytest.raises(pkg.LmotError):
                ctx.seq_set_ground_lines(k, on=1)
        ctx.seq_open(2)
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_ground_lines(2, on=1)
        ctx.set_ground_lines(on=1, max_slope=0.2)
        assert ctx.get_ground_lines() == {"on": 1, "max_slope": 0.2, "max_rmse": 0.08, "max_step": 0.3}
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError) as e:
            ctx.frame(p, 100_000.0)
        assert e.value.status == pkg.ERR_STATE
        ctx.enable_timing(False)
        ctx.frame(p, 100_000.0)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ quality
def test_quality(pkg):
    """objects found (a box centre within 2 m of theirs, 40 objects): on an 8 % grade and under 3 degrees of pitch at least 4 more than
    with the lines off, on flat ground at most 2 fewer"""
    found = {}
    for name in ("flat", "grade8", "pitch3"):
        pts, obj = _scene(name)
        for on in (0, 1):
            ctx = pkg.Lmot(_params(pkg))
            try:
                if on:
                    ctx.set_ground_lines(on=1)
                found[name, on] = gls.objects_found(ctx.frame(pts, 100_000.0)["boxes"], obj)
            finally:
                ctx.close()
    print(found)
    assert found["grade8", 1] >= found["grade8", 0] + 4
    assert found["pitch3", 1] >= found["pitch3", 0] + 4
    assert found["flat", 1] >= found["flat", 0] - 2
