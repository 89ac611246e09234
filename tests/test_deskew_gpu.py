"""Sweep deskew on the GPU (lmot_set_deskew / lmot_seq_set_deskew, include/lmot.h).

Contract: a context with deskew on, given frame P, returns bit for bit what the same context with deskew off returns for the deskewed
cloud P' (stride 4, w = 1, same stamps and ego inputs).  P' is built here in NumPy from lmot_deskew_table and the float formula of the
header, with omega from the stream's fold as restated below; frames come from synth.py with a per-point time in w taken from the
point's azimuth column (the sweep runs from -pi at tau = -0.1 s to +pi at tau = 0).  The physics test is the one that does not lean on
the restatement: it skews a static scene with the exact continuous motion and checks that deskew undoes it.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
f32 = np.float32
FIELDS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb", "boxes")
COUNTS = ("n_elevated", "n_ground", "num_cluster")
RINGS, AZ = 32, 900
N_FRAMES = 30
YAW_OFF = -0.63035 - math.pi / 2          # getOriginPoints' firstEgoYawOffset (the fold adds it to yaw_gps)
SETTING_KEYS = ("time_field", "time_scale", "time_offset", "t_min", "t_max")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


def _same(got, want, what):
    for k in COUNTS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    for k in FIELDS:
        assert got[k].shape == want[k].shape and np.array_equal(_bits(got[k]), _bits(want[k])), (what, k)


# ------------------------------------------------------------------------------------------------ data and the NumPy restatement
_FRAMES = {}


def _frames(synth, seed=7, n=N_FRAMES):
    """synth frames (rings x azimuths, ring-major) with the capture time of each point's azimuth column in w"""
    if (seed, n) not in _FRAMES:
        cfg = synth.SceneConfig(rings=RINGS, azimuths=AZ, n_objects=30, seed=seed)
        tau = (-0.1 + (np.arange(AZ) + 0.5) / AZ * 0.1).astype(f32)
        out = []
        for _, p in synth.frames(cfg, n):
            p = p.copy()
            p[:, 3] = np.tile(tau, RINGS)
            out.append(p)
        _FRAMES[(seed, n)] = out
    return _FRAMES[(seed, n)]


def _ts(f):
    return 1.0e6 + 100000.0 * f


def _ego(f):
    """a moving, turning vehicle: 6..15 m/s, yaw rate varying between about -0.3 and +0.5 rad/s"""
    return 6.0 + 0.3 * f, 0.02 * f + 0.0015 * f * f - 0.03 * math.sin(0.7 * f)


def omega_of(prev, cur):
    """the header's omega from the fold's diffYaw and dt; prev None: the stream's first frame"""
    if prev is None:
        return 0.0
    dt = (cur[0] - prev[0]) / 1e6
    diff = (cur[1] + YAW_OFF) - (prev[1] + YAW_OFF)
    if not (dt > 0 and math.isfinite(diff)):
        return 0.0
    return math.remainder(diff, 2 * math.pi) / dt


def deskew_np(pkg, rec, v, omega, mount=None, **setting):
    """P' of the records `rec` (x, y, z at 0..2, time at time_field): the header's slice rule and float formula, w = 1"""
    s = {**pkg.default_deskew(), **setting}
    tab = pkg.deskew_table(v, omega, mount, **{k: s[k] for k in SETTING_KEYS}).reshape(-1, 12)
    rec = np.asarray(rec, f32)
    tau = rec[:, s["time_field"]].astype(np.float64) * s["time_scale"] + s["time_offset"]
    fin = np.isfinite(tau)
    h = (s["t_max"] - s["t_min"]) / pkg.DESKEW_SLICES
    q = np.floor((np.where(fin, tau, 0.0) - s["t_min"]) / h)
    D = tab[np.clip(q, 0, pkg.DESKEW_SLICES - 1).astype(np.int64)]
    x, y, z = rec[:, 0], rec[:, 1], rec[:, 2]
    out = np.empty((len(rec), 4), f32)
    for r in range(3):
        out[:, r] = ((D[:, 4 * r] * x + D[:, 4 * r + 1] * y) + D[:, 4 * r + 2] * z) + D[:, 4 * r + 3]
    out[~fin, :3] = rec[~fin, :3]
    out[:, 3] = 1.0
    return out


def _stream(pkg, frames, setting, mounts=None, restarts=()):
    """P' of every frame of one stream (omega from the previous frame of the stream, 0 after a restart); mounts: per frame a list of
    per-sensor poses (batched ticks) -> per frame a list of clouds"""
    out, prev = [], None
    for f, P in enumerate(frames):
        if f in restarts:
            prev = None
        v, yaw = _ego(f)
        om = omega_of(prev, (_ts(f), yaw))
        Ps = P if isinstance(P, list) else [P]
        ms = mounts if mounts is not None else [None] * len(Ps)
        out.append([deskew_np(pkg, Pi, v, om, m, **setting) for Pi, m in zip(Ps, ms)])
        prev = (_ts(f), yaw)
    return out


def _params(pkg, gf=0):
    p = pkg.default_params()
    p.max_points = 1 << 16
    p.global_frame = gf
    return p


# ------------------------------------------------------------------------------------------------ 1. off is today's path
_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
P = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)][0]
P5 = np.concatenate([P, P[:, 3:4]], 1)
out = {}
for arm in ("off", "on_then_off", "on"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p)
    if arm != "off":
        ctx.set_deskew(on=1)
    if arm == "on_then_off":
        ctx.set_deskew()
    ctx.seq_open(8, ring=4)
    if arm == "on_then_off":
        ctx.seq_set_deskew(3, on=1); ctx.seq_set_deskew(3)
    if arm == "on":
        ctx.seq_set_deskew(3, on=1)
    d = torch.from_numpy(P).cuda(); torch.cuda.synchronize()
    def run(t):
        ctx.frame(P, t); ctx.frame(P5, t + 5e4)
        ctx.frame_dev(d.data_ptr(), len(P), t + 1e5); ctx.frame_fetch()
        ctx.seq([P] * 8, [t] * 8)
        ctx.seq_tick([dict(frames=P, timestamp=t + 1e5) if k % 2 else None for k in range(8)])
        torch.cuda.synchronize()
    run(1e6)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(2e6)
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    ctx.close()
print(json.dumps(out))
"""


def _names():
    import json
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_off_is_todays_path():
    """Catches a deskew launch or table copy issued while deskew is off (or after it was turned off again), and a deskewing context
    that still repacks its host frames: kernels, copies and memsets by name, deskew off / on-then-off / on, one process per run."""
    n = _names()
    kern = lambda arm: [x for x in n[arm] if "Memcpy" not in x and "Memset" not in x]
    assert n["off"] and not any("deskew" in x for x in n["off"]), n["off"]
    assert sorted(n["off"]) == sorted(n["on_then_off"])
    assert any("repack_kernel" in x for x in kern("off"))                      # the stride-5 host frame
    on = kern("on")
    assert sum("deskew_points_kernel" in x for x in on) == 3 + 1 + 1, on       # three frames, one seq tick, one subset tick
    assert sum("repack_kernel" in x for x in on) == 0
    assert sum("repack_kernel" in x for x in kern("off")) == 1


# ------------------------------------------------------------------------------------------------ 2. frames equal their twins
def _run_path(pkg, ctx, path, frames, tf):
    """ctx (deskew on) over every frame through `path` -> list of (status, result)"""
    out = []
    if path == "frame":
        for f, P in enumerate(frames):
            r = ctx.frame(P if tf == 3 else np.concatenate([P, P[:, 3:4]], 1), _ts(f), *_ego(f))
            out.append((ctx.last_warning, r))
    elif path == "submit":
        recs = [P if tf == 3 else np.ascontiguousarray(np.concatenate([P[:, :3], np.full((len(P), 1), 0.5, f32), P[:, 3:4]], 1))
                for P in frames]
        lag = 3
        for f, P in enumerate(recs):
            ctx.frame_submit(P, _ts(f), *_ego(f))
            while len(out) < len(recs) and (f >= lag + len(out) or f == len(recs) - 1):
                r = ctx.frame_collect()
                out.append((ctx.last_warning, r))
    else:
        import torch
        dev = [torch.from_numpy(P).cuda() for P in frames]
        torch.cuda.synchronize()
        for f, d in enumerate(dev):
            ctx.frame_dev(d.data_ptr(), len(frames[f]), _ts(f), *_ego(f))
            if f % 4 == 3 or f == len(dev) - 1:
                while ctx.frames_in_flight():
                    r = ctx.frame_collect()
                    out.append((ctx.last_warning, r))
    return out


@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("path,tf", [("frame", 3), ("submit", 3), ("submit", 4), ("dev", 3)],
                         ids=["frame", "submit-stride4", "submit-stride5-tf4", "dev"])
def test_frames_equal_twins(pkg, synth, gf, path, tf):
    """Catches a wrong omega (sign, the fold's offset, the first frame's zero), a wrong slice, a table copied for the wrong frame of
    the pipeline, the stride / time field misread, and any output that does not come from the deskewed cloud."""
    frames = _frames(synth)
    want_P = [x[0] for x in _stream(pkg, frames, {})]
    # frame 0 is deskewed with omega = 0: a nonzero omega would have given another cloud
    v0 = _ego(0)[0]
    assert not np.array_equal(deskew_np(pkg, frames[0], v0, 0.0), deskew_np(pkg, frames[0], v0, 0.2))
    assert np.abs(want_P[5][:, :2] - frames[5][:, :2]).max() > 0.5          # the ego moves enough to matter
    ctx, twin = pkg.Lmot(_params(pkg, gf)), pkg.Lmot(_params(pkg, gf))
    try:
        ctx.set_deskew(on=1, time_field=tf)
        got = _run_path(pkg, ctx, path, frames, tf)
        for f, P in enumerate(want_P):
            w = twin.frame(P, _ts(f), *_ego(f))
            assert got[f][0] == twin.last_warning, f
            _same(got[f][1], w, (path, tf, gf, f))
        assert np.array_equal(_bits(ctx.tracker_dump()), _bits(twin.tracker_dump()))
        if path == "frame":
            for a, b in zip(ctx.cluster_outputs(), twin.cluster_outputs()):     # the clouds that come back are the deskewed ones
                assert np.array_equal(_bits(a), _bits(b))
    finally:
        ctx.close(); twin.close()


# ------------------------------------------------------------------------------------------------ 3. against the reference
def test_deskewed_clouds_against_reference(pkg, synth, ref_intended):
    """The deskewed clouds run through the reference's own pipeline: the library's outputs with deskew on equal it (both clouds
    bit-exact from the stage entry point on P', counts and boxes bit-exact from the deskewing frame path, the tracker within the smoke()
    bars)."""
    ref = ref_intended
    frames = _frames(synth)[:15]
    want_P = [x[0] for x in _stream(pkg, frames, {})]
    ctx, stage = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        ctx.set_deskew(on=1)
        ref.tracker_reset()
        for f, (P, Pd) in enumerate(zip(frames, want_P)):
            v, yaw = _ego(f)
            e, g = ref.ground_remove(Pd)
            grid, k = ref.component_clustering(e)
            boxes, _ = ref.box_fitting(e, grid, k)
            want = ref.tracker_step(boxes, _ts(f), v, yaw)
            s = stage.ground_remove(Pd)
            assert np.array_equal(_bits(s["elevated"][:, :3]), _bits(e)) and np.array_equal(_bits(s["ground"][:, :3]), _bits(g)), f
            got = ctx.frame(P, _ts(f), v, yaw)
            assert (got["n_elevated"], got["n_ground"], got["num_cluster"]) == (len(e), len(g), k), f
            assert np.array_equal(_bits(got["boxes"]), _bits(boxes)), f
            assert np.array_equal(got["track_manage"], want["track_manage"]), f
            assert np.allclose(got["targets"], want["targets"], rtol=1e-4, atol=1e-4), f
    finally:
        ctx.close(); stage.close()


# ------------------------------------------------------------------------------------------------ 4. rig and sequences
def _pose(yaw_deg, tx, ty, tz):
    a = math.radians(yaw_deg)
    c, s = f32(math.cos(a)), f32(math.sin(a))
    return np.array([[c, -s, 0, tx], [s, c, 0, ty], [0, 0, 1, tz]], f32)


MOUNTS = [_pose(0, 1.5, 0.0, 0.0), _pose(90, 0.0, 0.8, 0.2), _pose(-135, -1.1, -0.6, 0.1)]


def test_rig_batch_equals_batch_on_deskewed_clouds(pkg, synth):
    """Catches every sensor deskewed with sensor 0's mount (or none), and the mount applied as M T M^-1."""
    import torch
    F = 3
    base = _frames(synth)[:12]
    frames = [[np.roll(P, 150 * i, axis=0) if i else P for i in range(F)] for P in base]   # (different clouds per sensor)
    want = _stream(pkg, frames, {}, mounts=MOUNTS)
    ctx, twin = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        for c in (ctx, twin):
            c.set_sensors(MOUNTS)
        ctx.set_deskew(on=1)
        for f, fr in enumerate(frames):
            dev = [torch.from_numpy(np.ascontiguousarray(P)).cuda() for P in fr]
            torch.cuda.synchronize()
            ctx.batch_dev([(d.data_ptr(), len(d)) for d in dev], _ts(f), *_ego(f))
            g = ctx.batch_fetch()
            w = twin.batch(want[f], _ts(f), *_ego(f))
            for k in ("n_elevated", "n_ground", "num_cluster", "n_boxes"):
                assert g[k] == w[k], (f, k)
            for k in FIELDS:
                assert np.array_equal(_bits(g[k]), _bits(w[k])), (f, k)
        assert np.array_equal(_bits(ctx.tracker_dump()), _bits(twin.tracker_dump()))
    finally:
        ctx.close(); twin.close()


# sequence k's deskew setting (None: off) and whether it has a one-sensor table
SEQ_SETTINGS = [dict(on=1), None, dict(on=1), dict(on=1), dict(on=1), None,
                dict(on=1, time_scale=1e-6, t_min=-0.12, t_max=0.01), dict(on=1, time_offset=-0.1, t_min=-0.1, t_max=0.0)]
SEQ_TABLE = {2: [_pose(30, 0.7, -0.3, 0.0)], 7: [_pose(-60, -0.5, 0.4, 0.0)]}
RESTART = {3: 9}                                  # sequence 3 restarts at tick 9


def _seq_frame(pkg, synth, k, t):
    """sequence k's frame at its tick t, its time field scaled / offset the way its setting reads it"""
    P = _frames(synth, seed=20 + k, n=14)[t].copy()
    s = SEQ_SETTINGS[k] or {}
    if "time_scale" in s:
        P[:, 3] = (P[:, 3].astype(np.float64) * 1e6).astype(f32)        # microseconds
    if "time_offset" in s:
        P[:, 3] = P[:, 3] + f32(0.1)                                      # seconds since the sweep's start
    return P


def test_sequences_equal_their_twins(pkg, synth):
    """Catches a sequence deskewed with another sequence's fold, setting or mount, a tick whose deskew-off sequences are moved, LISTS
    steps that read the setting, and a restart that keeps the old fold's omega.  Host and device ticks alternate."""
    import torch
    S, T = 8, 14
    rng = np.random.default_rng(3)
    sched = [[None if rng.random() < 0.2 else ("L" if k in (4, 5) and rng.random() < 0.4 else "F") for k in range(S)] for t in range(T)]
    for t in range(T):
        sched[t][0] = "F"
    sched[RESTART[3]][3] = "F"
    seq_ts = lambda k, t: 1.0e6 + 5000.0 * k + 100000.0 * t
    seq_ego = lambda k, t: (4.0 + k + 0.4 * t, 0.01 * k + 0.03 * t + 0.002 * t * t * (1 if k % 2 else -1))
    ctx = pkg.Lmot(_params(pkg))
    twins = [pkg.Lmot(_params(pkg)) for _ in range(S)]
    try:
        ctx.seq_open(S, ring=4)
        for k in range(S):
            if SEQ_SETTINGS[k]:
                ctx.seq_set_deskew(k, **SEQ_SETTINGS[k])
                twins[k].set_deskew(**SEQ_SETTINGS[k])
            if k in SEQ_TABLE:
                ctx.seq_set_sensors(k, SEQ_TABLE[k])
                twins[k].set_sensors(SEQ_TABLE[k])
        assert ctx.seq_get_deskew(6) == {**pkg.default_deskew(), **SEQ_SETTINGS[6]}
        for t in range(T):
            entries, host_frames = [], []
            for k in range(S):
                kind = sched[t][k]
                if kind is None:
                    entries.append(None)
                    continue
                v, yaw = seq_ego(k, t)
                d = dict(timestamp=seq_ts(k, t), v_gps=v, yaw_gps=yaw, restart=RESTART.get(k) == t)
                if kind == "F":
                    d["frames"] = _seq_frame(pkg, synth, k, t)
                else:
                    b = _frames(synth, seed=20 + k, n=14)[t][:96, :3].reshape(-1, 8, 3) * f32(0.05) + f32(3.0 * k)
                    d["lists"] = np.ascontiguousarray(b, f32)
                entries.append(d)
            if t % 2 == 0:
                res = ctx.seq_tick(entries)
            else:
                keep = []
                dev_entries = []
                for d in entries:
                    if d is None or "frames" not in d:
                        dev_entries.append(d)
                        continue
                    x = torch.from_numpy(d["frames"]).cuda()
                    keep.append(x)
                    dev_entries.append({**d, "frames": (x.data_ptr(), len(x))})
                if any(d is not None and "lists" in d for d in dev_entries):
                    res = ctx.seq_tick(entries)      # (device LISTS need padded device lists: this tick stays on the host form)
                else:
                    torch.cuda.synchronize()
                    ctx.seq_tick_dev(dev_entries)
                    res = ctx.seq_collect()
                    res = [r if d is not None else None for r, d in zip(res, dev_entries)]
            for k in range(S):
                d = entries[k]
                if d is None:
                    assert res[k] is None
                    continue
                tw = twins[k]
                if d.get("restart"):
                    tw.tracker_reset()
                if "frames" in d:
                    w = tw.batch([d["frames"]], d["timestamp"], d["v_gps"], d["yaw_gps"]) if k in SEQ_TABLE else \
                        tw.frame(d["frames"], d["timestamp"], d["v_gps"], d["yaw_gps"])
                    if k in SEQ_TABLE:
                        w.update({c: int(sum(w[c])) for c in COUNTS})
                else:
                    w = tw.track_step(d["lists"], d["timestamp"], d["v_gps"], d["yaw_gps"])
                    w.update(boxes=d["lists"], n_elevated=0, n_ground=0, num_cluster=0)
                for c in FIELDS:
                    assert np.array_equal(_bits(res[k][c]), _bits(np.asarray(w[c], res[k][c].dtype))), (t, k, c)
        for k in range(S):
            assert np.array_equal(_bits(ctx.seq_tracker_dump(k)), _bits(twins[k].tracker_dump())), k
    finally:
        ctx.close()
        for tw in twins:
            tw.close()


# ------------------------------------------------------------------------------------------------ 5. physics
def _pose_at(v, w, tau):
    """the exact continuous pose (heading, x, y) at times tau of a vehicle moving at v along +x and turning at w about +z"""
    th = w * tau
    return th, v * np.sin(th) / w, v * (1 - np.cos(th)) / w


def test_physics_static_scene_and_seam_object(pkg, synth):
    """The only test that catches a sign error shared by the library and the restatement: a static scene is skewed with the exact
    continuous motion of a vehicle at 20 m/s and 0.3 rad/s; deskew must put every point back within the slice bound, and a car on
    the sweep seam (behind the vehicle, turned so that two of its sides face the sensor) must come back as one box at its place,
    where the skewed frame splits its two sides 2 m apart."""
    cfg = synth.SceneConfig(rings=RINGS, azimuths=AZ, n_objects=6, seed=4)
    sc = synth.make_scene(cfg)
    sc.pos = np.array([[-12.0, 0.0], [9.0, 6.0], [10.0, -8.0], [-6.0, 12.0], [5.0, -14.0], [-15.0, -10.0]])
    sc.yaw = np.array([math.pi / 4, 0.3, 1.2, -0.4, 2.0, 0.0]); sc.vel = np.zeros(6); sc.yawrate = np.zeros(6)
    sc.size = np.tile([4.5, 1.8, 1.5], (6, 1))
    Q = synth.render(sc).astype(np.float64)                 # the static scene in the vehicle frame at the stamp
    az = np.tile(np.arange(AZ), RINGS)
    tau = -0.1 + (az + 0.5) / AZ * 0.1
    V, W = 20.0, 0.3
    th, tx, ty = _pose_at(V, W, tau)
    c, s = np.cos(th), np.sin(th)
    dx, dy = Q[:, 0] - tx, Q[:, 1] - ty                       # measured: the inverse of the pose at the point's time
    skew = np.stack([c * dx + s * dy, -s * dx + c * dy, Q[:, 2], tau], 1).astype(f32)
    # the NumPy restatement of the library undoes it within the slice bound (time error <= h/2 at the ego's speed and turn rate)
    h = 0.1 / pkg.DESKEW_SLICES
    r = np.hypot(Q[:, 0], Q[:, 1])
    bound = V * h / 2 + W * h / 2 * (r + 2.0) + 1e-4
    Pd = deskew_np(pkg, skew, V, W)
    err = np.hypot(Pd[:, 0] - Q[:, 0], Pd[:, 1] - Q[:, 1])
    assert (err <= bound).all() and bound.max() < 0.02, (err.max(), bound.max())
    assert np.hypot(skew[:, 0] - Q[:, 0], skew[:, 1] - Q[:, 1]).max() > 1.5
    # on the GPU: frame 0 sets the fold up (omega 0), frame 1 moves at (V, W)
    on, off = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        on.set_deskew(on=1)
        yaw0 = 0.4
        res = {}
        for name, ctx in (("on", on), ("off", off)):
            ctx.frame(skew, 1.0e6, V, yaw0)
            res[name] = ctx.frame(skew, 1.1e6, V, yaw0 + W * 0.1)
        assert abs(omega_of((1.0e6, yaw0), (1.1e6, yaw0 + W * 0.1)) - W) < 1e-9
        def seam_boxes(b):
            ctr = b.reshape(-1, 8, 3)[:, :, :2].mean(1)
            return ctr[np.hypot(ctr[:, 0] + 12.0, ctr[:, 1]) < 4.0]

        # the seam car at (-12, 0): with deskew one box where the unskewed scene gives its box; without, two boxes, none, or one
        # displaced by more than 1 m
        truth = pkg.Lmot(_params(pkg))
        try:
            truth.frame(Q.astype(f32), 1.0e6)
            truth_res = truth.frame(Q.astype(f32), 1.1e6)
            want = seam_boxes(truth_res["boxes"])
        finally:
            truth.close()
        good, bad = seam_boxes(res["on"]["boxes"]), seam_boxes(res["off"]["boxes"])
        # every car comes back where the unskewed scene puts it (the GPU's deskewed points themselves equal the restatement's, which
        # test_frames_equal_twins holds bit for bit)
        ctr = lambda r: r["boxes"].reshape(-1, 8, 3)[:, :, :2].mean(1)
        got_c, want_c = ctr(res["on"]), ctr(truth_res)
        d = np.hypot(got_c[:, None, 0] - want_c[None, :, 0], got_c[:, None, 1] - want_c[None, :, 1])
        assert len(want_c) >= 5 and d.min(0).max() < 0.3, (got_c, want_c)
        assert len(want) == 1, want
        assert len(good) == 1 and np.hypot(*(good[0] - want[0])) < 0.3, (good, want)
        assert len(bad) != 1 or np.hypot(*(bad[0] - want[0])) > 1.0, (bad, want)
    finally:
        on.close(); off.close()


# ------------------------------------------------------------------------------------------------ 6. in flight, reset, reopen
def test_setting_changes_apply_from_the_next_submission(pkg, synth):
    """Catches a table or setting read at collection (or on the device after submission) instead of captured at submission, a reset
    that keeps the old fold's omega, and the zero-copy path taken while deskewing."""
    frames = _frames(synth)[:16]
    settings = [dict(on=1)] * 5 + [dict(on=1, t_min=-0.15, t_max=0.05)] * 4 + [None] * 3 + [dict(on=1)] * 4
    os.environ["LMOT_ZERO_COPY"] = "1"
    try:
        ctx = pkg.Lmot(_params(pkg))
    finally:
        del os.environ["LMOT_ZERO_COPY"]
    twin = pkg.Lmot(_params(pkg))
    try:
        pinned = [ctx.pinned_array(P.shape) for P in frames]
        for a, P in zip(pinned, frames):
            a[:] = P
        prev = None
        want = []
        for f, P in enumerate(frames):
            if f == 12:                       # reset: the fold starts over, the next frame has omega 0
                ctx.tracker_reset(); twin.tracker_reset(); prev = None
            s = settings[f]
            if s:
                ctx.set_deskew(**s)
            else:
                ctx.set_deskew()
            ctx.frame_submit(pinned[f], _ts(f), *_ego(f))
            v, yaw = _ego(f)
            om = omega_of(prev, (_ts(f), yaw))
            want.append(deskew_np(pkg, P, v, om, **s) if s else P)
            prev = (_ts(f), yaw)
            if f == 11:                       # collect before the reset (a reset drains and drops uncollected results)
                got = [ctx.frame_collect() for _ in range(ctx.frames_in_flight())]
                for g, (ff, Pw) in zip(got, list(enumerate(want))[:12]):
                    _same(g, twin.frame(Pw, _ts(ff), *_ego(ff)), ("in flight", ff))
        got = [ctx.frame_collect() for _ in range(ctx.frames_in_flight())]
        for g, ff in zip(got, range(12, 16)):
            _same(g, twin.frame(want[ff], _ts(ff), *_ego(ff)), ("after reset", ff))
        assert ctx.get_deskew() == {**pkg.default_deskew(), "on": 1}
        # sequences: reset and load keep the setting, reopening turns it off
        ctx.seq_open(2, ring=2)
        ctx.seq_set_deskew(1, on=1, t_min=-0.05, t_max=0.05)
        ctx.seq_tracker_reset(1)
        ctx.seq_tracker_load(1, np.zeros((0, pkg.TRACK_DUMP_DOUBLES)), 0, 0.0)
        assert ctx.seq_get_deskew(1)["on"] == 1 and ctx.seq_get_deskew(1)["t_max"] == 0.05
        ctx.seq_open(2, ring=2)
        assert ctx.seq_get_deskew(1) == pkg.default_deskew() and ctx.seq_get_deskew(0) == pkg.default_deskew()
    finally:
        ctx.close(); twin.close()


# ------------------------------------------------------------------------------------------------ 7. validation
def test_validation(pkg, synth):
    """Every error of the header's list, each leaving the setting unchanged and nothing submitted."""
    import torch
    P = _frames(synth)[0]
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_deskew(on=1, t_min=-0.08)
        before = ctx.get_deskew()
        for bad in (dict(t_min=0.0, t_max=0.0), dict(t_min=0.2), dict(t_min=-1.5), dict(time_scale=float("nan")),
                    dict(t_max=float("inf")), dict(time_offset=float("nan")), dict(time_field=2)):
            with pytest.raises(pkg.LmotError) as e:
                ctx.set_deskew(on=1, **bad)
            assert e.value.status == pkg.ERR_INVALID, bad
            assert ctx.get_deskew() == before
        # a host frame without the time field, a device frame with the time elsewhere than w
        ctx.set_deskew(on=1, time_field=4)
        with pytest.raises(pkg.LmotError) as e:
            ctx.frame_submit(P, 1e6)
        assert e.value.status == pkg.ERR_INVALID and ctx.frames_in_flight() == 0
        d = torch.from_numpy(P).cuda()
        torch.cuda.synchronize()
        with pytest.raises(pkg.LmotError) as e:
            ctx.frame_dev(d.data_ptr(), len(P), 1e6)
        assert e.value.status == pkg.ERR_INVALID and ctx.frames_in_flight() == 0
        with pytest.raises(pkg.LmotError) as e:
            ctx.batch_dev([(d.data_ptr(), len(P))], 1e6)
        assert e.value.status == pkg.ERR_INVALID and ctx.frames_in_flight() == 0
        ctx.batch_detect_dev([(d.data_ptr(), len(P))])           # no stamp: not deskewed, not refused
        ctx.batch_fetch()
        # timing mode
        ctx.set_deskew(on=1)
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError) as e:
            ctx.frame(P, 1e6)
        assert e.value.status == pkg.ERR_STATE and ctx.frames_in_flight() == 0
        ctx.enable_timing(False)
        ctx.frame(P, 1e6)
        # sequences
        ctx.seq_open(2, ring=2)
        for k in (-1, 2):
            with pytest.raises(pkg.LmotError) as e:
                ctx.seq_set_deskew(k, on=1)
            assert e.value.status == pkg.ERR_INVALID
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_deskew(0, on=1, t_min=0.5, t_max=0.1)
        assert ctx.seq_get_deskew(0) == pkg.default_deskew()
        ctx.seq_set_deskew(1, on=1, time_field=4)
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_tick([dict(frames=P, timestamp=1e6), dict(frames=P, timestamp=1e6)])
        assert e.value.status == pkg.ERR_INVALID
        with pytest.raises(pkg.LmotError) as e:
            ctx.seq_tick_dev([None, dict(frames=(d.data_ptr(), len(P)), timestamp=1e6)])
        assert e.value.status == pkg.ERR_INVALID
        ctx.seq_tick([dict(frames=P, timestamp=1e6), dict(lists=np.zeros((0, 8, 3), f32), timestamp=1e6)])   # LISTS ignore it
    finally:
        ctx.close()
