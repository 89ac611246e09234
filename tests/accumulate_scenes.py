"""Sweep accumulation (include/lmot.h, lmot_set_accumulate): a NumPy restatement of the pose (step 2) and of E_acc (step 3), and a sparse
16-beam scene seen from a moving sensor.  Shared by test_accumulate_cpu.py and test_accumulate_gpu.py."""
import math

import numpy as np

f32 = np.float32


def pose_ref(fold_s, fold_t, mount=None):
    """step 2 in float64 with the host libm (math.cos / math.sin), left to right, one rounding per operation -> (3, 4) float32"""
    xs, ys, ws = (float(v) for v in fold_s)
    xt, yt, wt = (float(v) for v in fold_t)
    d = wt - ws
    c, sn = math.cos(d), math.sin(d)
    tx = xt - (c * xs - sn * ys)
    ty = yt - (sn * xs + c * ys)
    A = [[c, -sn, 0.0, tx], [sn, c, 0.0, ty], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]
    M = [[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]
    if mount is not None:
        m = np.asarray(mount, f32).reshape(3, 4)
        for r in range(3):
            for k in range(4):
                M[r][k] = float(m[r, k])
    Mi = [[0.0] * 4 for _ in range(3)] + [[0.0, 0.0, 0.0, 1.0]]
    for r in range(3):
        for k in range(3):
            Mi[r][k] = M[k][r]
        Mi[r][3] = -((M[0][r] * M[0][3] + M[1][r] * M[1][3]) + M[2][r] * M[2][3])

    def mul(X, Y):
        return [[((X[r][0] * Y[0][k] + X[r][1] * Y[1][k]) + X[r][2] * Y[2][k]) + X[r][3] * Y[3][k] for k in range(4)] for r in range(4)]

    D = mul(Mi, mul(A, M))
    return np.array([D[r] for r in range(3)], np.float64).astype(f32)


def rig_apply(m, pts):
    """((d00*x + d01*y) + d02*z) + d03 per row in float32, w = 1 -> (n, 4) float32"""
    m = np.asarray(m, f32).reshape(3, 4)
    p = np.asarray(pts, f32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    out = np.empty((len(p), 4), f32)
    for r in range(3):
        out[:, r] = ((m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z) + m[r, 3]
    out[:, 3] = f32(1)
    return out


def e_acc(e_t, ts_t, fold_t, history, max_age_s, max_points):
    """step 3: history = [(E_s, ts_s, fold_s), ...] newest first -> (E_acc, [(ts_s, D_s) of the used sweeps])"""
    parts, used, tot = [np.asarray(e_t, f32).reshape(-1, 4)], [], len(e_t)
    for e_s, ts_s, fold_s in history:
        age = (ts_t - ts_s) / 1e6
        if not (age > 0 and age <= max_age_s) or tot + len(e_s) > max_points:
            break
        D = pose_ref(fold_s, fold_t)
        parts.append(rig_apply(D, e_s))
        used.append((ts_s, D))
        tot += len(e_s)
    return np.concatenate(parts), used


# ------------------------------------------------------------------------------------------------ the sparse scene
SPARSE = dict(rings=16, azimuths=1024, elev_top_deg=15.0, elev_bot_deg=-15.0)   # a 16-beam sensor with a 30 degree field


def drive(kind, n):
    """(v_gps, yaw_gps) of n steps: straight at 4 m/s, or a left turn of 0.04 rad per step at 3 m/s"""
    if kind == "straight":
        return [(4.0, 0.3) for _ in range(n)]
    return [(3.0, 0.3 + 0.04 * t) for t in range(n)]


def static_objects(seed=3, n=40):
    """(pos (n, 2), yaw (n,), size (n, 3)) of static cars and pedestrians in the global frame, around the first 20 m of the route"""
    rng = np.random.default_rng(seed)
    pos = np.stack([rng.uniform(-20.0, 20.0, n), rng.uniform(-25.0, 5.0, n)], 1)
    pos = pos[np.hypot(pos[:, 0], pos[:, 1] + 8.0) > 5.0]
    ped = rng.random(len(pos)) < 0.4
    size = np.where(ped[:, None], np.array([0.6, 0.6, 1.7]), np.array([4.5, 1.8, 1.5]))
    return pos, rng.uniform(-math.pi, math.pi, len(pos)), size


def sensor_frame(fold, pos, yaw):
    """global -> sensor by G (p_sensor = R(fold yaw) p + (x, y)): the sensor pose at a step is G^-1"""
    x, y, w = (float(v) for v in fold)
    c, s = math.cos(w), math.sin(w)
    return np.stack([c * pos[:, 0] - s * pos[:, 1] + x, s * pos[:, 0] + c * pos[:, 1] + y], 1), yaw + w


def sparse_frames(pkg, synth, kind, n, seed=3):
    """[(ts, v, yaw, points, fold, object positions in the sensor frame)] of the sparse scene.  The folds come from the library's own
    dead reckoning (ego8[5..7] of a context stepped with empty box lists), so static objects register to float rounding."""
    pos, oyaw, size = static_objects(seed)
    cfg = synth.SceneConfig(n_objects=0, seed=seed, **SPARSE)
    ctx = pkg.Lmot(device=0)
    out = []
    try:
        for t, (v, yg) in enumerate(drive(kind, n)):
            ts = (t + 1) * synth.DT_US
            ctx.track_step(np.zeros((0, 8, 3), f32), ts, v, yg)
            fold = ctx.tracker_get_ego()[5:8].copy()
            p, w = sensor_frame(fold, pos, oyaw)
            sc = synth.Scene(cfg, p, w, size.copy(), np.zeros(len(p)), np.zeros(len(p)), t)
            out.append((ts, v, yg, synth.render(sc), fold, p))
    finally:
        ctx.close()
    return out


def hits(boxes, objects, radius=1.0):
    """objects (n, 2) with a box centre (mean of the 8 corners) within radius"""
    if len(boxes) == 0:
        return 0
    c = np.asarray(boxes, np.float64).reshape(-1, 8, 3)[:, :, :2].mean(1)
    d = np.hypot(objects[:, None, 0] - c[None, :, 0], objects[:, None, 1] - c[None, :, 1])
    return int((d.min(1) <= radius).sum())
