"""Scan-matched ego motion (include/lmot.h, lmot_ego_estimate): a NumPy restatement of one estimator call, a per-hypothesis brute
force for small clouds, and drives rendered from the library's fold (accumulate_scenes' straight and turning routes at 16, 32 and 64
beams, optionally with synth's movers).  Shared by test_ego_match_cpu.py, test_ego_match_gpu.py and scripts/ego_match_premise.py."""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import accumulate_scenes as acs  # noqa: E402

f32 = np.float32
MAX_BATCH = 8


def defaults():
    """lmot_default_ego_match"""
    return dict(grid=768, cell_m=0.1, z_min=-1.5, z_max=0.5, r_min=3.0, r_max=38.0, sub_m=0.4, max_points=4096, yaw_step=0.005,
                yaw_half=30, shift_half=30, refine=5, min_points=200, min_score_frac=0.3, sensor=-1)


def sub_side(s):
    """sub-cells per side: ceil(grid * cell_m / sub_m) + 1, in double"""
    return int(math.ceil(s["grid"] * s["cell_m"] / s["sub_m"])) + 1


def valid(s):
    """lmot_set_ego_match's validation (no device)"""
    d = ("cell_m", "z_min", "z_max", "r_min", "r_max", "sub_m", "yaw_step", "min_score_frac")
    if not all(math.isfinite(s[k]) for k in d):
        return False
    return (32 <= s["grid"] <= 1024 and s["grid"] % 32 == 0 and 0.01 <= s["cell_m"] <= 10.0 and s["grid"] * s["cell_m"] <= 400.0
            and s["z_min"] < s["z_max"] and 0.0 <= s["r_min"] < s["r_max"] <= 1000.0
            and s["sub_m"] > 0.0 and sub_side(s) <= 1024
            and 1 <= s["max_points"] <= 8192 and 0.0 < s["yaw_step"] <= 0.1 and 0 <= s["yaw_half"] <= 180
            and 0 <= s["shift_half"] <= 127 and 1 <= s["refine"] <= 15 and 1 <= s["min_points"]
            and 0.0 <= s["min_score_frac"] <= 1.0 and -1 <= s["sensor"] < MAX_BATCH)


def half_width(s):
    return f32(s["grid"] * float(s["cell_m"]) * 0.5)


# ------------------------------------------------------------------------------------------------ steps 1-3
def band(points, s, pose=None):
    """-> (x, y) float32 of the frame (moved by the sensor pose when given), band mask, window mask, cell indices (ix, iy)"""
    p = np.asarray(points, f32)
    p = p.reshape(len(p), -1) if p.size else np.zeros((0, 4), f32)
    if pose is not None:
        p = acs.rig_apply(pose, p[:, :3])
    x, y, z = p[:, 0].copy(), p[:, 1].copy(), p[:, 2].copy()
    with np.errstate(invalid="ignore", over="ignore"):
        r2 = x * x + y * y
        rmin, rmax = f32(s["r_min"]), f32(s["r_max"])
        ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & (z >= f32(s["z_min"])) & (z <= f32(s["z_max"]))
        ok &= (r2 >= rmin * rmin) & (r2 <= rmax * rmax)
        H, cf = half_width(s), f32(s["cell_m"])
        ix = np.where(ok, np.floor((x + H) / cf), -1).astype(np.int64)
        iy = np.where(ok, np.floor((y + H) / cf), -1).astype(np.int64)
    g = s["grid"]
    win = ok & (ix >= 0) & (ix < g) & (iy >= 0) & (iy < g)
    return x, y, ok, win, ix, iy


def field(ix, iy, win, grid):
    """L[iy, ix] = 3 - min(3, Chebyshev distance to the occupied cells), uint8"""
    O = np.zeros((grid, grid), bool)
    O[iy[win], ix[win]] = True
    L = O.astype(np.uint8)
    for r in (1, 2):
        P = np.pad(O, r)
        D = np.zeros_like(O)
        for dy in range(2 * r + 1):
            for dx in range(2 * r + 1):
                D |= P[dy: dy + grid, dx: dx + grid]
        L += D.astype(np.uint8)
    return L, int(O.sum())


def sample(x, y, win, s):
    """the lowest-index window point of each occupied sub-cell in raster order, every k-th when more than max_points -> (xs, ys)"""
    ns = sub_side(s)
    H, sf = half_width(s), f32(s["sub_m"])
    idx = np.nonzero(win)[0]
    sx = np.minimum(np.floor((x[idx] + H) / sf).astype(np.int64), ns - 1)
    sy = np.minimum(np.floor((y[idx] + H) / sf).astype(np.int64), ns - 1)
    key = sy * ns + sx
    _, first = np.unique(key, return_index=True)       # keys ascending; idx is ascending, so the first is the lowest index
    pick = idx[first]
    if len(pick) > s["max_points"]:
        k = -(-len(pick) // s["max_points"])
        pick = pick[::k]
    return x[pick], y[pick]


# ------------------------------------------------------------------------------------------------ step 4
def angle_table(thetas):
    """(float)cos, (float)sin of double angles with the host libm"""
    return (np.array([math.cos(t) for t in thetas], np.float64).astype(f32), np.array([math.sin(t) for t in thetas], np.float64).astype(f32))


def coarse_scores(L, xs, ys, s, j0, k0x, k0y):
    """score[j - (j0 - YH), kx - (k0x - SH), ky - (k0y - SH)] (int64), every hypothesis"""
    g, YH, SH = s["grid"], s["yaw_half"], s["shift_half"]
    W = 2 * SH + 1
    H, cf = half_width(s), f32(s["cell_m"])
    js = np.arange(j0 - YH, j0 + YH + 1)
    cs, sn = angle_table([float(j) * s["yaw_step"] for j in js])
    out = np.zeros((len(js), W, W), np.int64)
    for a in range(len(js)):
        xr = cs[a] * xs - sn[a] * ys
        yr = sn[a] * xs + cs[a] * ys
        bx = np.floor((xr + H) / cf).astype(np.int64) + (k0x - SH)
        by = np.floor((yr + H) / cf).astype(np.int64) + (k0y - SH)
        if len(bx) == 0:
            continue
        lo = min(int(bx.min()), int(by.min()), 0)
        hi = max(int(bx.max()), int(by.max()), g - 1) + W
        pad_lo, pad_hi = -lo, hi - (g - 1)
        Lp = np.pad(L, ((pad_lo, pad_hi), (pad_lo, pad_hi)))
        win = np.lib.stride_tricks.sliding_window_view(Lp, (W, W))      # win[y0, x0][dy, dx] = Lp[y0 + dy, x0 + dx]
        cells, cnt = np.unique(np.stack([by + pad_lo, bx + pad_lo], 1), axis=0, return_counts=True)
        tiles = win[cells[:, 0], cells[:, 1]].reshape(len(cells), W * W).astype(np.float32)     # (m, dy * W + dx)
        # integer sums below 2^24 are exact in float32 in any order
        out[a] = np.rint(cnt.astype(np.float32) @ tiles).astype(np.int64).reshape(W, W).T
    return out


def fine_scores(L, xs, ys, s, j1, k1x, k1y):
    """score[u + R, ax + R, ay + R] of the fine level around the coarse winner"""
    g, R = s["grid"], s["refine"]
    H, cf = half_width(s), f32(s["cell_m"])
    us = np.arange(-R, R + 1)
    cs, sn = angle_table([float(R * j1 + u) * s["yaw_step"] / R for u in us])
    tx = np.array([float(R * k1x + a) * s["cell_m"] / R for a in us], np.float64).astype(f32)
    ty = np.array([float(R * k1y + a) * s["cell_m"] / R for a in us], np.float64).astype(f32)
    out = np.zeros((len(us), len(us), len(us)), np.int64)
    for a in range(len(us)):
        xr = cs[a] * xs - sn[a] * ys
        yr = sn[a] * xs + cs[a] * ys
        cx = np.floor(((xr[None, :] + tx[:, None]) + H) / cf).astype(np.int64)      # (ax, point)
        cy = np.floor(((yr[None, :] + ty[:, None]) + H) / cf).astype(np.int64)      # (ay, point)
        okx, oky = (cx >= 0) & (cx < g), (cy >= 0) & (cy < g)
        v = L[np.clip(cy, 0, g - 1)[None, :, :], np.clip(cx, 0, g - 1)[:, None, :]].astype(np.int64)
        v *= okx[:, None, :] & oky[None, :, :]
        out[a] = v.sum(2)
    return out


def match(L, xs, ys, s, prior):
    """-> (best score, dx, dy, dtheta) of both levels; prior = (px, py, ptheta) in double"""
    j0 = round_half_away(prior[2] / s["yaw_step"])
    k0x, k0y = round_half_away(prior[0] / s["cell_m"]), round_half_away(prior[1] / s["cell_m"])
    YH, SH, R = s["yaw_half"], s["shift_half"], s["refine"]
    sc = coarse_scores(L, xs, ys, s, j0, k0x, k0y)
    a, ix, iy = np.unravel_index(int(np.argmax(sc)), sc.shape)
    j1, k1x, k1y = j0 - YH + a, k0x - SH + ix, k0y - SH + iy
    if R == 1:
        return int(sc[a, ix, iy]), k1x * s["cell_m"], k1y * s["cell_m"], j1 * s["yaw_step"]
    fs = fine_scores(L, xs, ys, s, j1, k1x, k1y)
    u, ax, ay = (int(v) - R for v in np.unravel_index(int(np.argmax(fs)), fs.shape))
    return (int(fs.max()), float(R * k1x + ax) * s["cell_m"] / R, float(R * k1y + ay) * s["cell_m"] / R,
            float(R * j1 + u) * s["yaw_step"] / R)


def round_half_away(v):
    """llround; a prior of 2^20 steps or more (or not finite) rounds to 0"""
    if not math.isfinite(v) or abs(v) >= 2.0 ** 20:
        return 0
    a = abs(v)
    r = math.floor(a)
    return (r + (1 if a - r >= 0.5 else 0)) * (1 if v >= 0 else -1)


# ------------------------------------------------------------------------------------------------ one stream
class Matcher:
    """The state of one stream and the call of steps 1-5 (the definition in include/lmot.h)"""

    def __init__(self, settings=None, poses=None):
        self.s = dict(defaults(), **(settings or {}))
        self.poses = poses                      # the stream's sensor table (list of (3, 4) poses) for sensor >= 0
        self.reset()

    def reset(self):
        self.ts = None
        self.L = None
        self.n_ref = 0
        self.delta = (0.0, 0.0, 0.0)
        self.dt = 0.0
        self.ok = False
        self.Y = 0.0

    def estimate(self, points, ts):
        s = self.s
        pose = None if s["sensor"] < 0 else self.poses[s["sensor"]]
        x, y, ok, win, ix, iy = band(points, s, pose)
        L, n_occ = field(ix, iy, win, s["grid"])
        xs, ys = sample(x, y, win, s)
        n_used = len(xs)
        dt = (ts - self.ts) / 1e6 if self.ts is not None else float("nan")
        dt_ok = self.ts is not None and math.isfinite(dt) and dt > 0
        out = dict(ok=0, n_used=n_used, n_ref=0, score=0, score_max=3 * n_used, dx=0.0, dy=0.0, dtheta=0.0, v=0.0, yaw=0.0)
        if dt_ok:
            if self.ok:
                r = dt / self.dt
                prior = (self.delta[0] * r, self.delta[1] * r, self.delta[2] * r)
            else:
                prior = (0.0, 0.0, 0.0)
            delta, good = prior, False
            if self.L is not None and n_used >= s["min_points"]:
                best, dx, dy, dth = match(self.L, xs, ys, s, prior)
                out["score"], out["n_ref"] = best, self.n_ref
                if best >= s["min_score_frac"] * 3 * n_used:
                    delta, good = (dx, dy, dth), True
            out["ok"] = int(good)
            out["dx"], out["dy"], out["dtheta"] = delta
            out["v"] = (delta[0] * math.cos(delta[2]) + delta[1] * math.sin(delta[2])) / dt
            self.Y += delta[2]
            self.delta, self.ok, self.dt = delta, good, dt
        else:
            self.delta, self.ok, self.dt = (0.0, 0.0, 0.0), False, 0.0
        out["yaw"] = self.Y
        self.L, self.n_ref, self.ts = L, n_occ, ts
        return out


# ------------------------------------------------------------------------------------------------ brute force (small clouds)
def brute_match(L, xs, ys, s, prior):
    """step 4 hypothesis by hypothesis, point by point, in Python scalars rounded through numpy float32"""
    g, YH, SH, R = s["grid"], s["yaw_half"], s["shift_half"], s["refine"]
    H, cf = half_width(s), f32(s["cell_m"])
    j0 = round_half_away(prior[2] / s["yaw_step"])
    k0x, k0y = round_half_away(prior[0] / s["cell_m"]), round_half_away(prior[1] / s["cell_m"])

    def at(cx, cy):
        return int(L[cy, cx]) if 0 <= cx < g and 0 <= cy < g else 0

    best = None
    for j in range(j0 - YH, j0 + YH + 1):
        cs, sn = f32(math.cos(float(j) * s["yaw_step"])), f32(math.sin(float(j) * s["yaw_step"]))
        base = [(int(np.floor((f32(cs * x) - f32(sn * y) + H) / cf)), int(np.floor((f32(sn * x) + f32(cs * y) + H) / cf)))
                for x, y in zip(xs, ys)]
        for kx in range(k0x - SH, k0x + SH + 1):
            for ky in range(k0y - SH, k0y + SH + 1):
                sc = sum(at(bx + kx, by + ky) for bx, by in base)
                if best is None or sc > best[0]:
                    best = (sc, j, kx, ky)
    sc, j1, k1x, k1y = best
    if R == 1:
        return sc, k1x * s["cell_m"], k1y * s["cell_m"], j1 * s["yaw_step"]
    best = None
    for u in range(-R, R + 1):
        th = float(R * j1 + u) * s["yaw_step"] / R
        cs, sn = f32(math.cos(th)), f32(math.sin(th))
        rot = [(f32(cs * x) - f32(sn * y), f32(sn * x) + f32(cs * y)) for x, y in zip(xs, ys)]
        for ax in range(-R, R + 1):
            tx = f32(float(R * k1x + ax) * s["cell_m"] / R)
            for ay in range(-R, R + 1):
                ty = f32(float(R * k1y + ay) * s["cell_m"] / R)
                sc = sum(at(int(np.floor(((xr + tx) + H) / cf)), int(np.floor(((yr + ty) + H) / cf))) for xr, yr in rot)
                if best is None or sc > best[0]:
                    best = (sc, u, ax, ay)
    sc, u, ax, ay = best
    return sc, float(R * k1x + ax) * s["cell_m"] / R, float(R * k1y + ay) * s["cell_m"] / R, float(R * j1 + u) * s["yaw_step"] / R


# ------------------------------------------------------------------------------------------------ drives
def fold_step(h, ts, v, yaw):
    """origin_points_fold (tracker.cu, getOriginPoints) on h = dict(init, ts, pre_yaw, fold) -> the fold after this step"""
    ego_yaw = yaw + (-0.63035 - math.pi / 2)
    if not h["init"]:
        h.update(init=True, fold=[0.0, 0.0, -math.pi / 2])
    else:
        dt = (ts - h["ts"]) / 1000000.0
        d = ego_yaw - h["pre_yaw"]
        dX, dY = dt * v * math.cos(d), dt * v * math.sin(d)
        x, y, w = h["fold"]
        x -= dX
        y -= dY
        r = d * -1
        w += r
        h["fold"] = [math.cos(r) * x - math.sin(r) * y, math.sin(r) * x + math.cos(r) * y, w]
    h["ts"], h["pre_yaw"] = ts, ego_yaw
    return np.array(h["fold"], np.float64)


BEAMS = {16: acs.SPARSE, 32: dict(rings=32, azimuths=1024, elev_top_deg=15.0, elev_bot_deg=-15.0),
         64: dict(rings=64, azimuths=1875, elev_top_deg=15.0, elev_bot_deg=-20.0)}


def drive_frames(synth, kind, n, beams=16, movers=0, seed=3):
    """[(ts, v_gps, yaw_gps, points, fold, static object positions in the sensor frame)] of accumulate_scenes' static scene seen along
    the drive, rendered through the fold (so the true delta of every step is the fold's own), plus `movers` of synth's moving objects
    (global frame, constant velocity / turn rate)"""
    pos, oyaw, size = acs.static_objects(seed)
    cfg = synth.SceneConfig(n_objects=0, seed=seed, **BEAMS[beams])
    mv = None
    if movers:
        m = synth.make_scene(synth.SceneConfig(n_objects=movers, seed=seed + 100, roi_half=20.0))
        keep = m.vel > 0
        mv = synth.Scene(m.cfg, m.pos[keep] + np.array([0.0, -10.0]), m.yaw[keep], m.size[keep], m.vel[keep], m.yawrate[keep], 0)
    h = dict(init=False, ts=0.0, pre_yaw=0.0, fold=None)
    out = []
    for t, (v, yg) in enumerate(acs.drive(kind, n)):
        ts = (t + 1) * synth.DT_US
        fold = fold_step(h, ts, v, yg)
        P, W, S = pos, oyaw, size
        if mv is not None:
            P, W, S = np.concatenate([pos, mv.pos]), np.concatenate([oyaw, mv.yaw]), np.concatenate([size, mv.size])
        p, w = acs.sensor_frame(fold, P, W)
        sc = synth.Scene(cfg, p, w, S.copy(), np.zeros(len(p)), np.zeros(len(p)), t)
        out.append((ts, v, yg, synth.render(sc), fold, p[: len(pos)]))
        if mv is not None:
            synth.advance(mv)
    return out


def true_delta(fold_prev, fold_t, dt, v):
    """the fold's delta of a step: dtheta = diffYaw, (dx, dy) = dt v (cos, sin) of it"""
    d = -(fold_t[2] - fold_prev[2])
    return dt * v * math.cos(d), dt * v * math.sin(d), d
