"""GPU parity of the tracker chain in the size regimes where its kernels switch to a second implementation.

TA (imm_predict_gate_kernel), TB (imm_update_kernel) and TC (spawn_output_kernel) each choose a code path by data size: a
compact list of at most 32 gated boxes per track and 512 boxes per step, a fast TC path for at most 256 / 512 active tracks,
unrolled copies of the previous result block for the first 1024..4096 table rows, a queue of 1024 (visible box, track) pairs,
grid-stride loops over more active tracks than CTAs.  Every test here feeds one of the far sides on synthetic box lists, compares
the CUDA tracker with the reference compiled from its own sources on every step (the bars of test_tracker_gpu), and proves from
the REFERENCE side -- never from the CUDA side -- that it reached its regime, printing what it reached.
"""
import numpy as np
import pytest

from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu

OFF = -0.63035 - np.pi / 2          # firstEgoYawOffset_, imm_ukf_jpda.cpp:70
D_STATIC, D_VIS, D_X, D_ZPRED, D_S, D_BB = 2, 3, 4, 127, 133, 187      # dump columns (api.cu, oracle/ref_harness.cpp)
GAMMA_G = 9.22                      # gate threshold, imm_ukf_jpda.cpp:26
STEP_US = 1e5                       # 10 Hz
CROWD = (31, 32, 33, 40, 64, 100)   # boxes around one track: both sides of the 32-entry compact list


# ------------------------------------------------------------------------------------------------ scene building (numpy)
def boxes_at(centres, half_extent=(1.0, 0.5)):
    """axis-aligned boxes (B, 8, 3) around `centres` (B, 2); half_extent (2,) or (B, 2).  (0, 0): four identical corners."""
    c = np.asarray(centres, np.float64).reshape(-1, 2)
    h = np.broadcast_to(np.asarray(half_extent, np.float64), c.shape)
    out = np.zeros((len(c), 8, 3), np.float32)
    sign = np.array([[-1.0, -1.0], [-1.0, 1.0], [1.0, 1.0], [1.0, -1.0]])
    for k in range(4):
        out[:, k, :2] = c + sign[k] * h; out[:, k, 2] = -2.0
        out[:, 4 + k, :2] = c + sign[k] * h; out[:, 4 + k, 2] = 0.0
    return out


def lattice(nx, ny, pitch, origin=(12.0, 12.0)):
    """sites away from (-1.5, -9), where the reference's first call puts its one hard-coded track (imm_ukf_jpda.cpp:741-795)"""
    gx, gy = np.meshgrid(np.arange(nx) * pitch + origin[0], np.arange(ny) * pitch + origin[1], indexing="ij")
    return np.stack([gx.ravel(), gy.ravel()], 1)


def disk(rng, n, radius):
    r = radius * np.sqrt(rng.random(n))
    a = rng.random(n) * 2 * np.pi
    return np.stack([r * np.cos(a), r * np.sin(a)], 1)


def clutter(rng, n):
    """isolated far boxes: none is gated by a track of the scene, so each spawns one"""
    return rng.uniform((-260.0, -150.0), (-120.0, 150.0), (n, 2))


# ------------------------------------------------------------------------------------------------ reference-side regime checks
def box_centres(boxes):
    """getCpFromBbox (imm_ukf_jpda.cpp:465-479): S1 / S2 in float, the rest in double"""
    b = np.asarray(boxes, np.float32)
    p1x, p1y, p2x, p2y = b[:, 0, 0], b[:, 0, 1], b[:, 1, 0], b[:, 1, 1]
    p3x, p3y, p4x, p4y = b[:, 2, 0], b[:, 2, 1], b[:, 3, 0], b[:, 3, 1]
    with np.errstate(all="ignore"):
        s1 = (((p4x - p2x) * (p1y - p2y) - (p4y - p2y) * (p1x - p2x)) / np.float32(2)).astype(np.float64)
        s2 = (((p4x - p2x) * (p2y - p3y) - (p4y - p2y) * (p2x - p3x)) / np.float32(2)).astype(np.float64)
        cx = p1x.astype(np.float64) + (p3x - p1x).astype(np.float64) * s1 / (s1 + s2)
        cy = p1y.astype(np.float64) + (p3y - p1y).astype(np.float64) * s1 / (s1 + s2)
    return np.stack([cx, cy], 1)


def gate_nis(dump_after, boxes, rows):
    """NIS of every box against each track of `rows`, as the gate evaluated it (imm_ukf_jpda.cpp:843-869, :205-257): zPred / S of
    the model with the largest det(S) (findMaxZandS), S scaled by 4.  zPred and S are written only by the prediction
    (ukf.cpp:882-899), so the dump taken after the step holds the values the gate used."""
    c = box_centres(boxes)
    out = np.full((len(rows), len(c)), np.inf)
    for r, i in enumerate(rows):
        d = dump_after[i]
        S = d[D_S:D_S + 12].reshape(3, 2, 2)
        z = d[D_ZPRED:D_ZPRED + 6].reshape(3, 2)
        det = S[:, 0, 0] * S[:, 1, 1] - S[:, 0, 1] * S[:, 1, 0]
        mm = ((0 if det[0] > det[2] else 2) if det[0] > det[1] else (1 if det[1] > det[2] else 2))
        with np.errstate(all="ignore"):
            Si = np.linalg.inv(4 * S[mm])
            dd = c - z[mm]
            out[r] = np.einsum("ni,ij,nj->n", dd, Si, dd)
    return out


def gated_counts(pre, post, boxes):
    """boxes in the gate of every track that was live before the step (index, count) -> {index: count}"""
    rows = np.nonzero(pre[:, 0] > 0)[0]
    if len(boxes) == 0 or len(rows) == 0:
        return {}
    g = gate_nis(post, boxes, rows) < GAMMA_G
    return dict(zip(rows.tolist(), g.sum(1).tolist()))


def active_count(d):
    """the rows TA / TB / TC visit: live, or dead with isVisBB_ still set"""
    return int(((d[:, 0] != 0) | (d[:, D_VIS] != 0)).sum())


def candidate_pairs(post, live, per=None):
    """(visible box, track of `live`) pairs whose position lies inside the box's axis-aligned bounds: with the live tracks, the
    pairs TC's bounds pre-test queues for its exact test (its margin only adds pairs).  per: the counts of every run of `per`
    visible boxes in track-index order (the general path stages 128 visible boxes per pass and empties its queue after each) as a
    list; otherwise the total."""
    vis = np.nonzero(post[:, D_VIS] > 0)[0]
    if len(vis) == 0 or len(live) == 0:
        return [0] if per else 0
    c = post[vis][:, D_BB:D_BB + 12].reshape(-1, 4, 3)[:, :, :2]
    lo, hi = c.min(1), c.max(1)
    p = post[live][:, D_X:D_X + 2]
    inside = np.all((p[None] >= lo[:, None]) & (p[None] <= hi[:, None]), axis=2)
    inside &= vis[:, None] != live[None, :]
    per_box = inside.sum(1)
    if per:
        return [int(per_box[i:i + per].sum()) for i in range(0, len(vis), per)]
    return int(per_box.sum())


def dead_decides_merge(pre, post):
    """visible tracks k that only lower-index visible boxes contain, whose own box holds no live position but a dead one, and that
    kept trackNum 5.  mergeOverSegmentation (imm_ukf_jpda.cpp:666-700) writes trackNum[k] = 0 for every box i < k containing k,
    then 5 when k's box contains any other track, dead ones included: without the dead row such a k would end at 0.  (Boxes here
    are axis-aligned, so "contains" is "strictly inside the bounds".)"""
    vis = np.nonzero(post[:, D_VIS] > 0)[0]
    live = np.ones(len(post), bool)
    live[:len(pre)] = pre[:, 0] > 0
    xy = post[:, D_X:D_X + 2]
    c = post[vis][:, D_BB:D_BB + 12].reshape(-1, 4, 3)[:, :, :2]
    lo, hi = c.min(1), c.max(1)
    inside = np.all((xy[None] > lo[:, None]) & (xy[None] < hi[:, None]), axis=2)      # [visible box, track]
    n = 0
    for v, k in enumerate(vis):
        containers = vis[inside[:, k] & (vis != k)]
        held = inside[v] & (np.arange(len(post)) != k)
        if len(containers) and containers.max() < k and not (held & live).any() and (held & ~live).any() and post[k, 0] == 5:
            n += 1
    return n


# ------------------------------------------------------------------------------------------------ comparison
def _compare(a, b, da, db, forced, f, n=None):
    """the project's bars on one step (test_teacher_forced_steps); n: compare the first n tracks only.  -> worst state error"""
    if n is None:
        n = len(a["track_manage"])
        assert da.shape == db.shape, (f, da.shape, db.shape)
    assert len(b["track_manage"]) == n and len(db) >= n, (f, len(b["track_manage"]), n)
    for k in ("track_manage", "is_static", "is_vis"):
        assert np.array_equal(a[k][:n], b[k][:n]), (f, k)
    da, db = da[:n], db[:n]
    assert np.array_equal(da[:, INTS], db[:, INTS]), f
    np.testing.assert_allclose(b["targets"][:n], a["targets"][:n], rtol=1e-5, atol=1e-5, err_msg=str(f))
    np.testing.assert_allclose(b["vandyaw"][:n], a["vandyaw"][:n], rtol=1e-4, atol=1e-6, err_msg=str(f))
    assert a["vis_bb"].shape == b["vis_bb"].shape, f
    np.testing.assert_allclose(b["vis_bb"], a["vis_bb"], rtol=1e-5, atol=1e-5, err_msg=str(f))
    rows = (da[:, 0] > 0) if forced else _pd_tracks(da)
    err = _rel_err(da[rows][:, STATE], db[rows][:, STATE])
    worst = float(err.max()) if err.size else 0.0
    assert worst < TOL, (f, worst)
    box = rows & (da[:, 186] > 0)            # box-tracker state (BBox_, bestBBox_, bestYaw_) of the tracks that have a box
    np.testing.assert_allclose(db[box][:, 186:236], da[box][:, 186:236], rtol=1e-5, atol=1e-5, err_msg=str(f))
    np.testing.assert_allclose(db[box][:, 175], da[box][:, 175], rtol=1e-5, atol=1e-6, err_msg=str(f))
    return worst


class _Lockstep:
    """the reference and one CUDA context stepped on the same box lists, every step compared"""

    def __init__(self, ref, ctx, forced=False, cuda_step=None):
        self.ref, self.ctx, self.forced = ref, ctx, forced
        self.cuda_step = cuda_step or ctx.track_step
        self.worst, self.steps = 0.0, 0

    def reset(self):
        self.ref.tracker_reset(); self.ctx.tracker_reset()

    def load(self, state, ts):
        for t in (self.ref, self.ctx):
            t.tracker_load(state, 1, ts, 0.0, OFF, OFF, -np.pi / 2)

    def step(self, boxes, ts, v=0.0, yaw=0.0, n=None):
        """-> (reference dump before, reference result, reference dump after, CUDA result)"""
        pre = self.ref.tracker_dump()
        a = self.ref.tracker_step(boxes, ts, v, yaw)
        b = self.cuda_step(boxes, ts, v, yaw)
        self.warning = getattr(self.ctx, "last_warning", None)      # (the dump below is a call of its own)
        da, db = self.ref.tracker_dump(), self.ctx.tracker_dump()
        self.worst = max(self.worst, _compare(a, b, da, db, self.forced, (self.steps, ts), n))
        self.steps += 1
        return pre, a, da, b


def _mature(rng, pos, n_frames=6, half=(1.0, 0.5)):
    """clean boxes on fixed sites: frame 1 spawns, frame 5 sees trackNum 5 with lifetime 4 (visible)"""
    return [boxes_at(pos + rng.normal(0, 0.02, pos.shape), half) for _ in range(n_frames)]


# ------------------------------------------------------------------------------------------------ 1. crowded gates
def _crowd_scene(seed, n_crowded, pad_to, n_steps):
    """8 x 8 lattice (8 m) plus one partner track 1 m from site 9.  Crowd steps: site i < n_crowded sees CROWD[(i + s) % 6] boxes
    within 0.3 m of its track, the pair one shared crowd of 40 between them, every other site one clean box, far clutter pads the
    list to pad_to[s] boxes."""
    rng = np.random.default_rng(seed)
    pos = np.concatenate([lattice(8, 8, 8.0), lattice(8, 8, 8.0)[9:10] + (0.0, 1.0)])
    mature = _mature(rng, pos)
    steps = []
    for s in range(n_steps):
        cs = []
        for i, p in enumerate(pos):
            if i in (9, 64):
                continue
            n = CROWD[(i + s) % len(CROWD)] if i < n_crowded else 1
            cs.append(p + (disk(rng, n, 0.3) if n > 1 else rng.normal(0, 0.02, (1, 2))))
        cs.append((pos[9] + pos[64]) / 2 + disk(rng, 40, 0.2))
        c = np.concatenate(cs)
        if pad_to[s] > len(c):
            c = np.concatenate([c, clutter(rng, pad_to[s] - len(c))])
        steps.append(boxes_at(c, (0.4, 0.25)))
    return mature, steps


def _crowd_regime(pre, post, boxes, reach):
    counts = gated_counts(pre, post, boxes)
    reach["gated"].update(counts.values())
    reach["M"].add(len(boxes))
    rows = np.array(sorted(counts))
    if len(rows):
        g = gate_nis(post, boxes, rows) < GAMMA_G
        reach["shared"] = max(reach["shared"], int((g.sum(0) >= 2).sum()))


def _check_crowd_reach(reach, big):
    assert {32, 33} <= reach["gated"] and max(reach["gated"]) >= 100, sorted(reach["gated"])
    assert reach["shared"] >= 40, reach["shared"]          # the shared crowd: every box in two gates
    if big:
        assert min(reach["M"]) > 512 and max(reach["M"]) == 1024, reach["M"]
    else:
        assert max(reach["M"]) <= 512, reach["M"]


def _run_crowd(ref, ctx, big, forced, seed=3):
    pad = (1024, 800, 1024, 700) if big else (0, 0, 0, 0)
    mature, steps = _crowd_scene(seed, 12 if big else 6, pad, 4)
    reach = dict(gated=set(), M=set(), shared=0)
    run = _Lockstep(ref, ctx, forced)
    ts = 0.0
    run.reset()
    if forced:
        for b in mature:
            ts += STEP_US
            ref.tracker_step(b, ts)
        for s, b in enumerate(steps):       # every load is followed by two steps: `full`, then TC's incremental path
            if s % 2 == 0:
                run.load(ref.tracker_dump(), ts)
            ts += STEP_US
            pre, a, da, _ = run.step(b, ts)
            _crowd_regime(pre, da, b, reach)
    else:
        for f, b in enumerate(mature + steps):
            ts += STEP_US
            pre, a, da, _ = run.step(b, ts)
            if f >= len(mature):
                _crowd_regime(pre, da, b, reach)
    return run, reach


@pytest.mark.parametrize("big", [False, True], ids=["M<=512", "M>512"])
@pytest.mark.parametrize("forced", [False, True], ids=["free", "forced"])
def test_crowded_gates(lm, ref_intended, big, forced):
    """more than 32 boxes in one track's gate: TA cuts its compact list at 32, TB rebuilds the list from the gate words and
    its model warps run the serial path (centres recomputed for k >= 32); above 512 boxes TA gates outside its unrolled chunks and
    hands TB no list at all.  One crowd is shared by two tracks 1 m apart (first_setter and lifetime ties)."""
    run, reach = _run_crowd(ref_intended, lm, big, forced)
    _check_crowd_reach(reach, big)
    print(f"crowded gates (M {'>' if big else '<='} 512, {'teacher-forced' if forced else 'free-running'}): regime reached: gated per "
          f"track {sorted(reach['gated'] - {0, 1})}, M {sorted(reach['M'])[-1]} max / {sorted(reach['M'])[0]} min, boxes in two gates "
          f"{reach['shared']}; worst relative state error {run.worst:.3g} over {run.steps} steps")


def _second_init_scene(seed):
    """8 x 8 lattice: frame 1 spawns; frame 2 (trackNum 1: secondInit) puts a crowd of > 32 boxes around 12 tracks, the box
    closest to the track at crowd position >= 32 and the first 32 in decreasing distance (the running minimum moves in every
    chunk); frames 3-4 crowd them again (trackNum 2: the PDA update with > 32 measurements)"""
    rng = np.random.default_rng(seed)
    pos = lattice(8, 8, 8.0)
    frames = [boxes_at(pos, (0.4, 0.25)) for _ in range(2)]
    for f in range(3):
        cs = []
        for i, p in enumerate(pos):
            if i >= 12:
                cs.append(p[None] + rng.normal(0, 0.02, (1, 2)))
                continue
            n = (33, 40, 47, 64, 100, 70)[(i + f) % 6]
            r = np.sort(rng.uniform(0.05, 0.3, n))[::-1]
            a = rng.random(n) * 2 * np.pi
            crowd = np.stack([r * np.cos(a), r * np.sin(a)], 1)
            crowd[32 + (i * 7) % (n - 32)] = (0.001, 0.0)      # the others are >= 5 cm away
            cs.append(p + crowd)
        frames.append(boxes_at(np.concatenate(cs), (0.4, 0.25)))
    return frames


@pytest.mark.parametrize("forced", [False, True], ids=["free", "forced"])
def test_second_init_crowd(lm, ref_intended, forced):
    """secondInit (the step after the spawn) with more than 32 gated boxes: TA carries the running minimum of the NIS across
    32-box chunks, TB's warp 3 takes the minimum over k >= 32"""
    ref = ref_intended
    frames = _second_init_scene(5)
    run = _Lockstep(ref, lm, forced)
    run.reset()
    hits, ts = [], 0.0
    for f, b in enumerate(frames):
        ts += STEP_US
        if forced and f < 2:
            ref.tracker_step(b, ts)
            continue
        if forced and f in (2, 4):
            run.load(ref.tracker_dump(), ts - STEP_US)
        pre, a, da, _ = run.step(b, ts)
        rows = np.nonzero(pre[:, 0] == 1)[0]
        if f == 2 and len(rows):
            nis = gate_nis(da, b, rows)
            for r, i in enumerate(rows):
                g = np.nonzero(nis[r] < GAMMA_G)[0]
                if len(g) > 32:
                    k = int(np.argmin(nis[r][g]))
                    hits.append((len(g), k))
    assert len(hits) >= 10 and all(k >= 32 for _, k in hits), hits
    print(f"secondInit crowds ({'teacher-forced' if forced else 'free-running'}): regime reached: (gated boxes, position of the "
          f"smallest NIS) {hits}; worst relative state error {run.worst:.3g}")


# ------------------------------------------------------------------------------------------------ 2. grid stride
def _churn_scene(seed, n_frames, n_obj=160):
    """objects that move, drop out for a frame, vanish and appear: a table of every kind (secondInit, mature, dying, dead)"""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-70, 70, (n_obj, 2)) + (90.0, 0.0)
    vel = rng.normal(0, 1.0, (n_obj, 2))
    frames = []
    for _ in range(n_frames):
        pos += 0.1 * vel
        gone = rng.random(n_obj) < 0.03
        pos[gone] = rng.uniform(-70, 70, (int(gone.sum()), 2)) + (90.0, 0.0)
        seen = rng.random(n_obj) < 0.85
        frames.append(boxes_at(pos[seen] + rng.normal(0, 0.02, (int(seen.sum()), 2))))
    return frames


def test_grid_stride_tracker_ctas(pkg, ref_intended, monkeypatch):
    """TA and TB walk the active list with grid-stride loops (trk_ctas CTAs, 4 per SM by default).  With 8 CTAs every CTA walks
    dozens of tracks of mixed kinds, reusing its shared state and leaving early on dead / killed / secondInit tracks."""
    monkeypatch.setenv("LMOT_TRK_CTAS", "8")
    ctx = pkg.Lmot()
    try:
        run, reach = _run_crowd(ref_intended, ctx, big=True, forced=False, seed=4)
        _check_crowd_reach(reach, True)
        churn = _Lockstep(ref_intended, ctx)
        churn.reset()
        kinds, act = set(), []
        for f, b in enumerate(_churn_scene(6, 16)):
            pre, a, da, _ = churn.step(b, (f + 1) * STEP_US)
            act.append(active_count(pre))
            kinds.update(pre[:, 0].astype(int).tolist())
        assert max(act) >= 20 * 8 and {0, 1, 2, 5} <= kinds, (max(act), kinds)
        print(f"grid stride, 8 CTAs: regime reached: crowd scene gated per track up to {max(reach['gated'])}, M up to "
              f"{max(reach['M'])}; churned scene up to {max(act)} active tracks, trackNum kinds {sorted(kinds)}; worst relative "
              f"state error {max(run.worst, churn.worst):.3g}")
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 3. TC width boundaries
@pytest.mark.parametrize("wide", ["0", "1", None], ids=["tc256", "tc512", "tc_by_count"])
@pytest.mark.parametrize("n", [256, 257, 512, 513])
def test_tc_width_boundaries(pkg, ref_intended, n, wide, monkeypatch):
    """exactly 256 / 257 / 512 / 513 active tracks: the last and the first count of spawn_output_kernel's one-track-per-thread
    fast path in its 256- and 512-thread variants"""
    if wide is not None:
        monkeypatch.setenv("LMOT_TC_WIDE", wide)
    rng = np.random.default_rng(n)
    pos = lattice(23, 23, 8.0)[:n]
    ctx = pkg.Lmot()
    try:
        run = _Lockstep(ref_intended, ctx)
        run.reset()
        act = []
        for f, b in enumerate(_mature(rng, pos, 9)):
            pre, a, da, _ = run.step(b, (f + 1) * STEP_US)
            if f >= 6:
                act.append((active_count(pre), active_count(da)))
        assert all(x == (n, n) for x in act), act
        print(f"TC width {wide}: regime reached: active tracks {act}; worst relative state error {run.worst:.3g}")
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 4. overlapping visible boxes
MERGE_A, MERGE_B, MERGE_DEAD = (200.0, 20.0), (208.0, 20.0), (208.5, 20.3)


def _overlap_frames(nx, n_frames):
    """tracks on a 4 m lattice whose boxes are 18 m wide from the first frame on: a box contains the positions of the 24 nearest
    other tracks.  Apart from the lattice (and after it in box order): track A with a 20 m box, and 8 m away (beyond A's gate),
    inside A's box, track B with a 2 m box around a dead row (a track spawned at frame 1 and starved at frame 2)."""
    pos = lattice(nx, nx, 4.0, origin=(20.0, 20.0))
    ghosts = boxes_at(np.array([MERGE_DEAD, (200.0, -60.0)]))
    frames = [ghosts, ghosts, boxes_at(np.zeros((0, 2)))]
    ab = np.concatenate([boxes_at([MERGE_A], (10.0, 10.0)), boxes_at([MERGE_B], (1.0, 1.0))])
    return frames + [np.concatenate([boxes_at(pos, (9.0, 9.0)), ab]) for _ in range(n_frames)]


@pytest.mark.parametrize("path", ["fast", "general_full", "general"])
def test_overlapping_visible_boxes(pkg, ref_intended, path, monkeypatch):
    """mergeOverSegmentation under load: every visible box contains many other tracks' positions, more pairs than TC's queue for
    the exact test holds (1024; the rest are tested inline).  The fast path queues the pairs of all visible boxes at once, the
    general path those of 128 visible boxes per pass, so there one pass must overflow.  fast: 16 x 16 tracks free-running on the
    512-thread variant; general_full: the same step right after lmot_tracker_load into a fresh context; general: 20 x 20 tracks
    on the 256-thread variant.  Track B (see _overlap_frames) keeps trackNum 5 only because pass B tests its box against every
    track, dead ones included."""
    ref = ref_intended
    if path != "general_full":
        monkeypatch.setenv("LMOT_TC_WIDE", "1" if path == "fast" else "0")
    nx = 20 if path == "general" else 16
    frames = _overlap_frames(nx, 10)
    ctx = pkg.Lmot()
    try:
        run = _Lockstep(ref, ctx)
        run.reset()
        reached = []
        for f, b in enumerate(frames):
            ts = (f + 1) * STEP_US
            if path == "general_full":
                state = ref.tracker_dump()
                ref.tracker_step(b, ts)
                if max(candidate_pairs(ref.tracker_dump(), np.nonzero(state[:, 0] > 0)[0], per=128)) <= 1024:
                    continue
                ref.tracker_load(state, 1, ts - STEP_US, 0.0, OFF, OFF, -np.pi / 2)
                ctx.close()
                ctx = pkg.Lmot()
                run = _Lockstep(ref, ctx)
                run.load(state, ts - STEP_US)
            pre, a, da, _ = run.step(b, ts)
            live = np.nonzero(pre[:, 0] > 0)[0]
            pairs = candidate_pairs(da, live)
            if pairs > 1024:
                reached.append((f, pairs, max(candidate_pairs(da, live, per=128)), active_count(pre), dead_decides_merge(pre, da)))
            if path == "general_full" and reached:
                break
        assert reached, "no step with more than 1024 candidate pairs"
        for f, pairs, pass_max, act, dead in reached:
            if path == "fast":
                assert act <= 512, reached
            else:
                assert pass_max > 1024 and (path == "general_full" or act > 256), reached
        assert any(r[-1] > 0 for r in reached), reached
        print(f"overlapping boxes ({path}): regime reached: (frame, candidate pairs, most pairs in one 128-box pass, active tracks "
              f"before, tracks kept alive by a dead row) {reached}; worst relative state error {run.worst:.3g}")
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 5. long-lived table
def _long_table(ref, n_dead=4620, seed=8):
    """n_dead dead rows (trackNum 0, spread over the scene, half of them static, a few inside the later visible boxes), then the
    rows of a reference run over a 6 x 10 lattice (60 live tracks and the dead first-call track)"""
    rng = np.random.default_rng(seed)
    pos = lattice(6, 10, 8.0)
    ref.tracker_reset()
    ts = 0.0
    for b in _mature(rng, pos, 7):
        ts += STEP_US
        ref.tracker_step(b, ts)
    live = ref.tracker_dump()
    assert (live[:, 0] == 5).sum() == 60
    dead = np.repeat(live[-1:], n_dead, 0)
    dead[:, 0] = 0; dead[:, 1] = rng.integers(0, 9, n_dead); dead[:, D_STATIC] = rng.random(n_dead) < 0.5; dead[:, D_VIS] = 0
    xy = rng.uniform(-40, 100, (n_dead, 2))
    xy[:40] = pos[rng.integers(0, 60, 40)] + rng.uniform(-0.5, 0.5, (40, 2)) * (1.0, 0.4)
    yaw = rng.uniform(-np.pi, np.pi, n_dead)
    for m in range(4):
        dead[:, D_X + 5 * m] = xy[:, 0]; dead[:, D_X + 5 * m + 1] = xy[:, 1]
        dead[:, D_X + 5 * m + 2] = rng.uniform(0, 3, n_dead); dead[:, D_X + 5 * m + 3] = yaw
    return np.concatenate([dead, live]), pos, ts


@pytest.mark.parametrize("route", ["track_step", "lists_dev"])
def test_long_table_moving_ego(pkg, ref_intended, route):
    """> 4600 rows, nearly all dead -- the steady state of a long drive (include/lmot.h).  Every row is re-emitted every step, a
    dead one with its yaw re-offset by the moving ego.  track_step patches the one result block in place; lists_dev steps a
    device box buffer through lmot_track_step_lists_dev into a ring of result blocks, so TC copies the previous block first
    (remainder copies beyond 1024 / 1365 / 2048 / 4096 rows).  track_step also fills the table in the middle of a spawn pass."""
    import torch
    ref = ref_intended
    table, pos, ts = _long_table(ref)
    T0 = len(table)
    rng = np.random.default_rng(9)
    p = pkg.default_params()
    if route == "track_step":
        p.max_tracks = T0 + 100
    ctx = pkg.Lmot(p)
    try:
        cuda_step = None
        if route == "lists_dev":
            assert ctx.params.result_ring >= 2
            cap = int(ctx.params.max_boxes)
            d_lists = torch.zeros((cap, 8, 3), dtype=torch.float32, device="cuda")
            d_count = torch.zeros(1, dtype=torch.int32, device="cuda")

            def cuda_step(boxes, ts_, v, yaw):
                d_lists[: len(boxes)].copy_(torch.from_numpy(boxes))
                d_count.fill_(len(boxes))
                torch.cuda.synchronize()
                ctx.track_step_lists_dev(d_lists.data_ptr(), d_count.data_ptr(), 1, cap, ts_, v, yaw)
                return ctx.frame_fetch()
        run = _Lockstep(ref, ctx, forced=True, cuda_step=cuda_step)
        run.load(table, ts)
        rows = []
        for f in range(12):
            ts += STEP_US
            b = boxes_at(pos + rng.normal(0, 0.02, pos.shape))
            pre, a, da, _ = run.step(b, ts, 3.0 + 0.1 * f, 0.02 * (f + 1))
            rows.append(len(pre))
            assert active_count(pre) == 60 and len(a["track_manage"]) == T0, f
        assert min(rows) > 4096, rows
        msg = ""
        if route == "track_step":
            for f in range(2):              # 300 unmatched boxes, room for 100: the table fills in the middle of the spawn pass
                ts += STEP_US
                extra = clutter(rng, 300) if f == 0 else np.zeros((0, 2))
                b = boxes_at(np.concatenate([pos + rng.normal(0, 0.02, pos.shape), extra]))
                pre, a, da, _ = run.step(b, ts, 4.0, 0.3, n=T0 + 100)
                if f == 0:
                    assert len(a["track_manage"]) == T0 + 300 and ref.tracker_num_tracks() == T0 + 300
                    assert run.warning == pkg.WARN_TRACK_TABLE_FULL and ctx.tracker_num_tracks() == T0 + 100
            msg = f", table full at {T0 + 100} rows with 300 boxes to spawn (warning {pkg.WARN_TRACK_TABLE_FULL})"
        print(f"long table ({route}): regime reached: {min(rows)}..{max(rows)} rows, 60 active{msg}; worst relative state error "
              f"{run.worst:.3g}")
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 6. degenerate lists
def test_degenerate_box_lists(lm, ref_intended):
    """What a ROS trackbox message may carry: exact duplicates (ties in first_setter, association and spawn order), alone and
    in a crowd; a zero-area box, whose centre is NaN (never gated, spawns a NaN track the reference's guards kill); boxes with one
    centre and different extents, and boxes at the same floor(distance) (associateBB takes the first)."""
    ref = ref_intended
    rng = np.random.default_rng(10)
    pos = lattice(4, 4, 8.0)
    frames = _mature(rng, pos)
    dup_site, nan_site = np.array([[80.0, 12.0]]), np.array([[80.0, 40.0]])
    unit = (1.0, 0.5)
    for f in range(6):
        lists = []                                       # (centres, half extents) in box order
        for i, p in enumerate(pos):
            if i == 0:                                   # a crowd of 12 boxes, each twice
                lists.append((np.repeat(p + disk(rng, 12, 0.3), 2, 0), unit))
            elif i == 1:                                 # one centre, three extents
                lists.append((np.repeat(p[None], 3, 0), [(1.5, 0.8), unit, (0.6, 0.3)]))
            elif i == 2:                                 # floor(dist) 0 twice: the farther one comes first
                lists.append((p + np.array([[0.7, 0.0], [0.2, 0.0]]), unit))
            else:
                lists.append((p[None] + rng.normal(0, 0.02, (1, 2)), unit))
        lists.append((np.repeat(dup_site, 2, 0), unit))  # duplicates alone: two tracks spawn on one spot
        if f < 4:
            lists.append((nan_site, (0.0, 0.0)))         # zero area
        frames.append(np.concatenate([boxes_at(c, h) for c, h in lists]))
    run = _Lockstep(ref, lm)
    run.reset()
    nan_spawned = nan_killed = dup_shared = 0
    for f, b in enumerate(frames):
        pre, a, da, _ = run.step(b, (f + 1) * STEP_US)
        nan_spawned += int(np.isnan(a["targets"][:, 0]).any())
        nan_killed = int((np.isnan(da[:, D_X]) & (da[:, 0] == 0)).sum())
        rows = np.nonzero(pre[:, 0] > 0)[0]
        if f >= 6 and len(rows):
            g = gate_nis(da, b, rows) < GAMMA_G
            d0 = len(b) - (3 if f - 6 < 4 else 2)        # the duplicate pair
            dup_shared = max(dup_shared, int((g[:, d0] & g[:, d0 + 1]).sum()))
    assert nan_spawned >= 4 and nan_killed >= 3, (nan_spawned, nan_killed)
    assert dup_shared >= 2, dup_shared
    print(f"degenerate lists: regime reached: steps with a NaN track {nan_spawned}, NaN tracks killed {nan_killed}, tracks gating "
          f"both duplicates {dup_shared}; worst relative state error {run.worst:.3g}")
