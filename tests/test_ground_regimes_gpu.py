"""GPU parity of ground removal in every regime where ground_fused_kernel switches paths, and at its label and cell ties.

The regimes are ground_scenes.py's (launch geometry restated there from the device's SM count, scenes and witnesses checked without a
GPU in test_ground_regimes_cpu.py): the exact-evaluation queue below, at and above its 2,048 points per CTA, with in-range points
evaluated inline; chunks on both sides of 2,048 (label limits gathered / staged), 1 to 16 tiles with resident and global tiles, the
largest frame a launch covers; phase 2's channel split for many CTA counts with filter rewrites in each CTA's first and last own
channel; label limits on their tie under tolerances 0.25 / 0.3 / 0.1, a zero threshold and positive ground heights; the half-SM cap
of the frame pipeline; ragged rig batches and sequence ticks with their own values; the node pre-filter; PDL chains across regimes.

Bars: the stage entry point (lmot_ground_remove) -- clouds and labels bit-exact, the fused kernel's isground / hground and the
inspection grids bit-exact; the frame, batch and sequence paths -- n_elevated, n_ground, num_cluster and boxes bit-exact against the
reference's groundRemove -> componentClustering -> boxFitting.  The checkerboard probes are one-sided (a wrong cell turns an elevated
point into ground or drops it) and the tie probes straddle the limit, so the counts alone see a wrong cell or limit.
"""
import contextlib
import os

import numpy as np
import pytest

import ground_scenes as S
from oracle.ref import labels_from_clouds

pytestmark = pytest.mark.gpu
MB = 8192


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _params(pkg, max_points=None, **kw):
    p = pkg.default_params()
    p.pipeline_depth = 1
    p.max_boxes = MB
    p.max_clusters = 50000
    if max_points:
        p.max_points = max_points
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@contextlib.contextmanager
def _ctx(pkg, ppc=None, max_points=None, **kw):
    """a context whose stage launches aim at ppc points per CTA (LMOT_PTS_PER_CTA, read at creation)"""
    old = os.environ.get("LMOT_PTS_PER_CTA")
    if ppc:
        os.environ["LMOT_PTS_PER_CTA"] = str(ppc)
    try:
        ctx = pkg.Lmot(_params(pkg, max_points, **kw), device=0)
    finally:
        if old is None:
            os.environ.pop("LMOT_PTS_PER_CTA", None)
        else:
            os.environ["LMOT_PTS_PER_CTA"] = old
    try:
        yield ctx
    finally:
        ctx.close()


@pytest.fixture(scope="module")
def ref(ref_intended):
    return ref_intended


@pytest.fixture(scope="module")
def ref_dt():
    from oracle import ref_detect_tunable
    if not ref_detect_tunable.have_ref("detect_tunable"):
        pytest.skip("oracle/_ref/libref_detect_tunable.so not built")
    return ref_detect_tunable.RefDetectTunable()


@pytest.fixture(scope="module")
def pool(ref):
    return S.checker_probe_pool(ref.cell_index, n=24000, seed=1)


@pytest.fixture(scope="module")
def floor():
    return S.full_floor(S.checker_heights())


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check_stage(ctx, ref, pts, grids=True):
    """lmot_ground_remove against the reference: clouds bit-exact, labels (every label-2 / label-1 point, in order, is the reference's
    elevated / ground cloud), the fused kernel's isground / hground and the inspection grids bit-exact"""
    out = ctx.ground_remove(pts)
    e_ref, g_ref = ref.ground_remove(pts)
    assert np.array_equal(_u32(out["elevated"][:, :3]), _u32(e_ref)) and np.array_equal(_u32(out["ground"][:, :3]), _u32(g_ref))
    lab = out["labels"]
    p = np.ascontiguousarray(pts[:, :3], np.float32)
    assert np.array_equal(_u32(p[lab == 2]), _u32(e_ref)) and np.array_equal(_u32(p[lab == 1]), _u32(g_ref))
    assert int((lab == 0).sum()) == len(p) - len(e_ref) - len(g_ref)
    if grids:
        g_gpu, g_r = ctx.debug_polar_grid(), ref.polar_grid(pts)
        for k in ("minz", "height", "smoothed", "hdiff"):
            assert np.array_equal(_u32(g_gpu[k]), _u32(g_r[k])), k
        assert np.array_equal(g_gpu["isground"], g_r["isground"])
        gm = g_r["isground"].astype(bool)
        assert np.array_equal(_u32(g_gpu["hground"][gm]), _u32(g_r["hground"][gm]))
    return out, e_ref, g_ref


def _ref_pipeline(ref, pts):
    e, g = ref.ground_remove(pts)
    grid, k = ref.component_clustering(e)
    b, _ = ref.box_fitting(e, grid, k, MB)
    return (len(e), len(g), k), b


def _got(r):
    return (int(r["n_elevated"]), int(r["n_ground"]), int(r["num_cluster"]))


# ------------------------------------------------------------------------------------------------ queue and size switches (stage)
def _queue_regimes(sms):
    """name -> (n, pts_per_cta, queued points per CTA)"""
    return {
        "T=4 queue 1500 / 2048 / 2049 / 4096": (8 * 4096, 4096, [1500, 2048, 2049, 4096] * 2),
        "chunk 2048 all queued (gathered limits)": (16 * 2048, 2048, [2048] * 8 + [0] * 8),
        "chunk 2049 all queued (staged limits)": (16 * 2049, 2049, [2049] * 8 + [0] * 8),
        "T=9 global tiles, queue 2100 / 9000": (8 * 9000 - 700, 9000, [2100, 9000] * 4),
        "T=16 at 8 CTAs, queue 2049 / 16384": (8 * 16384, 16384, [2049, 16384] * 4),
    }


@pytest.mark.parametrize("regime", sorted(_queue_regimes(132)))
def test_queue_regimes_stage(pkg, ref, pool, floor, regime):
    sms = _sms()
    n, ppc, q = _queue_regimes(sms)[regime]
    geo = S.launch([n], sms, ppc=ppc)
    pts = S.layout(geo, q, pool, floor, seed=5)
    per = S.queued_per_cta(pts, geo)[:, 0]
    print(f"{regime}: {S.describe(geo)} queued per CTA {sorted(set(per.tolist()))}")
    assert per.max() >= S.PEND_CAP and len(pts) - per.sum() >= S.NUM_CHANNEL * S.NUM_BIN
    with _ctx(pkg, ppc) as ctx:
        out, e, g = _check_stage(ctx, ref, pts)
    assert np.all(out["labels"][S.certainly_queued(pts)] == 2)        # one-sided: every probe elevated


SIZE_REGIMES = {      # name -> (n, pts_per_cta, expected tiles per CTA)
    "T=1 cnt 1024": (16 * 1024, 1024, {1}),
    "T=2 chunk 2000": (8 * 2000, 2000, {2}),
    "T=3 odd tail, last CTA partial": (8 * 2500 - 300, 2500, {3}),
    "T=8 all resident": (8 * 8192, 8192, {8}),
    "T=9 one global tile, last CTA partial": (8 * 8700 - 5, 8700, {9}),
    "ppc 256 partial tiles": (40000, 256, {1}),
}


@pytest.mark.parametrize("regime", sorted(SIZE_REGIMES))
def test_size_switches_stage(pkg, ref, pool, floor, regime):
    sms = _sms()
    n, ppc, Ts = SIZE_REGIMES[regime]
    geo = S.launch([n], sms, ppc=ppc)
    f = geo["frames"][0]
    q = [min(c["cnt"] // 2, 2100 if i % 2 == 0 else 300) for i, c in enumerate(f["ctas"])]
    pts = S.layout(geo, q, pool, floor, seed=6)
    covered = len(pts) - sum(q) >= S.NUM_CHANNEL * S.NUM_BIN      # every cell has its floor: the probes are one-sided
    print(f"{regime}: {S.describe(geo)} full pairs {sorted({c['full_pairs'] for c in f['ctas']})} last cnt {f['ctas'][-1]['cnt']}")
    assert {c["T"] for c in f["ctas"]} == Ts
    with _ctx(pkg, ppc) as ctx:
        out, _, _ = _check_stage(ctx, ref, pts)
    assert not covered or np.all(out["labels"][S.certainly_queued(pts)] == 2)


def test_largest_frame_sixteen_tiles_on_every_sm(pkg, ref, pool, floor):
    """n = SMs x 16,384, the most one launch covers: T = 16 in every CTA (labels in bits 30-31, a queued index up to 16,383), 4,000
    queued points per CTA"""
    sms = _sms()
    n = sms * 16384
    geo = S.launch([n], sms, ppc=16384)
    assert geo["G"] == sms and not geo["capacity"]
    pts = S.layout(geo, [4000] * sms, pool, floor, seed=7)
    # the last point of every chunk certainly queued: the highest queued index
    for c in geo["frames"][0]["ctas"]:
        pts[c["beg"] + c["cnt"] - 1] = pool[c["beg"] % len(pool)]
    print(f"largest frame: n={n} {S.describe(geo)}")
    with _ctx(pkg, 16384, max_points=n) as ctx:
        out, _, _ = _check_stage(ctx, ref, pts, grids=False)
        assert np.all(out["labels"][S.certainly_queued(pts)] == 2)
        with pytest.raises(pkg.LmotError) as err:
            ctx.ground_remove(np.concatenate([pts, pts[:1]]))
        assert err.value.status == pkg.ERR_CAPACITY


# ------------------------------------------------------------------------------------------------ phase 2 channel split
@pytest.mark.parametrize("which", ["8", "9", "13", "33", "SMs/2", "79", "80", "81", "SMs"])
def test_channel_split_with_seam_filters(pkg, ref, which):
    sms = _sms()
    G = {"SMs/2": sms // 2, "SMs": sms}.get(which) or int(which)
    base, marks = S.seam_scene(min(G, S.NUM_CHANNEL))
    reps = max(1, -(-300 * G // len(base)))
    pts = np.tile(base, (reps, 1))                       # duplicates leave every cell minimum as it is
    ppc = S.ppc_for(G, len(pts))
    geo = S.launch([len(pts)], sms, ppc=ppc)
    print(f"G={G}: {S.describe(geo)} seam cells {len(marks)} own channels {geo['own'][:3]}...{geo['own'][-2:]}")
    assert geo["G"] == G
    with _ctx(pkg, ppc) as ctx:
        out, _, _ = _check_stage(ctx, ref, pts)
        g = ctx.debug_polar_grid()
    for _, ch, b in marks:
        assert g["isground"][ch, b]


# ------------------------------------------------------------------------------------------------ label limits
TIE_CASES = {
    "tol0.25": (dict(), dict(centre=-1.6)),
    "tol0.3": (dict(ground_tolerance=0.3), dict(centre=-1.6)),
    "tol0.1": (dict(ground_tolerance=0.1), dict(centre=-1.6)),
    "thr0": (dict(t_hmax=-0.1), dict(centre=-0.3, amp=0.05, exact=(-0.25, 0.3))),
    "h>0": (dict(t_hmin=-0.8, t_hmax=0.8, h_sensor=0.8), dict(centre=0.3)),
}


def _tie_scene(ref_dt, values, hk, zero):
    base = S.full_floor(S.smooth_heights(**hk))
    with ref_dt.detect_params(values):
        g0 = ref_dt.polar_grid(base)
    probes, want = S.tie_probes(g0["hground"], g0["isground"], values.get("ground_tolerance", 0.25), zero)
    return np.concatenate([base, probes]), want


@pytest.mark.parametrize("case", sorted(TIE_CASES))
def test_label_limit_ties_stage(pkg, ref_dt, case):
    """context values vs the reference with the same globals; gathered limits (default chunking) and staged ones (4,096 per CTA)"""
    values, hk = TIE_CASES[case]
    pts, want = _tie_scene(ref_dt, values, hk, case == "thr0")
    for ppc in (None, 4096):
        geo = S.launch([len(pts)], _sms(), ppc=ppc or S.DEFAULT_PPC)
        with _ctx(pkg, ppc, **values) as ctx, ref_dt.detect_params(values):
            out, _, _ = _check_stage(ctx, ref_dt, pts)
        lab = out["labels"][len(pts) - len(want):]
        print(f"{case} ({S.describe(geo)}): {len(want)} tie probes, {int((want == 1).sum())} ground")
        assert np.array_equal(lab, want)


def test_label_limit_ties_on_filter_rewrites(pkg, ref):
    """limits of cells whose height the median / outlier filters rewrote"""
    base, marks = S.seam_scene(8)
    g0 = ref.polar_grid(base)
    probes, want = S.tie_probes(g0["hground"], g0["isground"], 0.25, minz=g0["minz"])
    pts = np.concatenate([base, probes])
    with _ctx(pkg) as ctx:
        out, _, _ = _check_stage(ctx, ref, pts)
    assert np.array_equal(out["labels"][len(base):], want)
    print(f"filter rewrites: {len(marks)} rewritten cells, {len(want)} tie probes")


# ------------------------------------------------------------------------------------------------ frame pipeline
@pytest.mark.parametrize("side", ["cap on", "cap off"])
def test_half_sm_cap_frame(pkg, ref, pool, floor, side):
    sms = _sms()
    n = max(sms // 2, 8) * 8192 + (side == "cap off")
    geo = S.launch([n], sms, entry="frame")
    q = [min(c["cnt"], 2500) for c in geo["frames"][0]["ctas"]]
    pts = S.layout(geo, q, pool, floor, seed=8)
    print(f"half-SM cap {side}: n={n} {S.describe(geo)}")
    assert geo["half"] == (side == "cap on")
    want, b = _ref_pipeline(ref, pts)
    with _ctx(pkg) as ctx:
        r = ctx.frame(pts, 1e6)
    assert _got(r) == want and np.array_equal(_u32(r["boxes"]), _u32(b))
    assert want[0] >= int(S.certainly_queued(pts).sum())


def test_organized_frame_with_missing_returns(pkg, ref):
    """128 x 2048 ring-major frame with rows of (0, 0, 0) / NaN returns beside rows of in-range boundary probes, through lmot_frame and
    lmot_ground_remove"""
    pts = S.organized(ref.cell_index)
    geo = S.launch([len(pts)], _sms(), entry="frame")
    per = S.queued_per_cta(pts, geo)[:, 0]
    print(f"organized: {S.describe(geo)} queued per CTA max {per.max()}, {(per > S.PEND_CAP).sum()} CTAs over the cap")
    assert per.max() > S.PEND_CAP
    want, b = _ref_pipeline(ref, pts)
    with _ctx(pkg) as ctx:
        r = ctx.frame(pts, 1e6)
        assert _got(r) == want and np.array_equal(_u32(r["boxes"]), _u32(b))
        _check_stage(ctx, ref, pts, grids=False)


# ------------------------------------------------------------------------------------------------ rig batch and sequence ticks
def _ragged_frames(sms, F, pool, floor, first, shift_pool=None):
    """[first, empty, 9 points, a 16-tile frame with every chunk overflowing the queue] under F frames per launch"""
    G = sms // F
    big_n = G * 16384
    geo = S.launch([len(first), 0, 9, big_n], sms, entry="batch")
    assert geo["G"] == G and geo["frames"][3]["chunk"] == 16384
    big = S.layout(S.launch([big_n], G, ppc=16384), [2100] * G, shift_pool if shift_pool is not None else pool, floor, seed=9)
    nine = np.concatenate([floor[:5], pool[:4]])
    return [first, np.zeros((0, 3), np.float32), nine, big], geo


def test_ragged_rig_batch(pkg, ref, ref_dt, pool, floor):
    """lmot_batch with a 4-sensor rig (ground_fused_rig_kernel): a tie frame of a 0.8 m mount (positive ground heights), an empty
    frame, a 9-point frame, a 16-tile overflowing frame; each against the reference with its sensor's globals (ref_mount)"""
    from test_sensor_rig_gpu import ref_mount, set_rig, yaw_pose
    sms = _sms()
    tie, want_tie = _tie_scene(ref_dt, TIE_CASES["h>0"][0], TIE_CASES["h>0"][1], False)
    frames, geo = _ragged_frames(sms, 4, pool, floor, tie)
    heights = [0.8, 2.0, 1.2, 2.0]
    rig = [(yaw_pose(1, 0, 0.0, 0.0, 0.0), h) for h in heights]
    print(f"rig batch: G={geo['G']} chunks {geo['chunks']} smem {geo['smem']}")
    want, boxes = [], []
    for fr, h in zip(frames, heights):
        with ref_mount(ref, h):
            w, b = _ref_pipeline(ref, fr)
        want.append(w); boxes.append(b)
    with _ctx(pkg) as ctx:
        set_rig(ctx, rig)
        r = ctx.batch(frames, 1e6)
    got = list(zip(r["n_elevated"], r["n_ground"], r["num_cluster"]))
    print(f"rig batch (n_elev, n_ground, K): {want}")
    assert [tuple(map(int, g)) for g in got] == want
    assert np.array_equal(_u32(r["boxes"]), _u32(np.concatenate(boxes)))
    assert want[0][1] == int((want_tie == 1).sum()) + S.NUM_CHANNEL * S.NUM_BIN


def test_ragged_sequence_tick_with_own_values(pkg, ref_dt, pool, floor):
    """lmot_seq with every sequence's own detection values (ground_fused_frame_kernel, its own copy of the exact evaluation): tolerance
    0.3 on a tie frame, an empty and a 9-point frame, tolerance 0.1 on a 16-tile overflowing frame"""
    sms = _sms()
    tie, want_tie = _tie_scene(ref_dt, TIE_CASES["tol0.3"][0], TIE_CASES["tol0.3"][1], False)
    frames, geo = _ragged_frames(sms, 4, pool, floor, tie)
    values = [dict(ground_tolerance=0.3), dict(ground_tolerance=0.2), dict(t_hmax=-0.3), dict(ground_tolerance=0.1)]
    want, boxes = [], []
    for fr, v in zip(frames, values):
        with ref_dt.detect_params(v):
            w, b = _ref_pipeline(ref_dt, fr)
        want.append(w); boxes.append(b)
    with _ctx(pkg) as ctx:
        ctx.seq_open(4, ring=2)
        for k, v in enumerate(values):
            ctx.seq_set_detect_params(k, **v)
        out = ctx.seq(frames, [1e6] * 4)
    print(f"sequence tick G={geo['G']} (n_elev, n_ground, K): {want}")
    for k in range(4):
        assert _got(out[k]) == want[k], k
        assert np.array_equal(_u32(out[k]["boxes"]), _u32(boxes[k])), k
    assert want[0][1] == int((want_tie == 1).sum()) + S.NUM_CHANNEL * S.NUM_BIN


# ------------------------------------------------------------------------------------------------ node pre-filter
def test_node_prefilter_global_tiles_and_overflow(pkg, ref):
    """pre-filter on (no full-pair fast loop), 12 tiles per chunk (4 re-read from global memory), 2,100+ queued in-window probes"""
    inside = lambda x, y: (x > -15) & (x < 5) & (y > -50) & (y < 50)
    wpool = S.checker_probe_pool(ref.cell_index, n=1500, seed=11, window=inside)
    floor = S.full_floor(S.checker_heights())
    n, ppc = 8 * 12000, 12000
    geo = S.launch([n], _sms(), ppc=ppc, prefilter=True)
    pts = S.layout(geo, [2100, 3000] * 4, wpool, floor, seed=12)
    pts[5, 2] = np.nan; pts[17, 0] = np.inf
    print(f"pre-filter: {S.describe(geo)} full pairs {geo['frames'][0]['ctas'][0]['full_pairs']}")
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    with np.errstate(invalid="ignore"):
        keep = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & (z >= -3.0) & (z <= 1.0) & inside(x, y)
    aux = pts[keep]
    e_ref, g_ref = ref.ground_remove(aux)
    with _ctx(pkg, ppc, node_prefilter=1) as ctx:
        out = ctx.ground_remove(pts)
    assert np.array_equal(_u32(out["elevated"][:, :3]), _u32(e_ref)) and np.array_equal(_u32(out["ground"][:, :3]), _u32(g_ref))
    assert np.array_equal(out["labels"] != 0, keep)
    assert np.array_equal(out["labels"][keep] % 3, labels_from_clouds(aux, e_ref, g_ref))


# ------------------------------------------------------------------------------------------------ PDL chains
def test_chain_across_regimes(pkg, ref, pool, floor):
    """lmot_ground_remove_dev back to back over frames in different regimes (CTA count, tiles, shared memory, label-limit path): with
    each frame in turn last, the polar grid is the last frame's; then an ordinary call is exact"""
    import torch
    sms = _sms()
    sizes = [5000, 200000, 600000, sms * 8192 + 5000, 40000]
    clouds = []
    for i, n in enumerate(sizes):
        geo = S.launch([n], sms)
        q = [min(c["cnt"] // 2, 2100) for c in geo["frames"][0]["ctas"]]
        clouds.append(S.layout(geo, q, pool, floor, seed=20 + i))
        print(f"chain frame {i}: n={n} {S.describe(geo)}")
    grids = [ref.polar_grid(c) for c in clouds]
    with _ctx(pkg, max_points=max(sizes)) as ctx:
        dev = [torch.from_numpy(np.concatenate([c, np.ones((len(c), 1), np.float32)], 1)).cuda() for c in clouds]
        torch.cuda.synchronize()
        for last in range(len(clouds)):
            order = [(last + 1 + j) % len(clouds) for j in range(len(clouds))]
            for j in order:
                ctx.ground_remove_dev(dev[j].data_ptr(), len(clouds[j]))
            ctx.sync()
            g = ctx.debug_polar_grid()
            for k in ("minz", "height", "smoothed", "hdiff"):
                assert np.array_equal(_u32(g[k]), _u32(grids[last][k])), (last, k)
            assert np.array_equal(g["isground"], grids[last]["isground"]), last
        _check_stage(ctx, ref, clouds[1], grids=True)


# ------------------------------------------------------------------------------------------------ launch geometry on the device
_GEOM_SCRIPT = r"""
import importlib, json, os, sys, tempfile
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
import ground_scenes as S
sms = torch.cuda.get_device_properties(0).multi_processor_count
rng = np.random.default_rng(0)
def cloud(n):
    p = rng.uniform(-60, 60, (n, 3)).astype(np.float32); p[:, 2] = rng.uniform(-2.5, 0.5, n); return p
def ctx(ppc=None, mp=None):
    if ppc: os.environ["LMOT_PTS_PER_CTA"] = str(ppc)
    p = pkg.default_params(); p.pipeline_depth = 1; p.max_boxes = 8192; p.max_clusters = 50000
    if mp: p.max_points = mp
    c = pkg.Lmot(p)
    os.environ.pop("LMOT_PTS_PER_CTA", None)
    return c
def events(fn):
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    path = os.path.join(tempfile.mkdtemp(), "t.json")
    prof.export_chrome_trace(path)
    ev = json.load(open(path))["traceEvents"]
    return [dict(name=e["name"], grid=e.get("args", {}).get("grid"), smem=e.get("args", {}).get("shared memory"))
            for e in ev if e.get("cat") == "kernel" and "ground_fused" in e.get("name", "")]
out = []
for n, ppc in ((8 * 2048, 2048), (8 * 2049, 2049), (8 * 9000, 9000), (40000, 256), (sms * 16384, 16384)):
    c = ctx(ppc, max(n, 1 << 20)); pts = cloud(n)
    out.append(dict(kind="stage", ns=[n], ppc=ppc, ev=events(lambda: c.ground_remove(pts)))); c.close()
half = max(sms // 2, 8) * 8192
for n in (half, half + 1):
    c = ctx(); pts = cloud(n)
    out.append(dict(kind="frame", ns=[n], ppc=768, ev=events(lambda: c.frame(pts, 1e6)))); c.close()
c = ctx(); fr = [cloud(30000), np.zeros((0, 3), np.float32), cloud(9), cloud((sms // 4) * 16384)]
out.append(dict(kind="batch", ns=[len(f) for f in fr], ppc=768, ev=events(lambda: c.batch(fr, 1e6)))); c.close()
print(json.dumps(dict(sms=sms, out=out)))
"""


def test_launch_geometry_on_the_device():
    """the grid and dynamic shared memory of every ground_fused* launch equal ground_scenes.launch (torch.profiler's kernel records, in a
    process of its own); the static part of the shared memory is the same for every launch"""
    import json
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _GEOM_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    sms = res["sms"]
    statics = set()
    for o in res["out"]:
        geo = S.launch(o["ns"], sms, ppc=o["ppc"], entry=o["kind"])
        ev = o["ev"]
        print(f"{o['kind']} {o['ns']}: expected grid {geo['G'] * geo['F']} smem {geo['smem']} | profiler {ev}")
        assert ev, o
        if ev[0]["grid"] is None or ev[0]["smem"] is None:
            pytest.skip("the profiler's kernel records carry no grid / shared memory")
        for e in ev:
            assert list(e["grid"])[:1] == [geo["G"] * geo["F"]], (o["kind"], o["ns"], e)
            statics.add(int(e["smem"]) - geo["smem"])
    print("static shared memory of the kernels:", statics)
    assert len(statics) == 1 and 0 <= statics.pop() < 1024
