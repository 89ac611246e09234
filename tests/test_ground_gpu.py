"""GPU parity: lmot_ground_remove vs the reference's groundRemove (oracle/_ref, unmodified sources).

Bar (BASELINE.json north_star): BIT-EXACT polar cell per point, ground/elevated label per point, and the
order-preserving output clouds.  The 80x120 grid stages are compared bit-for-bit too.
"""
import numpy as np
import pytest

from oracle.ref import labels_from_clouds

pytestmark = pytest.mark.gpu


def _check_frame(lm, ref, pts):
    out = lm.ground_remove(pts)
    e_ref, g_ref = ref.ground_remove(pts)
    assert out["elevated"].shape[0] == e_ref.shape[0]
    assert out["ground"].shape[0] == g_ref.shape[0]
    assert np.array_equal(out["elevated"][:, :3].view(np.uint32), e_ref.view(np.uint32))
    assert np.array_equal(out["ground"][:, :3].view(np.uint32), g_ref.view(np.uint32))
    if len(out["elevated"]):
        assert np.all(out["elevated"][:, 3] == 1.0)
    lab_ref = labels_from_clouds(pts, e_ref, g_ref)
    assert np.array_equal(out["labels"], lab_ref)
    # point -> polar cell, bit exact (reference getCellIndexFromPoints on the range-filtered points)
    n = len(pts)
    ch, b = lm.debug_cell_index(n)
    ch_r, b_r = ref.cell_index(pts)
    d = np.hypot(pts[:, 0].astype(np.float32), pts[:, 1].astype(np.float32))
    kept = ch >= 0
    assert np.array_equal(ch[kept], ch_r[kept]) and np.array_equal(b[kept], b_r[kept])
    # points the GPU dropped are exactly those the reference filters or cannot index
    dropped_ref = (lab_ref == 0)
    assert np.array_equal(~kept, dropped_ref)
    # grid stages
    g_gpu, g_r = lm.debug_polar_grid(), ref.polar_grid(pts)
    for k in ("minz", "height", "smoothed", "hdiff"):
        assert np.array_equal(g_gpu[k].view(np.uint32), g_r[k].view(np.uint32)), k
    assert np.array_equal(g_gpu["isground"], g_r["isground"])
    gm = g_r["isground"].astype(bool)
    assert np.array_equal(g_gpu["hground"][gm].view(np.uint32), g_r["hground"][gm].view(np.uint32))
    return out


def test_hdl64_frames_bit_exact(lm, ref_intended, synth):
    cfg = synth.SceneConfig(seed=3)
    for ts, pts in synth.frames(cfg, 4):
        out = _check_frame(lm, ref_intended, pts)
        assert len(out["elevated"]) > 10000 and len(out["ground"]) > 10000


def test_uniform_random_clouds_bit_exact(lm, ref_intended, synth):
    for seed, n in ((1, 120000), (2, 50001), (3, 1000)):
        _check_frame(lm, ref_intended, synth.uniform_cloud(n, seed))


def test_grid_filters_stress(lm, ref_intended):
    """Sparse clouds around the thresholds exercise applyMedianFilter / outlierFilter (tHmin runs of 1-2 cells)."""
    rng = np.random.default_rng(7)
    for it in range(6):
        n = 40000
        r = rng.uniform(3.5, 119.0, n).astype(np.float32)
        a = rng.uniform(-np.pi, np.pi, n).astype(np.float32)
        z = rng.choice(np.array([-2.5, -2.0, -1.9, -1.7, -1.5, -0.41, -0.4, -0.39, 0.5], np.float32), n)
        z = (z + rng.normal(0, 0.02, n) * (rng.random(n) < 0.5)).astype(np.float32)
        pts = np.stack([r * np.cos(a), r * np.sin(a), z, np.zeros(n, np.float32)], 1).astype(np.float32)
        _check_frame(lm, ref_intended, pts)


def test_edge_cases(lm, ref_intended):
    # empty cloud
    out = lm.ground_remove(np.zeros((0, 4), np.float32))
    assert len(out["elevated"]) == 0 and len(out["ground"]) == 0
    # single point, points on the range limits, atan2 == +pi (chI == 80 -> dropped), zeros
    pts = np.array([[10, 0, -1.7, 0], [-10, 0.0, -1.7, 0], [-10, -0.0, -1.7, 0], [3.4, 0, -1.7, 0], [0, 120, 0, 0],
                    [0, 0, 0, 0], [3.4000001, 0, -1.7, 0], [0, -119.99999, -1.0, 0], [1e-20, -5, -1.8, 0]], np.float32)
    _check_frame(lm, ref_intended, pts)
    # stride 3 input gives the same answer as stride 4
    cloud = np.random.default_rng(5).uniform(-30, 30, (5000, 3)).astype(np.float32)
    cloud[:, 2] = np.random.default_rng(6).uniform(-2.5, 1, 5000)
    a = lm.ground_remove(cloud)
    b = lm.ground_remove(np.concatenate([cloud, np.ones((5000, 1), np.float32)], 1))
    assert np.array_equal(a["labels"], b["labels"])
    e_ref, g_ref = ref_intended.ground_remove(cloud)
    assert np.array_equal(a["elevated"][:, :3], e_ref)


def test_non_finite_points(lm, ref_intended, synth):
    """NaN / Inf coordinates as the reference treats them: a non-finite x or y never passes the range filter; a NaN z never wins
    `z < minZ` and is never `< hGround + 0.25` (elevated); +Inf z is elevated, -Inf z becomes its cell's minimum."""
    nan, inf = np.nan, np.inf
    pts = synth.uniform_cloud(6000, 21).copy()
    special = np.array([[nan, 1, -1.7, 0], [5, nan, -1.7, 0], [5, 5, nan, 0], [inf, 0, -1.7, 0], [5, -inf, -1.7, 0], [6, 6, inf, 0],
                        [6, 6, -inf, 0], [-inf, inf, nan, 0], [nan, nan, nan, 0], [7, 7, -1.7, 0]], np.float32)
    for k, row in enumerate(special):
        pts[37 + 599 * k] = row
    out = lm.ground_remove(pts)
    e_ref, g_ref = ref_intended.ground_remove(pts)
    assert np.array_equal(out["elevated"][:, :3].view(np.uint32), e_ref.view(np.uint32))
    assert np.array_equal(out["ground"][:, :3].view(np.uint32), g_ref.view(np.uint32))
    g_gpu, g_r = lm.debug_polar_grid(), ref_intended.polar_grid(pts)
    for k in ("minz", "height", "smoothed", "hdiff"):
        assert np.array_equal(g_gpu[k].view(np.uint32), g_r[k].view(np.uint32)), k
    assert np.array_equal(g_gpu["isground"], g_r["isground"])


def test_repeatable_and_stateless(lm, synth):
    pts = synth.uniform_cloud(30000, 11)
    a = lm.ground_remove(pts)
    lm.ground_remove(synth.uniform_cloud(1000, 12))
    b = lm.ground_remove(pts)
    assert np.array_equal(a["labels"], b["labels"]) and np.array_equal(a["elevated"], b["elevated"])


def test_chained_device_launches_leave_the_last_frames_grid(lm, ref_intended, synth):
    """lmot_ground_remove_dev back to back on one stream (what bench.py times for roofline_dense_1m): consecutive launches are chained
    as programmatic dependents, the next launch's CTAs are resident and set up while the previous one drains.  They share the slot's
    two key grids (one re-armed by the launch before), barrier counters and count descriptors: after a chain over different clouds
    the polar grid of the LAST cloud must be the reference's, bit for bit, and the next ordinary call must be exact too."""
    import torch
    clouds = [synth.uniform_cloud(200000 + 1000 * i, 50 + i) for i in range(6)]
    dev = [torch.from_numpy(c).cuda() for c in clouds]
    torch.cuda.synchronize()
    for rep in range(4):
        for d, c in zip(dev, clouds):
            lm.ground_remove_dev(d.data_ptr(), len(c))
    lm.sync()
    g_gpu, g_r = lm.debug_polar_grid(), ref_intended.polar_grid(clouds[-1])
    for k in ("minz", "height", "smoothed", "hdiff"):
        assert np.array_equal(g_gpu[k].view(np.uint32), g_r[k].view(np.uint32)), k
    assert np.array_equal(g_gpu["isground"], g_r["isground"])
    out = lm.ground_remove(clouds[0])
    e, g = ref_intended.ground_remove(clouds[0])
    assert np.array_equal(out["elevated"][:, :3].view(np.uint32), e.view(np.uint32))
    assert np.array_equal(out["ground"][:, :3].view(np.uint32), g.view(np.uint32))


def test_channel_boundaries_fast_and_exact_paths_agree(lm, ref_intended):
    """polar_bin_kernel takes a guarded fast path for the channel index (ground.cu, kChanGuard) and the exact fdlibm
    restatement near channel boundaries: clouds that hug the 80 boundaries from both sides, from 1e-7 rad to 1e-3 rad,
    must land in the reference's cells bit for bit."""
    rng = np.random.default_rng(42)
    n_per = 600
    pts = []
    for c in range(81):
        theta0 = -np.pi + c * (2 * np.pi / 80)
        off = np.concatenate([rng.uniform(-1e-3, 1e-3, n_per // 3), rng.uniform(-2e-5, 2e-5, n_per // 3), rng.uniform(-4e-7, 4e-7, n_per // 3)])
        th = theta0 + off
        r = rng.uniform(3.5, 119.0, len(th))
        z = rng.uniform(-2.2, 0.5, len(th))
        pts.append(np.stack([r * np.cos(th), r * np.sin(th), z, np.zeros_like(z)], 1))
    pts = np.concatenate(pts).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]
    out = lm.ground_remove(pts)
    ch, b = lm.debug_cell_index(len(pts))
    ch_r, b_r = ref_intended.cell_index(pts)
    d = np.hypot(pts[:, 0], pts[:, 1])
    kept = ch >= 0
    assert kept.sum() > 0.9 * len(pts)
    assert np.array_equal(ch[kept], ch_r[kept]) and np.array_equal(b[kept], b_r[kept])
    e_ref, g_ref = ref_intended.ground_remove(pts)
    assert np.array_equal(out["elevated"][:, :3].view(np.uint32), e_ref.view(np.uint32))
    assert np.array_equal(out["ground"][:, :3].view(np.uint32), g_ref.view(np.uint32))


def _ctx_with(pkg_mod, pts_per_cta, max_points=None):
    import os
    old = os.environ.get("LMOT_PTS_PER_CTA")
    os.environ["LMOT_PTS_PER_CTA"] = str(pts_per_cta)
    try:
        p = pkg_mod.default_params()
        if max_points:
            p.max_points = max_points
        p.pipeline_depth = 1
        return pkg_mod.Lmot(p, device=0)
    finally:
        if old is None:
            del os.environ["LMOT_PTS_PER_CTA"]
        else:
            os.environ["LMOT_PTS_PER_CTA"] = old


def test_fused_kernel_chunkings_bit_exact(pkg, ref_intended, synth):
    """ground_fused_kernel splits the frame into per-CTA chunks of 16 KB tiles: the result must not depend on the split.
    256 points per CTA = every SM gets a partial tile; 16384 = the minimum of 8 CTAs with multi-tile chunks."""
    pts = synth.uniform_cloud(120000, 21)
    for ppc in (256, 1000, 16384):
        ctx = _ctx_with(pkg, ppc)
        try:
            _check_frame(ctx, ref_intended, pts)
            _check_frame(ctx, ref_intended, pts[:777])
        finally:
            ctx.close()


def test_fused_kernel_tiles_beyond_shared_memory_bit_exact(pkg, ref_intended, synth):
    """Chunks longer than the 8 shared-memory-resident tiles (frames > ~1.08 M points on 132 SMs) re-read their tail from
    global memory in the classification phase: 1.6 M points, bit-exact against the reference."""
    pts = synth.uniform_cloud(1_600_000, 22)
    ctx = _ctx_with(pkg, 16384, max_points=1_600_000)
    try:
        out = ctx.ground_remove(pts)
        e_ref, g_ref = ref_intended.ground_remove(pts)
        assert np.array_equal(out["elevated"][:, :3].view(np.uint32), e_ref.view(np.uint32))
        assert np.array_equal(out["ground"][:, :3].view(np.uint32), g_ref.view(np.uint32))
        assert np.array_equal(out["labels"], labels_from_clouds(pts, e_ref, g_ref))
    finally:
        ctx.close()


def test_node_prefilter_matches_filter_then_ground_remove(pkg, ref_intended, synth):
    """SURVEY.md §8(f)2: the `ground` ROS node runs pcl::PassThrough (z in [-3, 1], inclusive, non-finite removed) and
    pcl::ConditionalRemoval (x in (-15, 5), y in (-50, 50), strict) in front of groundRemove
    (/root/reference/object_tracking/src/groundremove/main.cpp:56-89,104-112).  With node_prefilter on, the fused kernel must give
    what groundRemove gives on the pre-filtered cloud, and label 3 / 1 / 2 must mark exactly the node's aux_points cloud."""
    p = pkg.default_params()
    p.node_prefilter = 1
    p.pipeline_depth = 1
    ctx = pkg.Lmot(p, device=0)
    try:
        for seed in (4, 5):
            pts = next(iter(synth.frames(synth.SceneConfig(seed=seed), 1)))[1].copy()
            rng = np.random.default_rng(seed)
            # points exactly on the limits, and a few non-finite ones
            pts[:6, :3] = [[-15.0, 0, -1.7], [5.0, 0, -1.7], [1, -50.0, -1.7], [1, 50.0, -1.7], [1, 1, -3.0], [1, 8, 1.0]]
            pts[6, 0] = np.nan; pts[7, 2] = np.inf; pts[8, 1] = -np.inf
            x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
            with np.errstate(invalid="ignore"):
                keep = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & (z >= -3.0) & (z <= 1.0) & (x > -15) & (x < 5) & (y > -50) & (y < 50)
            aux = pts[keep]
            e_ref, g_ref = ref_intended.ground_remove(aux)
            out = ctx.ground_remove(pts)
            assert np.array_equal(out["elevated"][:, :3].view(np.uint32), e_ref.view(np.uint32))
            assert np.array_equal(out["ground"][:, :3].view(np.uint32), g_ref.view(np.uint32))
            assert np.array_equal(out["labels"] != 0, keep)
            lab_aux = labels_from_clouds(aux, e_ref, g_ref)
            assert np.array_equal(out["labels"][keep] % 3, lab_aux)      # 3 = aux point in neither output
            assert keep[4] and keep[5] and not keep[:4].any() and not keep[6:9].any()
    finally:
        ctx.close()
