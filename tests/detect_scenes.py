"""Scene builders for the detection regime suites (numpy only, no GPU).

Clustering and box fitting pick code paths by data size: lanes per cluster and scan rounds in the segment-offset scan, tiles per
lane, the shared-memory size of the counting sort, clusters per box-fitting CTA, batches of the per-point pass, rounds of the box
compaction, the CCL pair list.  The builders here make elevated clouds that sit on a chosen side of each switch, and the witnesses
at the bottom restate, from the REFERENCE's outputs only, which side a scene reached.

Grid geometry (component_clustering.cpp:43-48, box_fitting.cpp:53-58): roiM = 50, 250 x 250 cells of 0.2 m, cell index
floor(250 * (x + 25) / 50) in float; box fitting pixelises at picScale = 18 px/m (box_fitting.cpp:218-251).
"""
from __future__ import annotations

import numpy as np

ROI = 50.0
NUM_GRID = 250
CELL = ROI / NUM_GRID              # 0.2 m
PIC = 18.0                         # px per m
PITCH = 4                          # seed cells of a lattice are 4 cells apart: 3x3 dilated blocks + one empty row / column
SITES = 62                         # seeds at cells 1, 5, ..., 245 per axis: 62 x 62 = 3,844 components, the most a grid holds
TILE = 1024                        # points per tile of the counting sort (boxfit.cu kTile)
PAIR_CAP = 4096                    # CCL pair list (ccl_device.cuh kPairCap)
Z_KEEP = (-1.0, 0.0)               # box heights maxZ + 2 inside (0.8, 2.6): every cluster passes RULE_GCC13_O2_COMPAT


def cell_centre(i):
    return -ROI / 2 + CELL * (np.asarray(i, np.float64) + 0.5)


def _cells(rng, ix, iy, n, spread=0.07):
    """n points well inside cell (ix, iy): at most `spread` m from its centre (the cell is +-0.1 m)"""
    x = cell_centre(ix) + rng.uniform(-spread, spread, n)
    y = cell_centre(iy) + rng.uniform(-spread, spread, n)
    return x, y


def lattice_sites(K, rng=None, keep=None):
    """K seed cells (ix, iy) of the 62 x 62 lattice, in raster order.  rng: a random subset (else the first K in raster order);
    keep(ix, iy) -> bool mask restricts the candidates (room for other objects, sensor range)."""
    a = np.arange(SITES) * PITCH + 1
    ix, iy = np.meshgrid(a, a, indexing="ij")
    ix, iy = ix.ravel(), iy.ravel()
    if keep is not None:
        m = keep(ix, iy)
        ix, iy = ix[m], iy[m]
    if K > len(ix):
        raise ValueError(f"{K} sites asked, {len(ix)} available")
    sel = np.sort(rng.choice(len(ix), K, replace=False)) if rng is not None else np.arange(K)
    return ix[sel], iy[sel]


def lattice(K, pts_per_cluster, z=Z_KEEP, seed=0, neighbours=0, keep=None, random_sites=True, shuffle=True):
    """Elevated cloud (N, 3) float32 with exactly K components: K seed cells 4 cells apart, each holding pts_per_cluster points
    (an int, or one count >= 2 per cluster) well inside the cell; `neighbours` (0..8) of its 8 neighbour cells get ONE point each,
    so no neighbour becomes a seed and the dilated 3x3 blocks stay separated by an empty row / column.  shuffle: clusters
    interleaved in cloud order (the counting sort's stable ranks then matter)."""
    rng = np.random.default_rng(seed)
    ix, iy = lattice_sites(K, rng if random_sites else None, keep)
    cnt = np.broadcast_to(np.asarray(pts_per_cluster, np.int64), (K,))
    if K and cnt.min() < 2:
        raise ValueError("a seed cell needs two points")
    xs, ys, zs = [], [], []
    for k in range(K):
        x, y = _cells(rng, ix[k], iy[k], int(cnt[k]))
        xs.append(x); ys.append(y)
        top = rng.uniform(z[0] + 0.3 * (z[1] - z[0]), z[1])        # every cluster its own maxZ
        zs.append(rng.uniform(top - 0.3 * (z[1] - z[0]), top, len(x)))
        if neighbours:
            nb = [(dx, dy) for dx in (-1, 0, 1) for dy in (-1, 0, 1) if dx or dy]
            for j in rng.choice(8, neighbours, replace=False):
                x, y = _cells(rng, ix[k] + nb[j][0], iy[k] + nb[j][1], 1, spread=0.05)
                xs.append(x); ys.append(y); zs.append(np.full(1, top - 0.1 * (z[1] - z[0])))
    if not xs:
        return np.zeros((0, 3), np.float32)
    pts = np.stack([np.concatenate(xs), np.concatenate(ys), np.concatenate(zs)], 1).astype(np.float32)
    return pts[rng.permutation(len(pts))] if shuffle else pts


def cells_of(points):
    """(ix, iy) cell of every point inside the ROI (-1 outside), the reference's float arithmetic"""
    p = np.asarray(points, np.float32)
    half, roi, ng = np.float32(ROI / 2), np.float32(ROI), np.float32(NUM_GRID)
    xc, yc = p[:, 0] + half, p[:, 1] + half
    inside = (xc >= 0) & (xc < roi) & (yc >= 0) & (yc < roi)
    with np.errstate(invalid="ignore"):
        xi = np.floor(ng * xc / roi).astype(np.int64)
        yi = np.floor(ng * yc / roi).astype(np.int64)
    xi[~inside] = -1; yi[~inside] = -1
    return xi, yi


def keep_away(points, margin=2):
    """keep(ix, iy) for lattice(): sites whose dilated block stays `margin` cells clear of every cell `points` occupy"""
    xi, yi = cells_of(points)
    occ = np.zeros((NUM_GRID, NUM_GRID), bool)
    ok = xi >= 0
    occ[xi[ok], yi[ok]] = True
    r = 1 + margin
    pad = np.zeros((NUM_GRID + 2 * r, NUM_GRID + 2 * r), bool)
    pad[r:-r, r:-r] = occ
    near = np.zeros_like(occ)
    for dx in range(-r, r + 1):
        for dy in range(-r, r + 1):
            near |= pad[r + dx: r + dx + NUM_GRID, r + dy: r + dy + NUM_GRID]
    return lambda ix, iy: ~near[ix, iy]


# ------------------------------------------------------------------------------------------------ big objects
def _z(rng, n, z=Z_KEEP):
    return rng.uniform(z[0], z[1], n)


def disc(n, centre, radius, seed=0, z=Z_KEEP):
    rng = np.random.default_rng(seed)
    r = radius * np.sqrt(rng.random(n))
    a = rng.random(n) * 2 * np.pi
    return np.stack([centre[0] + r * np.cos(a), centre[1] + r * np.sin(a), _z(rng, n, z)], 1).astype(np.float32)


def rect(n, centre, length, width, yaw=0.0, seed=0, z=Z_KEEP, hollow=False):
    """a filled rectangle, or (hollow) its two sides facing -x / -y: the L an object shows the sensor"""
    rng = np.random.default_rng(seed)
    u = rng.uniform(-0.5, 0.5, (n, 2)) * [length, width]
    if hollow:
        u[: n // 2, 1] = -width / 2
        u[n // 2:, 0] = -length / 2
    c, s = np.cos(yaw), np.sin(yaw)
    x = centre[0] + c * u[:, 0] - s * u[:, 1]
    y = centre[1] + s * u[:, 0] + c * u[:, 1]
    return np.stack([x, y, _z(rng, n, z)], 1).astype(np.float32)


def ring(n, centre=(12.4, 0.0), r_in=11.9, r_out=12.2, seed=0, z=Z_KEEP):
    """a large annulus: a strict pixel hull of well over 100 vertices.  Centred off the origin so that its max-slope point sits at
    |y| < 5 and box fitting takes the minimum-area-rectangle branch."""
    rng = np.random.default_rng(seed)
    r = np.sqrt(rng.uniform(r_in ** 2, r_out ** 2, n))
    a = rng.random(n) * 2 * np.pi
    return np.stack([centre[0] + r * np.cos(a), centre[1] + r * np.sin(a), _z(rng, n, z)], 1).astype(np.float32)


def dense_cells(cells, seed=0, z=Z_KEEP):
    """two points in every cell of `cells` (an iterable of (ix, iy)): a solid block of occupancy"""
    rng = np.random.default_rng(seed)
    c = np.asarray(list(cells), np.int64).reshape(-1, 2)
    c = np.repeat(c, 2, 0)
    x, y = _cells(rng, c[:, 0], c[:, 1], len(c), spread=0.06)
    return np.stack([x, y, _z(rng, len(c), z)], 1).astype(np.float32)


def pair_scene(extra_cells, rows=190, seed=0):
    """CCL pair-list scene: solid rows 0..rows-1 (about 21 pairs per grid row), `extra_cells` seeds of row rows+1 from y = 0 on (one
    more piece edge each), and a lattice of small components in the rows beyond -- pairs tuned across the 4,096-entry list"""
    block = dense_cells([(x, y) for x in range(rows) for y in range(NUM_GRID)] + [(rows + 1, y) for y in range(extra_cells)], seed)
    lat = lattice(200, 30, seed=seed, keep=lambda ix, iy: ix > rows + 4)
    return interleave([block, lat], seed)


# ------------------------------------------------------------------------------------------------ degenerate clusters
def one_pixel(n=40, at=(10.02, 3.02), seed=0):
    """every point inside one 1/18 m pixel (and one cell): W = 1 column, hull m = 1"""
    rng = np.random.default_rng(seed)
    x = at[0] + rng.uniform(0.0, 0.03, n)
    y = at[1] + rng.uniform(0.0, 0.03, n)
    return np.stack([x, y, _z(rng, n)], 1).astype(np.float32)


def pixel_column(n=40, at=(10.02, 6.0), rows=6, seed=0):
    """one pixel column spanning `rows` pixel rows: W = 1, hull m = 2"""
    rng = np.random.default_rng(seed)
    x = at[0] + rng.uniform(0.0, 0.03, n)
    y = at[1] + (rng.integers(0, rows, n) + rng.uniform(0.2, 0.8, n)) / PIC
    y[:2] = at[1] + np.array([0.5, rows - 0.5]) / PIC          # both end rows are present
    return np.stack([x, y, _z(rng, n)], 1).astype(np.float32)


def pixel_diagonal(n=40, at=(-10.0, 3.0), length=8, seed=0):
    """pixels (i, i) of a diagonal line, several columns: hull m = 2"""
    rng = np.random.default_rng(seed)
    i = rng.integers(0, length, n)
    i[:2] = (0, length - 1)
    x = at[0] + (i + rng.uniform(0.3, 0.7, n)) / PIC
    y = at[1] + (i + rng.uniform(0.3, 0.7, n)) / PIC
    return np.stack([x, y, _z(rng, n)], 1).astype(np.float32)


def duplicates(n=40, at=(-10.0, -3.0), distinct=5, seed=0):
    """a few distinct points repeated: equal slopes at equal points, first occurrence decides"""
    rng = np.random.default_rng(seed)
    base = np.stack([at[0] + rng.uniform(0, 0.15, distinct), at[1] + rng.uniform(0, 0.15, distinct), _z(rng, distinct)], 1)
    return base[rng.integers(0, distinct, n)].astype(np.float32)


def slope_ray(n=400, ties=12, seed=0, y_over_x=2.0, x_range=(4.05, 6.0), width=0.3):
    """an L-shape-eligible band above the ray y = 2x (max-slope point near (4.05, 8.4): maxMy > 8), `ties` DISTINCT points exactly
    on the ray at x >= 5 (y/x == 2 in float for each of them): the band's smallest slope, so the min-slope point is the first of
    them in cloud order, more than 1 m from the max-slope point"""
    rng = np.random.default_rng(seed)
    x = rng.uniform(x_range[0], x_range[1], n)
    y = y_over_x * x + rng.uniform(0.02, width, n)
    xt = np.linspace(5.0, x_range[1], ties).astype(np.float32)
    xt = np.float32(np.round(xt * 64) / 64)                      # y = 2x exactly representable
    yt = np.float32(y_over_x) * xt
    pts = np.stack([x, y, _z(rng, n)], 1).astype(np.float32)
    tie = np.stack([xt, yt, _z(rng, ties).astype(np.float32)], 1).astype(np.float32)
    out = np.concatenate([pts, tie])
    out = out[rng.permutation(len(out))]
    assert np.all((out[:, 1] / out[:, 0]) >= np.float32(y_over_x))
    return out


def zero_slope_arm(seed=0):
    """an L: an arm on the x axis (points with y = +0.0 and y = -0.0, slope +-0: the smallest, tied) and an arm up to y = 8.6
    (max-slope point at y > 8: the L-shape branch)"""
    rng = np.random.default_rng(seed)
    n1, n2 = 200, 200
    x1 = rng.uniform(1.0, 3.0, n1)
    y1 = np.where(rng.random(n1) < 0.5, 0.0, -0.0)
    y1[: n1 // 2] = rng.uniform(0.0, 0.1, n1 // 2)                   # and some above the axis
    y1[rng.permutation(n1)[:20]] = -0.0
    x2 = rng.uniform(1.0, 1.1, n2)
    y2 = rng.uniform(0.0, 8.6, n2)
    y2[0] = 8.6
    out = np.stack([np.concatenate([x1, x2]), np.concatenate([y1, y2]), _z(rng, n1 + n2)], 1).astype(np.float32)
    return out[rng.permutation(len(out))]


def on_axis(y0, sign_x, n=200, zeros=10, seed=0):
    """a band at y in [y0, y0 + 1.2], x between 0 and 1.2 * sign_x, `zeros` points exactly at x = +0.0 (sign_x > 0) or -0.0: slope
    +-inf there, tied.  y0 = 9.4 / -9.2 put the cluster's max-slope point beyond y = 8 / -5 (the L-shape branch)."""
    rng = np.random.default_rng(seed)
    x = sign_x * rng.uniform(0.02, 1.2, n)
    y = y0 + rng.uniform(0.0, 1.2, n)
    xz = np.full(zeros, 0.0 if sign_x > 0 else -0.0)
    yz = y0 + rng.uniform(0.1, 1.1, zeros)
    out = np.stack([np.concatenate([x, xz]), np.concatenate([y, yz]), _z(rng, n + zeros)], 1).astype(np.float32)
    return out[rng.permutation(len(out))]


def origin_nan(n=40, seed=0):
    """a cluster round the origin with points exactly at (+-0, +-0): slope NaN, never an extreme"""
    rng = np.random.default_rng(seed)
    p = np.stack([rng.uniform(-0.08, 0.08, n), rng.uniform(-0.08, 0.08, n), _z(rng, n)], 1)
    p[:4, :2] = [[0.0, 0.0], [-0.0, 0.0], [0.0, -0.0], [-0.0, -0.0]]
    return p.astype(np.float32)


def degenerate_set(seed=0):
    """every degenerate cluster above, far enough apart to stay separate components"""
    parts = [one_pixel(seed=seed), pixel_column(seed=seed + 1), pixel_diagonal(seed=seed + 2), duplicates(seed=seed + 3),
             slope_ray(seed=seed + 4), zero_slope_arm(seed=seed + 5),
             on_axis(9.4, +1, seed=seed + 6), on_axis(12.4, -1, seed=seed + 7), on_axis(-10.6, +1, seed=seed + 8),
             on_axis(-13.6, -1, seed=seed + 9), origin_nan(seed=seed + 10)]
    return parts


def interleave(parts, seed=0):
    """concatenate clouds and shuffle their points together"""
    p = np.concatenate([np.asarray(q, np.float32) for q in parts if len(q)])
    return p[np.random.default_rng(seed).permutation(len(p))]


# ------------------------------------------------------------------------------------------------ the scenes of the regime suites
K_SWEEP = (128, 129, 256, 257, 512, 513, 1024, 1025, 3844)   # both sides of every lanes-per-cluster switch, two scan rounds, a full grid
BIG_SIZES = (2047, 2048, 2049, 20000)                         # around one 4 x 512-point batch of box_fit_kernel's per-point pass
HUGE = 200000
PAIR_SIDES = {"at_cap": 31, "over_cap": 32}                   # extra seeds of pair_scene(., rows=195): 4,096 and 4,101 pairs
# raw frames (frame(pair_scene(extra, rows))): groundRemove cuts a disc of 3.4 m out of the block, so other sizes: 4,095 and 4,101 pairs
PAIR_FRAME_SIDES = {"at_cap": (72, 199), "over_cap": (99, 199)}


def k_sweep(K):
    """K lattice clusters of 30 points (min_cluster_points: each is accepted under RULE_GCC13_O2_COMPAT)"""
    return lattice(K, 30, seed=K)


def tiles_few_clusters():
    """128 clusters, 131,840 points: 129 tiles over 8 lanes per cluster -> 17 tiles per lane"""
    return lattice(128, 1030, seed=1)


def tiles_many_clusters():
    """600 clusters, 18,000 points: 18 tiles on one lane per cluster"""
    return lattice(600, 30, seed=2)


def big_clusters(sizes=BIG_SIZES, seed=0):
    """discs of the given sizes twice: on the x axis (minimum-area-rectangle branch) and at y = 12 (L-shape branch)"""
    parts = []
    for i, n in enumerate(sizes):
        parts.append(disc(n, (6.0 + 4.0 * i, 0.0), 0.8, seed=seed + i))
        parts.append(disc(n, (-6.0 + 4.0 * i, 12.0), 0.8, seed=seed + 100 + i))
    return interleave(parts, seed)


def huge_cluster(l_shape):
    """one cluster of 200,000 points"""
    return disc(HUGE, (-4.0, 14.0) if l_shape else (10.0, -1.0), 2.0, seed=7 if l_shape else 8)


def mixed(seed=0):
    """big objects, degenerate clusters, L-shape objects at |y| > 8, and a lattice of clusters of 2..59 points around them (those
    below 30 are rejected by ruleBasedFilter's first test before any fit), interleaved in cloud order"""
    rng = np.random.default_rng(seed)
    objs = [disc(2049, (18.0, 1.0), 0.8, seed=seed), ring(20000, centre=(-12.0, -12.0), r_in=5.0, r_out=5.3, seed=seed + 1),
            rect(3000, (14.0, 14.0), 4.0, 1.8, 0.4, seed=seed + 2, hollow=True), rect(1500, (-16.0, 10.0), 3.0, 1.5, -0.3, seed=seed + 3, hollow=True),
            rect(800, (8.0, -12.0), 4.5, 2.0, 1.2, seed=seed + 4, hollow=True)] + degenerate_set(seed + 5)
    obj = np.concatenate(objs)
    keep = keep_away(obj)
    n_free = int(keep(*lattice_sites(SITES * SITES)).sum())
    K = n_free - 10
    lat = lattice(K, rng.integers(2, 60, K), seed=seed + 6, keep=keep, neighbours=2)
    return interleave([obj, lat], seed)


def grid_sequence():
    """frames for the sparse label-grid update: a full lattice, one cluster, nothing, the lattice shifted by one cell"""
    full = lattice(3844, 2, seed=11, random_sites=False)
    one = lattice(1, 40, seed=12)
    shifted = full.copy()
    shifted[:, :2] += np.float32(CELL)
    return [full, one, np.zeros((0, 3), np.float32), shifted]


def batch_scenes():
    """eight elevated clouds in different regimes, all beyond the sensor's 3.4 m minimum range: K > 256, K > 1024, clusters of
    1,023 / 1,024 / 1,025 / 3,000 points (one 4 x 256-point batch of the batched per-point pass and more), many tiles per lane, a ring,
    an empty frame"""
    far = sensor_range()
    big = [disc(n, (8.0 + 3.0 * i, -6.0), 0.7, seed=20 + i) for i, n in enumerate((1023, 1024, 1025, 3000))]
    big_keep = keep_away(np.concatenate(big))
    return [lattice(300, 30, seed=21, keep=far),
            lattice(1100, 30, seed=22, keep=far),
            interleave(big + [lattice(100, 30, seed=23, keep=lambda ix, iy: far(ix, iy) & big_keep(ix, iy))], 24),
            lattice(128, 200, seed=25, keep=far),
            lattice(513, 31, seed=26, keep=far),
            np.zeros((0, 3), np.float32),
            lattice(40, 60, seed=27, keep=far),
            ring(30000, seed=28)]


# ------------------------------------------------------------------------------------------------ raw frames for ground removal
def ground_disc(r_min=3.5, r_max=36.0, n_r=160, n_a=720, z=-2.0):
    """flat ground at z = -2 in every polar cell the lattice can reach, so that the reference's ground estimate sits there and
    points at Z_KEEP heights stay elevated"""
    r = np.linspace(r_min, r_max, n_r)
    a = np.linspace(-np.pi, np.pi, n_a, endpoint=False) + 0.5 * np.pi / n_a
    R, A = np.meshgrid(r, a, indexing="ij")
    return np.stack([R.ravel() * np.cos(A.ravel()), R.ravel() * np.sin(A.ravel()), np.full(R.size, z)], 1).astype(np.float32)


def sensor_range(r_min=4.0):
    """keep(ix, iy) for lattice(): whole 3x3 blocks beyond r_min of the sensor (groundRemove drops points nearer than 3.4 m)"""
    return lambda ix, iy: np.hypot(cell_centre(ix), cell_centre(iy)) > r_min + 0.5


def frame(elevated, ground=None):
    """a raw frame: the elevated cloud and ground points, interleaved, XYZ"""
    g = ground_disc() if ground is None else ground
    return interleave([elevated, g], seed=len(elevated))


# ------------------------------------------------------------------------------------------------ reference-side witnesses
def cluster_ids(elevated, grid):
    """the cluster id of every point by box_fitting.cpp:53-58 (0: outside the ROI or unlabelled)"""
    xi, yi = cells_of(elevated)
    cid = np.zeros(len(xi), np.int64)
    ok = xi >= 0
    cid[ok] = np.asarray(grid)[xi[ok], yi[ok]]
    return cid


def cluster_sizes(elevated, grid, k):
    """points per cluster 1..k from the reference's label grid"""
    return np.bincount(cluster_ids(elevated, grid), minlength=k + 1)[1: k + 1]


def n_tiles(n):
    return (n + TILE - 1) // TILE


def seg_lanes(k):
    """lanes per cluster of the segment-offset scan (boxfit.cu seg_offsets_body)"""
    return 8 if k <= 128 else (4 if k <= 256 else (2 if k <= 512 else 1))


def tiles_per_lane(n, k):
    P = seg_lanes(k)
    return (n_tiles(n) + P - 1) // P


def _pieces(word):
    """(start, length) of the maximal runs of set bits of a 32-bit word"""
    out, b = [], 0
    while b < 32:
        if (word >> b) & 1:
            s = b
            while b < 32 and (word >> b) & 1:
                b += 1
            out.append((s, b - s))
        else:
            b += 1
    return out


def ccl_pairs(occupied):
    """adjacencies the CCL kernel cannot express as a piece's first parent (ccl_device.cuh step C), restated from the occupancy:
    rows = x, 250 bits per row in eight 32-bit words, a piece = a run of set bits inside one word; a piece's candidates are the
    piece it continues from the previous word, the touching pieces of the row above in the same word, and those across the word
    borders above; every candidate but one is a pair."""
    occ = np.asarray(occupied, bool)
    words = np.zeros((NUM_GRID, 8), np.int64)
    for k in range(8):
        seg = occ[:, 32 * k: 32 * k + 32]
        words[:, k] = (seg.astype(np.int64) << np.arange(seg.shape[1], dtype=np.int64)).sum(1)
    pairs = 0
    for x in range(NUM_GRID):
        for k in range(8):
            m = int(words[x, k])
            if not m:
                continue
            up = int(words[x - 1, k]) if x > 0 else 0
            upl = int(words[x - 1, k - 1]) if x > 0 and k > 0 else 0
            upr = int(words[x - 1, k + 1]) if x > 0 and k < 7 else 0
            left = int(words[x, k - 1]) if k > 0 else 0
            up_pieces = _pieces(up)
            for a, ln in _pieces(m):
                pm = ((1 << ln) - 1) << a
                touch = (pm | (pm << 1) | (pm >> 1)) & 0xFFFFFFFF
                cand = 0
                cand += 1 if a == 0 and (left >> 31) & 1 else 0
                cand += 1 if a + ln == 32 and upr & 1 else 0
                cand += sum(1 for s, l in up_pieces if touch & (((1 << l) - 1) << s))
                cand += 1 if a == 0 and (upl >> 31) & 1 else 0
                pairs += max(0, cand - 1)
    return pairs


def pixels(points):
    """(picX, picY) of box_fitting.cpp:244-251 (the cluster's offset to point #0 is a translation: it leaves the hull's shape)"""
    p = np.asarray(points, np.float32)
    half, pic = np.float32(ROI / 2), np.float32(PIC)
    x = np.floor((p[:, 0] + half) * pic).astype(np.int64)
    y = np.floor((p[:, 1] + half) * pic).astype(np.float32)
    return np.stack([x, (pic * np.float32(ROI) - y).astype(np.int64)], 1)


def hull_size(points):
    """vertices of the strict convex hull of a cluster's pixel set (the minimum-area-rectangle input)"""
    from test_mar_contract import _hull
    return len(_hull(pixels(points).tolist()))


def pixel_columns(points):
    return len(np.unique(pixels(points)[:, 0]))


def takes_l_shape(points, l_slope_dist=1.0, l_num_points=5):
    """box_fitting.cpp:296-300 on a cluster in cloud order: first-occurrence min / max slope points, then the L-shape gate"""
    p = np.asarray(points, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = p[:, 1] / p[:, 0]
    lo = np.where(m < 999)[0]
    hi = np.where(m > -999)[0]
    i_min = lo[np.argmin(m[lo])]                       # argmin / argmax: first occurrence
    i_max = hi[np.argmax(m[hi])]
    dx, dy = p[i_max, 0] - p[i_min, 0], p[i_max, 1] - p[i_min, 1]
    dist = np.sqrt(np.float32(dx * dx + dy * dy))
    return bool(dist > l_slope_dist and len(p) > l_num_points and (p[i_max, 1] > 8 or p[i_max, 1] < -5))


def slope_ties(points):
    """(points tied at the smallest slope, at the largest), counting DISTINCT points only"""
    p = np.asarray(points, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = p[:, 1] / p[:, 0]
    lo, hi = m[m < 999], m[m > -999]
    at_min = np.unique(p[:, :2][(m < 999) & (m == lo.min())], axis=0)
    at_max = np.unique(p[:, :2][(m > -999) & (m == hi.max())], axis=0)
    return len(at_min), len(at_max)
