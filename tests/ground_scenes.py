"""Scene builders and witnesses for the ground-removal regime suites (numpy only, no GPU).

ground_fused_kernel (csrc/ground.cu) switches paths by data size and content: the CTA count G and chunk per CTA of a launch
(ground_launch_batch, with the half-SM cap of the frame pipeline), tiles per chunk T (pairs of full resident tiles vs the tail, 8
resident tiles then global re-reads, 16 at most), the queue of points whose cell needs the exact evaluation (2,048 per CTA, the rest
evaluated inline), label limits staged in shared memory for chunks above 2,048 points or gathered per point below, and phase 2's
split of the 80 channels over min(G, 80) CTAs.  `launch` restates that geometry as a pure function of the frame sizes and the
device's SM count; the builders make clouds that sit on a chosen side of each switch, and the witnesses restate from the
REFERENCE's outputs (passed in) which side a scene reached and that its probes are one-sided or on a tie.

Polar grid (ground_removal.cpp:67-76): 80 channels of 2 pi / 80 from -pi, 120 bins of (rMax - rMin) / 120 from rMin = 3.4 m.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
NUM_CHANNEL, NUM_BIN = 80, 120
R_MIN, R_MAX = 3.4, 120.0
TILE = 1024                     # points per TMA tile == threads per CTA
RES_TILES = 8                   # tiles of a chunk that stay in shared memory
MAX_TILES = 16                  # tiles per chunk at most
PEND_CAP = 2048                 # queued points per CTA; the rest are evaluated inline
MIN_CTAS = 8
DENSE_SMEM = 32000 * 4 + 3 * 2000 * 4 + 2008 * 4 + 4096 * 4 + 64 * 4     # ccl_device.cuh kDenseSmem (fused clustering tail)
DEFAULT_PPC = 768               # Ctx::pts_per_cta
T_HMIN, T_HMAX, H_SENSOR = -2.0, -0.4, 2.0
# documented distance of the fast path's coordinates from the reference's (ground.cu), and its guards
CHAN_SURE, BIN_SURE = 1e-4, 3e-4          # certainly queued: within this of an integer (exact float64 coordinates)
CHAN_GUARD, BIN_GUARD = 2e-4, 6e-4


# ------------------------------------------------------------------------------------------------ launch geometry
def _smem_layout():
    off_cnt = 128
    off_wex = off_cnt + MAX_TILES * 32 * 4
    off_ttot = off_wex + MAX_TILES * 32 * 4
    off_base = off_ttot + MAX_TILES * 4
    off_pend = (off_base + 16 + 15) & ~15
    off_g = off_pend + PEND_CAP * 2
    loc = (NUM_CHANNEL // MIN_CTAS + 2) * NUM_BIN
    off_h = (off_g + loc + 127) & ~127
    off_keys = (off_h + loc * 4 + 127) & ~127
    return (off_keys + NUM_CHANNEL * NUM_BIN * 4 + 127) & ~127


OFF_PTS = _smem_layout()


def fused_smem_bytes(res_tiles, tiles):
    return OFF_PTS + res_tiles * TILE * 16 + tiles * TILE * 2


def launch(ns, sms, ppc=DEFAULT_PPC, entry="stage", prefilter=False):
    """ground_launch_batch's geometry for frames of ns points on a device whose cooperative limit is `sms` CTAs.  entry: "stage"
    (lmot_ground_remove / _dev), "frame" (lmot_frame*: one frame, fused counts, half-SM cap), "batch" or "seq".  -> dict with G, the
    chunk of every frame, per frame and CTA (beg, cnt, T, res_tiles, full pairs), stage_lim, gc with its own channels, and the dynamic
    shared memory; capacity=True where the launch refuses the frame."""
    ns = [int(n) for n in ns]
    F, n_max = len(ns), max(ns)
    G = max(-(-n_max // ppc), MIN_CTAS)
    cap = sms // F
    half = False
    if entry == "frame" and F == 1:
        h = max(cap // 2, MIN_CTAS)
        if h * RES_TILES * TILE >= n_max:
            cap, half = h, True
    G = min(G, cap)
    chunks = [-(-n // G) for n in ns]
    geo = dict(G=G, F=F, ns=ns, chunks=chunks, half=half, sms=sms, entry=entry,
               capacity=any(c > MAX_TILES * TILE for c in chunks))
    tiles = -(-max(chunks) // TILE)
    smem = fused_smem_bytes(min(tiles, RES_TILES), max(tiles, 1))
    if entry != "stage":                          # lmot_frame / batch / seq fuse the clustering into the kernel's tail
        smem = max(smem, DENSE_SMEM)
    geo["smem"] = smem
    frames = []
    for n, chunk in zip(ns, chunks):
        t_max = -(-chunk // TILE)
        res = min(t_max, RES_TILES)
        ctas = []
        for c in range(G):
            beg = min(c * chunk, n)
            cnt = min(n, beg + chunk) - beg
            T = -(-cnt // TILE)
            full = 0 if prefilter else (min(cnt // TILE, res) & ~1) // 2
            ctas.append(dict(beg=beg, cnt=cnt, T=T, full_pairs=full))
        frames.append(dict(n=n, chunk=chunk, res_tiles=res, stage_lim=chunk > 2 * TILE, ctas=ctas))
    geo["frames"] = frames
    gc = min(G, NUM_CHANNEL)
    geo["gc"] = gc
    geo["own"] = [(c * NUM_CHANNEL // gc, (c + 1) * NUM_CHANNEL // gc) for c in range(gc)]
    return geo


def ppc_for(G, n):
    """LMOT_PTS_PER_CTA that makes a stage launch of n points run on exactly G CTAs (None: no value in [256, 16384] does)"""
    for ppc in range(max(256, -(-n // G)), 16385):
        if max(-(-n // ppc), MIN_CTAS) == G:
            return ppc
        if -(-n // ppc) < G:
            return None
    return None


def describe(geo, frame=0):
    f = geo["frames"][frame]
    Ts = sorted({c["T"] for c in f["ctas"]})
    return (f"G={geo['G']} chunk={f['chunk']} T={Ts} res_tiles={f['res_tiles']} stage_lim={f['stage_lim']} gc={geo['gc']} "
            f"half_cap={geo['half']} smem={geo['smem']}")


# ------------------------------------------------------------------------------------------------ polar coordinates
def coords(pts, r_min=R_MIN, r_max=R_MAX):
    """exact float64 (channel, bin) coordinates of float32 points (NaN where x or y is not finite)"""
    p = np.asarray(pts, f32)
    x, y = p[:, 0].astype(np.float64), p[:, 1].astype(np.float64)
    with np.errstate(invalid="ignore"):
        d = np.hypot(x, y)
        rmin = float(f32(r_min))
        span = float(f32(f32(r_max) - f32(r_min)))
        b = (d - rmin) * NUM_BIN / span
        ch = (np.arctan2(y, x) + np.pi) / (2 * np.pi) * NUM_CHANNEL
    return ch, b


def _frac_dist(v):
    return np.abs(v - np.round(v))


def certainly_queued(pts, r_min=R_MIN, r_max=R_MAX):
    """points the fast path certainly hands to the exact evaluation: x or y not finite, x = y = 0 (its t is NaN), and points whose
    exact channel / bin coordinate is within 1e-4 channel / 3e-4 bin widths of an integer (inside the guards by more than the
    fast path's documented error), inside the range window the fast path tests first"""
    p = np.asarray(pts, f32)
    x, y = p[:, 0], p[:, 1]
    ch, b = coords(p, r_min, r_max)
    with np.errstate(invalid="ignore"):
        bad = ~np.isfinite(x) | ~np.isfinite(y) | ((x == 0) & (y == 0))
        window = (b >= -BIN_SURE) & (b <= NUM_BIN + BIN_SURE)
        near = (_frac_dist(ch) < CHAN_SURE) | (_frac_dist(b) < BIN_SURE)
    return bad | (window & near)


def certainly_fast(pts, r_min=R_MIN, r_max=R_MAX):
    """points the fast path certainly decides itself (cell id or out of range): both coordinates well clear of every integer"""
    ch, b = coords(pts, r_min, r_max)
    with np.errstate(invalid="ignore"):
        inside = (_frac_dist(ch) > 3 * CHAN_GUARD) & (_frac_dist(b) > 3 * BIN_GUARD) & (b > 0.01) & (b < NUM_BIN - 0.01)
        outside = (b < -0.01) | (b > NUM_BIN + 0.01)
    return np.isfinite(ch) & (inside | outside)


def queued_per_cta(pts, geo, frame=0, **kw):
    """(certainly queued, certainly fast) point counts of every CTA of one frame of a launch"""
    q = certainly_queued(pts, **kw)
    s = certainly_fast(pts, **kw)
    out = []
    for c in geo["frames"][frame]["ctas"]:
        sl = slice(c["beg"], c["beg"] + c["cnt"])
        out.append((int(q[sl].sum()), int(s[sl].sum())))
    return np.array(out, np.int64).reshape(-1, 2)


# ------------------------------------------------------------------------------------------------ cells and limits
def cell_xy(ch, b, fc=0.5, fb=0.5, r_min=R_MIN, r_max=R_MAX):
    """float32 (x, y) at channel / bin coordinate ch + fc, b + fb"""
    span = float(f32(f32(r_max) - f32(r_min)))
    r = float(f32(r_min)) + (np.asarray(b, np.float64) + fb) * span / NUM_BIN
    a = -np.pi + (np.asarray(ch, np.float64) + fc) * 2 * np.pi / NUM_CHANNEL
    return (r * np.cos(a)).astype(f32), (r * np.sin(a)).astype(f32)


def cloud(x, y, z):
    return np.stack([np.asarray(x, f32), np.asarray(y, f32), np.broadcast_to(np.asarray(z, f32), np.shape(x))], 1).astype(f32)


def label_limit(h, tol):
    """the largest float L with (double)L < (double)h + tol, per cell (ground_removal.cpp:239 as one float compare z <= L)"""
    h = np.asarray(h, f32)
    thr = h.astype(np.float64) + tol
    f = thr.astype(f32)
    f = np.where(f.astype(np.float64) > thr, np.nextafter(f, f32(-np.inf)), f)
    f = np.where(f.astype(np.float64) == thr, np.nextafter(f, f32(-np.inf)), f)
    return f.astype(f32)


def full_floor(heights, r_min=R_MIN, r_max=R_MAX, per_cell=1):
    """per_cell points at the centre of every cell, z = heights[ch, b] (80 x 120): the cell minima"""
    ch, b = np.meshgrid(np.arange(NUM_CHANNEL), np.arange(NUM_BIN), indexing="ij")
    x, y = cell_xy(ch.ravel(), b.ravel(), r_min=r_min, r_max=r_max)
    p = cloud(x, y, np.asarray(heights, f32).ravel())
    return np.tile(p, (per_cell, 1)) if per_cell > 1 else p


# ------------------------------------------------------------------------------------------------ one-sided checkerboard
LOW, HIGH, PROBE_Z = -1.8, -1.45, -1.4


def checker_heights(shift=0.0):
    """floor -1.8 where channel + bin is even, -1.45 where odd: bin neighbours differ by 0.35 < tHDiff, so every cell is ground"""
    ch, b = np.meshgrid(np.arange(NUM_CHANNEL), np.arange(NUM_BIN), indexing="ij")
    return np.where((ch + b) % 2 == 0, f32(LOW + shift), f32(HIGH + shift)).astype(f32)


def checker_probe_pool(cell_index, n=24000, seed=0, shift=0.0, window=None):
    """boundary-hugging probes at z = -1.4 (+ shift) inside LOW cells, kept where the reference's cell (cell_index: the reference's
    getCellIndexFromPoints) is that low cell, the neighbour across the nearest boundary is a high cell of the grid, and the point is
    certainly queued.  In the low cell -1.4 is elevated (limit -1.55 at tolerance 0.25, -1.5 at 0.3, -1.7 at 0.1), in the high one
    ground: a wrong cell turns elevated into ground, a dropped point removes an elevated one.  window(x, y) -> bool restricts them."""
    rng = np.random.default_rng(seed)
    out, m = [], 3 * n
    for _ in range(40):
        out.append(_probe_batch(cell_index, rng, m, shift, window))
        if sum(len(p) for p in out) >= n:
            return np.concatenate(out)[:n]
    raise ValueError(f"only {sum(len(p) for p in out)} probes")


def _probe_batch(cell_index, rng, m, shift, window):
    ch = rng.integers(0, NUM_CHANNEL, m)
    b = rng.integers(1, NUM_BIN - 1, m)
    b = np.where((ch + b) % 2 == 0, b, b + np.where(b < NUM_BIN - 2, 1, -1))           # a low cell
    side = rng.integers(0, 4, m)
    eps_c = rng.uniform(2e-6, 8e-5, m)
    eps_b = rng.uniform(2e-5, 2.5e-4, m)
    fc = np.where(side == 0, eps_c, np.where(side == 1, 1 - eps_c, rng.uniform(0.3, 0.7, m)))
    fb = np.where(side == 2, eps_b, np.where(side == 3, 1 - eps_b, rng.uniform(0.3, 0.7, m)))
    x, y = cell_xy(ch, b, fc, fb)
    p = cloud(x, y, f32(PROBE_Z + shift))
    rc, rb = cell_index(p)
    keep = (rc == ch) & (rb == b) & certainly_queued(p)          # channels wrap (0 | 79 across -pi); b in 1..118: both bin neighbours exist
    if window is not None:
        keep &= window(p[:, 0], p[:, 1])
    return p[keep]


def layout(geo, queued, probes, floor, seed=0, frame=0):
    """a frame for one launch geometry: CTA c's chunk holds queued[c] probes (cycled) and floor points for the rest (cycled across the
    whole frame, so every cell gets its minimum), shuffled inside the chunk"""
    rng = np.random.default_rng(seed)
    out, ip, iflo = [], 0, 0
    for c, q in zip(geo["frames"][frame]["ctas"], queued):
        cnt = c["cnt"]
        q = min(int(q), cnt)
        pi = (ip + np.arange(q)) % len(probes); ip += q
        fi = (iflo + np.arange(cnt - q)) % len(floor); iflo += cnt - q
        chunk = np.concatenate([probes[pi], floor[fi]])
        out.append(chunk[rng.permutation(cnt)])
    return np.concatenate(out) if out else np.zeros((0, 3), f32)


# ------------------------------------------------------------------------------------------------ tie probes
def smooth_heights(centre, amp=0.12, seed=0, exact=None):
    """an all-ground floor: centre + a smooth wave + jitter (bin neighbours well within tHDiff); exact: (value, fraction of cells)
    pins that many cells to exactly `value`"""
    rng = np.random.default_rng(seed)
    ch, b = np.meshgrid(np.arange(NUM_CHANNEL), np.arange(NUM_BIN), indexing="ij")
    h = centre + amp * np.sin(ch * 0.37 + b * 0.11) + rng.uniform(-0.03, 0.03, ch.shape)
    if exact is not None:
        h = np.where(rng.random(ch.shape) < exact[1], exact[0], h)
    return h.astype(f32)


def tie_probes(hground, isground, tol, zero=False, minz=None):
    """cell-centre points on the tie of every ground cell: z = L, the floats either side of it, and float(h + tol) rounded to
    nearest (L the reference's limit); zero: also +-0 and +-denormal, for cells whose limit is -denormal (h + tol == 0).
    minz: only cells whose minimum stays below every probe (a filter may have lowered a cell's height under its minimum).
    -> (points, expected reference label 1 / 2)"""
    ch, b = np.nonzero(np.asarray(isground).astype(bool))
    h = np.asarray(hground, f32)[ch, b]
    L = label_limit(h, tol)
    if minz is not None:
        keep = np.nextafter(L, f32(-np.inf)) >= np.asarray(minz, f32)[ch, b]
        ch, b, h, L = ch[keep], b[keep], h[keep], L[keep]
    zs = [L, np.nextafter(L, f32(-np.inf)), np.nextafter(L, f32(np.inf)), (h.astype(np.float64) + tol).astype(f32)]
    want = [np.ones_like(L, np.uint8), np.ones_like(L, np.uint8), np.full(L.shape, 2, np.uint8),
            np.where((h.astype(np.float64) + tol).astype(f32).astype(np.float64) < h.astype(np.float64) + tol, 1, 2).astype(np.uint8)]
    if zero:
        den = np.float32(np.finfo(f32).smallest_subnormal)
        z0 = L == -den
        for z, w in ((f32(-0.0), 2), (f32(0.0), 2), (-den, 1), (den, 2)):
            zs.append(np.where(z0, z, L)); want.append(np.where(z0, w, 1).astype(np.uint8))
    x, y = cell_xy(ch, b)
    pts = np.concatenate([cloud(x, y, z) for z in zs])
    return pts, np.concatenate(want)


# ------------------------------------------------------------------------------------------------ filter patterns at CTA seams
BG = -1.7


def seam_channels(gc):
    """first and last own channel of every phase-2 CTA for gc CTAs, where both filters may act (channels 1..78)"""
    chans = set()
    for c in range(gc):
        a, e = c * NUM_CHANNEL // gc, (c + 1) * NUM_CHANNEL // gc
        chans.update((a, e - 1))
    return sorted(ch for ch in chans if 1 <= ch <= NUM_CHANNEL - 2)


def seam_scene(gc):
    """floor BG = -1.7 in every cell; per seam channel ch a median-filter hole at (ch, bm): floor -1.2 (hDiff 0.5: not ground) with
    channel neighbours (ch +- 1, bm - 1..bm + 1) at -0.9, rewritten to -1.3 and ground, so its -1.2 minimum turns ground; and an
    outlier-filter cell at (ch, bo): minimum -2.1 (height tHmin) between ground neighbours, rewritten to -1.7, with a probe at z = -1.5
    that the rewrite turns ground.  -> (points, [(kind, ch, b)])"""
    h = np.full((NUM_CHANNEL, NUM_BIN), BG, f32)
    probes, marks = [], []
    for ch in seam_channels(gc):
        bm = 6 + 12 * (ch % 4)
        bo = 62 + 12 * (ch % 4)
        h[ch, bm] = -1.2
        for d in (-1, 1):
            h[ch + d, bm - 1: bm + 2] = -0.9
        h[ch, bo] = -2.1
        x, y = cell_xy([ch, ch], [bo, bm])
        probes.append(cloud(x, y, [-1.5, -1.1]))
        marks += [("median", ch, bm), ("outlier", ch, bo)]
    pts = np.concatenate([full_floor(h)] + probes)
    return pts, marks


def rewritten(grid, ch, b, t_hmin=T_HMIN, t_hmax=T_HMAX, h_sensor=H_SENSOR):
    """did the reference's filters rewrite cell (ch, b): its final height differs from the clamp of its minimum"""
    zi = grid["minz"][ch, b]
    h = zi if t_hmin < zi < t_hmax else (h_sensor if zi > t_hmax else t_hmin)
    return bool(grid["height"][ch, b] != f32(h))


# ------------------------------------------------------------------------------------------------ organized frames
def organized(cell_index, rings=128, azimuths=2048, seed=0, nan_rows=True):
    """a ring-major organized frame: groups of four rows -- two rows of in-range boundary probes (checkerboard), one row of missing
    returns ((0, 0, 0), or NaN in every other group), one row of floor points -- so a chunk of two rows queues ~4,000 in-range points"""
    floor = full_floor(checker_heights())
    probes = checker_probe_pool(cell_index, n=2 * azimuths * rings // 4, seed=seed)
    rows, ip, iflo = [], 0, 0
    for r in range(rings):
        k = r % 4
        if k in (0, 1):
            rows.append(probes[ip: ip + azimuths]); ip += azimuths
        elif k == 2:
            v = np.nan if (nan_rows and (r // 4) % 2) else 0.0
            rows.append(np.full((azimuths, 3), v, f32))
        else:
            rows.append(floor[(iflo + np.arange(azimuths)) % len(floor)]); iflo += azimuths
    return np.concatenate(rows).astype(f32)
