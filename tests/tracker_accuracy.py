"""Per-step accuracy of a tracker evaluation against the extended-precision restatement of the reference (oracle.ref.PortOracleHP).

One teacher-forced step gives three evaluations of the same function from the same track table: the reference in double, the
restatement in x87 long double (`hp`, error ~1e-19, taken as exact) and the evaluation under test (`got`: the CUDA kernels, or a
mutated copy of an oracle's arrays).  For every live track each block -- x and P per model (merge, cv, ctrv, rm), the mode
probabilities, zPred, S and K per model, the step's (v, yaw) output -- has an error
    e = max |value - hp| / max |hp|   over the block,
yaw entries compared modulo 2 pi (remainder), NaN on both sides agreeing and NaN on one side an infinite error.  e_ref is the
reference's, e_got the evaluation's; a block passes if

    e_got <= max(C * e_ref, F)  and  e_got <= CEIL.

Setting the bar from e_ref makes it as tight as the step's own conditioning allows: a well-conditioned step has e_ref ~ 1e-16 and
the bar sits at F, an ill-conditioned one (a covariance near singular, a cancelling P - K S K^T) has a larger e_ref and the bar
follows it up to the hard ceiling.  Blocks with e_ref > CEIL are ill-conditioned beyond what double can resolve: they are
excluded and counted.  A step on which hp and the reference disagree on any integer (trackManage, lifetime, static, visible) is
a different function and is excluded as a whole.  Float outputs (targets, vis_bb and each track's BBox / bestBBox) are compared
with the reference and must be within 1 ulp; how many are not bit-equal is counted.

Constants:
  C = 16     : the CUDA kernels evaluate the same sums and products in a different order (warp reductions over sigma points, FMA
               contraction, CUDA's libm): a few roundings more or fewer than the reference per output, each of the size of the
               reference's own.  Measured on an H100 SXM (700 W limit), 21 cases: e_cuda / e_ref has median 1.0 and p99 2-4 per
               block kind; ratios up to ~1e3 occur only where e_ref is ~1e-16, with e_cuda far below F.  Worst e_cuda 1.7e-12.
  F = 2^-40  : ~9.1e-13.  Blocks the reference evaluates exactly (e_ref = 0: a freshly spawned track, K of a one-box update)
               still allow rounding at this level; it is ~4000x double's epsilon and ~2000x below a float intermediate (1e-7
               relative would show as >= 6e-8).
  CEIL = 1e-9: never loosened.
"""
from __future__ import annotations

import numpy as np

C_RATIO = 16.0
F_FLOOR = 2.0 ** -40
CEIL = 1e-9
EXCLUDED_SHARE = 0.01
TWO_PI = 2 * np.pi

D_X, D_P, D_MODE, D_ZPRED, D_S, D_K = 4, 24, 124, 127, 133, 145     # dump columns (oracle/port/api.cpp, api.cu)
D_BB, D_BESTBB = 187, 212
INTS = slice(0, 4)                                                   # trackNum, lifetime, isStatic, isVisBB

# (block kind, model, first column, width, yaw entry or None)
DUMP_BLOCKS = ([("x", m, D_X + 5 * m, 5, 3) for m in range(4)] + [("P", m, D_P + 25 * m, 25, None) for m in range(4)]
               + [("modeProb", 0, D_MODE, 3, None)] + [("zPred", m, D_ZPRED + 2 * m, 2, None) for m in range(3)]
               + [("S", m, D_S + 4 * m, 4, None) for m in range(3)] + [("K", m, D_K + 10 * m, 10, None) for m in range(3)])
KINDS = ("x", "P", "modeProb", "zPred", "S", "K", "vandyaw")
PRED_BLOCKS = (("x", 5, 3), ("P", 25, None), ("mode_prob", 3, None), ("gate_z", 2, None), ("gate_S", 4, None))


def block_error(got, hp, yaw=None):
    """rows of `got` / `hp` (n, w) -> (n,) errors max|got - hp| / max|hp|, evaluated in long double"""
    g, h = np.asarray(got, np.longdouble), np.asarray(hp, np.longdouble)
    g, h = g.reshape(len(g), int(np.prod(g.shape[1:]))), h.reshape(len(h), int(np.prod(h.shape[1:])))
    with np.errstate(all="ignore"):
        d = g - h
        if yaw is not None:
            d[:, yaw] -= TWO_PI * np.round(d[:, yaw] / TWO_PI)
        d = np.abs(d)
        gn, hn = np.isnan(g), np.isnan(h)
        d[gn & hn] = 0
        d[g == h] = 0                                   # equal infinities
        d[gn ^ hn] = np.inf
        scale = np.where(hn, 0, np.abs(h)).max(1)
        num = d.max(1)
        e = np.where(scale > 0, num / np.where(scale > 0, scale, 1), np.where(num > 0, np.inf, 0))
    return e.astype(np.float64)


def ulp_distance(a, b):
    """|a - b| in float32 ulps (NaN on both sides: 0, on one side: a huge distance)"""
    def ordered(x):
        i = np.ascontiguousarray(np.asarray(x, np.float32)).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    d = np.abs(ordered(a) - ordered(b))
    d[np.isnan(a) & np.isnan(b)] = 0
    d[np.isnan(a) ^ np.isnan(b)] = 1 << 40
    return d


def passes(e_got, e_ref, C=C_RATIO, F=F_FLOOR):
    return (e_got <= np.maximum(C * e_ref, F)) & (e_got <= CEIL)


class Accuracy:
    """Blockwise errors of one test's steps; check() applies the bar to everything collected and prints the distributions."""

    def __init__(self, name, C=C_RATIO, F=F_FLOOR):
        self.name, self.C, self.F = name, C, F
        self.kind, self.e_got, self.e_ref, self.where = [], [], [], []
        self.steps = self.excluded_steps = 0
        self.float_outputs = self.float_not_equal = 0
        self.float_worst_ulp = 0

    # ---------------------------------------------------------------- collection
    def _add(self, kind, e_got, e_ref, where):
        self.kind += [kind] * len(e_got)
        self.e_got.append(np.asarray(e_got, np.float64)); self.e_ref.append(np.asarray(e_ref, np.float64))
        self.where += where

    def _floats(self, a, b):
        a, b = np.asarray(a, np.float32).ravel(), np.asarray(b, np.float32).ravel()
        assert a.shape == b.shape, (a.shape, b.shape)
        u = ulp_distance(a, b)
        self.float_outputs += u.size
        self.float_not_equal += int((u > 0).sum())
        self.float_worst_ulp = max(self.float_worst_ulp, int(u.max()) if u.size else 0)

    def step(self, ref, hp, got, where):
        """one teacher-forced step; ref / hp / got = (step result dict, dump after the step).  -> False if the step was excluded
        (hp and the reference took different decisions).  The evaluation under test must take the reference's decisions."""
        (a, da), (h, dh), (b, db) = ref, hp, got
        self.steps += 1
        if (da.shape != dh.shape or any(not np.array_equal(a[k], h[k]) for k in ("track_manage", "is_static", "is_vis"))
                or not np.array_equal(da[:, INTS], np.asarray(dh[:, INTS], np.float64))):
            self.excluded_steps += 1
            return False
        for k in ("track_manage", "is_static", "is_vis"):
            assert np.array_equal(a[k], b[k]), (self.name, where, k)
        assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (self.name, where, "integers")
        live = np.nonzero(da[:, 0] > 0)[0]
        w = [(where, int(i)) for i in live]
        for kind, m, c0, n, yaw in DUMP_BLOCKS:
            cols = slice(c0, c0 + n)
            hpb = dh[live, cols]
            self._add(kind, block_error(db[live, cols], hpb, yaw), block_error(da[live, cols], hpb, yaw), [(ww, m) for ww in w])
        hv = np.asarray(h["vandyaw"])[live]
        self._add("vandyaw", block_error(np.asarray(b["vandyaw"])[live], hv, 1), block_error(np.asarray(a["vandyaw"])[live], hv, 1),
                  [(ww, 0) for ww in w])
        self._floats(b["targets"], a["targets"])
        self._floats(b["vis_bb"], a["vis_bb"])
        box = live[da[live, D_BB - 1] > 0]
        self._floats(db[box, D_BB:D_BB + 24], da[box, D_BB:D_BB + 24])
        best = live[da[live, D_BESTBB - 1] > 0]
        self._floats(db[best, D_BESTBB:D_BESTBB + 24], da[best, D_BESTBB:D_BESTBB + 24])
        return True

    def predict(self, want, hp, got, where):
        """one prediction call (dicts of Lmot.predict_tracks / PortOracle.tracker_predict), rows with the valid flag"""
        self.steps += 1
        if not (np.array_equal(want["track_manage"], hp["track_manage"]) and np.array_equal(want["flags"], hp["flags"])):
            self.excluded_steps += 1
            return False
        assert np.array_equal(got["track_manage"], want["track_manage"]) and np.array_equal(got["flags"], want["flags"]), where
        j, i = np.nonzero(want["flags"] & 1)
        w = [(where, (int(jj), int(ii))) for jj, ii in zip(j, i)]
        for kind, n, yaw in PRED_BLOCKS:
            hpb = np.asarray(hp[kind])[j, i].reshape(-1, n)
            self._add(kind, block_error(np.asarray(got[kind])[j, i].reshape(-1, n), hpb, yaw),
                      block_error(np.asarray(want[kind])[j, i].reshape(-1, n), hpb, yaw), [(ww, 0) for ww in w])
        return True

    # ---------------------------------------------------------------- verdict
    def arrays(self):
        kind = np.array(self.kind)
        e_got = np.concatenate(self.e_got) if self.e_got else np.zeros(0)
        e_ref = np.concatenate(self.e_ref) if self.e_ref else np.zeros(0)
        return kind, e_got, e_ref

    def failures(self):
        """[(kind, (where, track), model, e_got, e_ref)] of the blocks that fail the bar (excluded blocks left out)"""
        kind, e_got, e_ref = self.arrays()
        bad = ~passes(e_got, e_ref, self.C, self.F) & ~(e_ref > CEIL)
        return [(kind[i], self.where[i][0], self.where[i][1], float(e_got[i]), float(e_ref[i])) for i in np.nonzero(bad)[0]]

    def report(self, label="e_got"):
        kind, e_got, e_ref = self.arrays()
        excl = e_ref > CEIL
        lines = [f"{self.name}: {self.steps} steps ({self.excluded_steps} excluded: decisions of hp != reference), {len(e_got)} blocks "
                 f"({int(excl.sum())} excluded: e_ref > {CEIL:g}); bar e <= max({self.C:g} e_ref, {self.F:.3g}), <= {CEIL:g}"]
        q = lambda a: "-" if a.size == 0 else f"{np.median(a):.2e} / {np.quantile(a, 0.99):.2e} / {a.max():.2e}"
        for k in sorted(set(self.kind), key=lambda k: (KINDS + tuple(p[0] for p in PRED_BLOCKS)).index(k)):
            s = (kind == k) & ~excl
            r = e_ref[s] > 0
            ratio = e_got[s][r] / e_ref[s][r]
            lines.append(f"  {k:9s} {label} median/p99/max {q(e_got[s])}   e_ref {q(e_ref[s])}   {label}/e_ref {q(ratio)}"
                         f"   (e_ref = 0 on {int((~r).sum())})")
        if len(e_got):
            ok = np.nonzero(~excl)[0]
            i = ok[np.argmax(e_got[ok])] if len(ok) else 0
            lines.append(f"  worst block: {kind[i]} model {self.where[i][1]} at {self.where[i][0]}, {label} {e_got[i]:.3g}, "
                         f"e_ref {e_ref[i]:.3g}")
        if self.float_outputs:
            lines.append(f"  float outputs: {self.float_not_equal} of {self.float_outputs} not bit-equal to the reference, worst "
                         f"{self.float_worst_ulp} ulp")
        print("\n".join(lines))

    def check(self, max_excluded_steps=0):
        self.report()
        kind, e_got, e_ref = self.arrays()
        assert len(e_got) > 0, self.name
        fails = self.failures()
        assert not fails, (self.name, len(fails), sorted(fails, key=lambda f: -f[3])[:10])
        share = float((e_ref > CEIL).mean())
        assert share <= EXCLUDED_SHARE, (self.name, "excluded blocks", share)
        assert self.excluded_steps <= max_excluded_steps, (self.name, "excluded steps", self.excluded_steps)
        assert self.float_worst_ulp <= 1, (self.name, "float outputs", self.float_worst_ulp)
