"""The detection front end's configuration matrix (numpy only, no device): every combination of per-stream settings a sequence tick can
mix, tick layouts that put every two of them into one tick, and a plain restatement of which kernels the front end launches for a tick.

A FRAMES stream's configuration is (table, own detection values, deskew):
  * table: "none" (one frame per step), "sep" (a sensor table, each sensor's boxes moved into the vehicle frame), "merge" (a sensor
    table whose elevated clouds are clustered and boxed as one vehicle-frame cloud);
  * own: lmot_seq_set_detect_params with OWN, which moves sensor_height, the ground window, h_sensor and min_cluster_points, so a
    stream that silently fell back to lmot_params (or took another stream's values) gets other boxes;
  * dsk: lmot_seq_set_deskew(on=1), the time of every point in its fourth float.
The front end decides tick-wide (csrc/api.cu, detect_front / seq_tick_common) which kernel variant every launch gets, as an OR over the
tick's FRAMES streams; `launch_rule` restates that decision so the tests can check it by kernel name.

A layout is a set of sequences (at most 8 frames per step over all of them, lmot_seq_set_sensors) and a schedule: per tick and sequence
one code -- "F" frames, "R" frames and LMOT_SEQ_RESTART, "e" frames with sensor 1's frame empty (a table) or the one frame empty (none),
"E" frames all empty, "L" box lists, "-" skip.
"""
import itertools
import re

import numpy as np

f32 = np.float32

TABLES = ("none", "sep", "merge")
# own detection values: ground window and mount height moved (a table's sensor values replace those four), the box-fitting reference
# height moved, small clusters kept, a narrower width gate
OWN = dict(sensor_height=1.6, h_sensor=2.2, t_hmin=-2.3, t_hmax=-0.6, min_cluster_points=4, t_width_max=2.2)
H_VEHICLE = 2.0                                  # lmot_params.sensor_height of every context here: the vehicle frame's origin height
HEIGHTS = [2.0, 1.2, 0.8, 1.8, 1.6, 1.0, 2.2, 1.4]
MAX_FRAMES = 8
FRAME_CODES = set("FReE")


def config_name(table, own, dsk):
    return table + ("+own" if own else "") + ("+dsk" if dsk else "")


def _sensors(table, own, dsk):
    """sensor count: separate rigs of 2 or 3, merging rigs of 3 (quarter-turn yaws: overlapping fields of view) or 2"""
    if table == "none":
        return 0
    if table == "sep":
        return 3 if (dsk and not own) else 2
    return 2 if own else 3


CONFIGS = {config_name(t, o, d): dict(table=t, own=bool(o), dsk=bool(d), n_sensors=_sensors(t, o, d))
           for t in TABLES for o in (0, 1) for d in (0, 1)}


def frames_of(name):
    """frames the sequence sends per FRAMES step (1 without a table)"""
    return max(CONFIGS[name]["n_sensors"], 1)


# every two configurations share a layout (and its all-FRAMES first tick); each layout fills at most MAX_FRAMES frames
LAYOUTS = [
    ["none+own+dsk", "sep", "sep+dsk", "merge+own+dsk"],
    ["none+own", "sep+own+dsk", "merge+dsk", "merge+own"],
    ["none", "none+own+dsk", "merge", "merge+dsk"],
    ["none", "none+dsk", "sep+own", "sep+own+dsk", "merge+own+dsk"],
    ["none+dsk", "sep", "merge", "merge+own"],
    ["none+own", "sep+own", "merge", "merge+own+dsk"],
    ["none+dsk", "none+own", "sep+dsk", "merge+dsk"],
    ["sep+dsk", "sep+own+dsk", "merge"],
    ["none", "none+dsk", "none+own", "none+own+dsk", "sep", "sep+own+dsk"],
    ["none", "sep+dsk", "sep+own", "merge+own"],
    ["none+own+dsk", "sep", "sep+own", "merge+dsk"],
    ["none+own+dsk", "merge+dsk", "merge+own", "merge+own+dsk"],
]


def schedule(layout):
    """the layout's ticks: per tick one code per sequence (see the module docstring).  Tick 0 steps everyone from frames; the others
    step subsets, so that the tick-wide switches take both states: only the tableless streams' frames, only the merging streams',
    alternating frames / lists / skips, a restart, an empty frame inside every rig, and a tick whose frames are all empty."""
    tab = [CONFIGS[n]["table"] for n in layout]
    n = len(layout)
    ticks = [["F"] * n,
             ["F" if k % 2 == 0 else "L" for k in range(n)],
             ["F" if t == "none" else ("L" if k % 2 else "-") for k, t in enumerate(tab)],
             ["F" if t == "merge" else ("L" if t == "none" else "-") for t in tab],
             ["F" if k % 2 else "-" for k in range(n)],
             ["e" if t != "none" else "F" for t in tab],
             ["R"] + ["F"] * (n - 1),
             ["E" if k % 2 == 0 else "L" for k in range(n)],
             ["F" if t == "sep" else ("F" if t == "none" and k % 2 else "L") for k, t in enumerate(tab)]]
    # a tick needs a stepped sequence; one without any FRAMES entry steps everyone from lists
    return [tk if any(c != "-" for c in tk) else ["L"] * n for tk in ticks]


# a merging rig whose merged cloud exceeds max_points (test_rig_merge_gpu.test_merged_cloud_above_max_points): 7 sensors + one
# tableless stream, every frame below max_points
OVER_MAX = dict(layout=["merge7", "none"], sensors=7, seed=61, view_seed=62, ticks=[["F", "F"], ["F", "L"], ["L", "F"], ["F", "F"]])


# ------------------------------------------------------------------------------------------------ the switch rule
def switches(cfgs, gf):
    """the front end's tick-wide switches for the configurations of a tick's FRAMES entries (in sequence order)"""
    c = [CONFIGS[n] for n in cfgs]
    return dict(rigged=any(x["table"] != "none" for x in c), own_det=any(x["own"] for x in c),
                merging=any(x["table"] == "merge" for x in c), deskew=any(x["dsk"] for x in c),
                rig_fit=any(x["table"] == "sep" for x in c), gf=bool(gf))


def launch_rule(cfgs, gf, empty=(), lists=False):
    """the front end's launches of one tick, by kernel, as a sorted list of names -- the ground kernel (with the pose table iff some
    stream has a sensor table, with per-frame values iff some stream has its own), CCL apart from it iff some stream merges, the merge,
    deskew iff some deskewing stream sent a point (`empty`: the entries whose frames are all empty), box fitting's segment pass
    (seg_offsets_kernel when no unit has a point, else the tile histogram and the scatter), its fit kernel (per-frame values iff some stream has its own, else the pose table's sensor heights iff some unit is an
    unmerged frame of a separate rig), the per-sequence concatenation iff some FRAMES stream has a table, the global-frame step iff
    global_frame, the pack of the LISTS entries."""
    out = []
    all_empty = bool(cfgs) and set(cfgs) <= set(empty)
    if cfgs:
        s = switches(cfgs, gf)
        out.append("ground_fused_frame_kernel" if s["own_det"] else "ground_fused_rig_kernel" if s["rigged"] else "ground_fused_kernel")
        if s["merging"]:
            out += ["rig_merge_kernel", "ccl_dense_kernel"]
        if any(CONFIGS[n]["dsk"] and n not in empty for n in cfgs):
            out.append("deskew_points_kernel")
        out += ["seg_offsets_kernel"] if all_empty else ["tile_hist_kernel", "scatter_kernel"]
        out.append("box_fit_frame_kernel" if s["own_det"] else "box_fit_kernel<true>" if s["rig_fit"] else "box_fit_kernel<false>")
        if s["rigged"]:
            out.append("concat_boxes_seq_kernel")
    if gf:
        out.append("boxes_to_global_seq_kernel")
    if lists:
        out.append("pack_lists_seq_kernel")
    return sorted(out)


FRONT_KERNELS = ("ground_fused", "rig_merge_kernel", "ccl_dense_kernel", "deskew_points_kernel", "seg_offsets_kernel", "tile_hist_kernel",
                 "scatter_kernel", "box_fit", "concat_boxes_seq_kernel", "boxes_to_global_seq_kernel", "pack_lists_seq_kernel")


def kernel_key(name):
    """a profiler kernel name -> the name launch_rule uses (None: not a front-end kernel).  box_fit_kernel keeps its bool argument."""
    for m in re.finditer(r"\w+", name):
        base = m.group(0)
        if not base.startswith(FRONT_KERNELS):
            continue
        if base == "box_fit_kernel":
            args = name[m.end():].split(">")[0]
            assert "true" in args or "false" in args, name
            return "box_fit_kernel<true>" if "true" in args else "box_fit_kernel<false>"
        return base
    return None


def tick_cfgs(layout, tick):
    """(configurations of the tick's FRAMES entries, those of them whose frames are all empty, whether it has LISTS entries)"""
    cf = [n for n, c in zip(layout, tick) if c in FRAME_CODES]
    return cf, [n for n, c in zip(layout, tick) if c == "E"], "L" in tick


def all_empty(cfgs, empty):
    return bool(cfgs) and set(cfgs) <= set(empty)


def all_ticks():
    """(layout index, tick index, layout, tick) over the matrix"""
    for i, lay in enumerate(LAYOUTS):
        for t, tk in enumerate(schedule(lay)):
            yield i, t, lay, tk


def switch_states():
    """every distinct (switch state, all frames empty) of the matrix's ticks under global_frame 0 and 1 -> the first (layout, tick)"""
    seen = {}
    for gf in (0, 1):
        for i, t, lay, tk in all_ticks():
            cf, empty, _ = tick_cfgs(lay, tk)
            if not cf:
                continue
            key = (tuple(sorted(switches(cf, gf).items())), all_empty(cf, empty))
            seen.setdefault(key, (i, t, gf))
    return seen


# ------------------------------------------------------------------------------------------------ scenes
def quarter_rig(n, heights, h_vehicle=H_VEHICLE):
    """rig_merge_scenes.overlap_rig without the reference import: n sensors yawed by quarter turns (n = 2: 0 and pi), mounted at heights"""
    from rig_merge_scenes import overlap_rig
    return overlap_rig(n, heights=heights, h_vehicle=h_vehicle)


def timed(p):
    """stride-4 records with the deskew time (seconds before the stamp, -0.1 .. 0 over the record order) in the fourth float"""
    q = np.zeros((len(p), 4), f32)
    q[:, :3] = p[:, :3]
    if len(p):
        q[:, 3] = (-0.1 * (np.arange(len(p)) / len(p))).astype(f32)
    return q


def stream_ts(k, t):
    return 1.0e6 + 7000.0 * k + 100000.0 * t


def stream_ego(k, t):
    """a moving, turning vehicle per stream (deskew has something to undo)"""
    return 5.0 + 0.7 * k + 0.3 * t, 0.05 * k + 0.03 * t + 0.002 * t * t * (1 if k % 2 else -1)


def some_boxes(k, t, n=3):
    b = np.zeros((n, 8, 3), f32)
    for i in range(n):
        cx, cy = 8.0 + 4 * i + 0.3 * t + k, -6.0 + 5 * i
        b[i, :, 0] = cx + np.array([1, 1, -1, -1, 1, 1, -1, -1], f32)
        b[i, :, 1] = cy + np.array([0.5, -0.5, -0.5, 0.5] * 2, f32)
        b[i, :, 2] = np.array([-1.7] * 4 + [-0.2] * 4, f32)
    return b


class Stream:
    """sequence k of a layout: its configuration, rig (rig_merge_scenes.overlap_rig: [(pose, h, quarter)], None without a table) and
    per tick its frames (stride 4, deskew time in the fourth float) from the overlapping scene: a rig's sensors see one vehicle view,
    so objects in their overlaps reach two sensors"""

    def __init__(self, synth, name, k, n_ticks, seed, n_sensors=None, rings=32):
        from rig_merge_scenes import overlap_ticks
        self.name, self.k = name, k
        c = CONFIGS.get(name, dict(table="merge", own=False, dsk=False))
        self.table, self.own, self.dsk = c["table"], c["own"], c["dsk"]
        n = n_sensors or c.get("n_sensors", 0)
        if self.table == "none":
            self.rig = None
            cfg = synth.SceneConfig(seed=seed, rings=rings, azimuths=900, n_objects=30)
            self.frames = [[timed(p)] for _, p in synth.frames(cfg, n_ticks)]
        else:
            self.rig = quarter_rig(n, HEIGHTS[k % 3: k % 3 + n] if n <= 5 else HEIGHTS[:n])
            self.frames = [[timed(p) for p in fr] for _, fr, _, _ in overlap_ticks(synth, self.rig, n_ticks, seed=seed)]

    def ts(self, t):
        return stream_ts(self.k, t)

    def ego(self, t):
        return stream_ego(self.k, t)

    def frames_for(self, t, code):
        """the frames sent at tick t for a FRAMES code"""
        fr = list(self.frames[t])
        if code == "E":
            fr = [np.zeros((0, 4), f32) for _ in fr]
        elif code == "e":
            fr[1 if len(fr) > 1 else 0] = np.zeros((0, 4), f32)
        return fr

    def lists_for(self, t):
        return [some_boxes(self.k, t + j) for j in range(len(self.frames[t]))]


def pairs_covered():
    """the configuration pairs that share at least one tick as FRAMES entries"""
    got = set()
    for _, _, lay, tk in all_ticks():
        cf, _, _ = tick_cfgs(lay, tk)
        got |= {tuple(sorted(p)) for p in itertools.combinations(cf, 2)}
    return got
