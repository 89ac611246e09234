"""Diagnostic (not the bench contract): device time of the streaming detection kernels, CUDA events on the launching stream,
inputs cycling through a ring larger than the 50 MB L2:
  ground_fused_kernel alone on 120 k / 1 M-point frames, and the batched tick (8 x 120 k): ground + CCL as two launches."""
import importlib, json, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = "3d-lidar-multi-object-tracking_b200"
lmot = importlib.import_module(PKG)
synth = importlib.import_module(PKG + ".synth")
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
SCENE = dict(n_objects=150, lattice_pitch=3.8, ped_fraction=0.65)


def timed(fn, reps, st):
    for i in range(5):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for i in range(reps):
        fn(i)
    e1.record(st); torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / reps


st = torch.cuda.Stream(); torch.cuda.set_stream(st)
for name, cfg, n, ring in (("hdl64_120k", synth.SceneConfig(seed=1, **SCENE), 120000, 80), ("dense_1m", synth.dense_config(seed=7, **SCENE), 1000000, 10)):
    fr = [p[:n] for _, p in synth.frames(cfg, ring)]
    d = torch.from_numpy(np.stack(fr)).cuda()
    prm = lmot.default_params(); prm.pipeline_depth = 1
    ctx = lmot.Lmot(prm); ctx.set_stream(st.cuda_stream)
    us = timed(lambda i: ctx.ground_remove_dev(d[i % ring].data_ptr(), n), 4 * ring, st)
    r = ctx.ground_remove(fr[0])
    nf = len(r["elevated"]) + len(r["ground"])
    b = 16 * n + 16 * nf + 9600 * 24
    print(json.dumps(dict(case=name + " ground stand-alone", us_per_launch=us, gbs=b / us / 1e3, frac=b / us / 1e3 / peak)), flush=True)
    ctx.close(); del d

F, ring = 8, 12
streams = [[p for _, p in synth.frames(synth.SceneConfig(seed=1 + s, **SCENE), ring)] for s in range(F)]
dev = [torch.from_numpy(np.stack(s_)).cuda() for s_ in streams]
ctx = lmot.Lmot(); ctx.set_stream(st.cuda_stream)
n = 120000
prep = [ctx.batch_prepare([(dev[s][t].data_ptr(), n) for s in range(F)]) for t in range(ring)]
us = timed(lambda i: ctx.batch_ground_ccl_dev(prep[i % ring]), 5 * ring, st)
ne = nf = 0
for s in range(F):
    r = ctx.ground_remove(streams[s][0]); ne += len(r["elevated"]); nf += len(r["elevated"]) + len(r["ground"])
bg = F * (16 * n + 9600 * 24) + 16 * nf
bc = 20 * ne + F * 2 * 62500 * 4
print(json.dumps(dict(case=f"batched tick {F} x 120 k: ground + CCL (one launch unless LMOT_FUSE_CCL=0)", us_per_tick=us, ground_bytes=bg, ccl_bytes=bc,
                      gbs=(bg + bc) / us / 1e3, frac=(bg + bc) / us / 1e3 / peak)), flush=True)
ctx.enable_timing(True)
ctx.tracker_reset()
km = []
for i in range(10):
    ctx.batch_dev(prep[i % ring], 1e5 * (i + 1))
    ctx.batch_fetch()
    km.append(ctx.last_kernel_ms())
print("batched tick kernels (us, event to event, timing mode):", [round(1e3 * x, 1) for x in np.mean(np.array(km[3:]), 0)], "stage ms:", ctx.last_stage_ms())
ctx.enable_timing(False)
ctx.close()
