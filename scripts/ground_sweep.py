"""Diagnostic (not part of the bench contract): device time of the ground stage alone vs frame size and CTA count.
Each (size, LMOT_PTS_PER_CTA) point: ring of frames larger than L2, CUDA events on the launching stream."""
import importlib, json, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = "3d-lidar-multi-object-tracking_b200"
lmot = importlib.import_module(PKG)
synth = importlib.import_module(PKG + ".synth")

peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
out = []
sizes = [("hdl64_120k", synth.SceneConfig(n_objects=150, lattice_pitch=3.8, ped_fraction=0.65, seed=1), 120000, 80),
         ("dense_1m", synth.dense_config(n_objects=150, lattice_pitch=3.8, ped_fraction=0.65, seed=7), 1000000, 10)]
ppcs = [int(x) for x in os.environ.get("SWEEP_PPC", "1024,2048,4096,8192").split(",")]
for name, cfg, n, ring in sizes:
    fr = [p[:n] for _, p in synth.frames(cfg, ring)]
    d = torch.from_numpy(np.stack(fr)).cuda()
    for ppc in ppcs:
        os.environ["LMOT_PTS_PER_CTA"] = str(ppc)
        prm = lmot.default_params(); prm.pipeline_depth = 1
        ctx = lmot.Lmot(prm)
        st = torch.cuda.Stream(); torch.cuda.set_stream(st); ctx.set_stream(st.cuda_stream)
        for i in range(5):
            ctx.ground_remove_dev(d[i % ring].data_ptr(), n)
        torch.cuda.synchronize()
        reps = 4 * ring
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for i in range(reps):
            ctx.ground_remove_dev(d[i % ring].data_ptr(), n)
        e1.record(st); torch.cuda.synchronize()
        us = 1e3 * e0.elapsed_time(e1) / reps
        r = ctx.ground_remove(fr[0])
        nf = len(r["elevated"]) + len(r["ground"])
        b = 16 * n + 16 * nf + 9600 * 24
        out.append(dict(size=name, pts_per_cta=ppc, us_per_launch=us, gbs=b / us / 1e3, frac=b / us / 1e3 / peak))
        print(json.dumps(out[-1]), flush=True)
        ctx.close()
    del d
