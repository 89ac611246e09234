"""Diagnostic: does the footprint of the mostly-idle tracker / box-fit grids limit the frame pipeline?  Device-resident frames,
host never blocking; frames/s for a few grid sizes and pipeline depths."""
import importlib, json, os, sys, time
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
lmot = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
import bench
K, W = 300, 20
ts, frames = bench.make_frames(synth, W + K)
n = frames.shape[1]
d = torch.from_numpy(frames).cuda()
torch.cuda.synchronize()
for coop, trk, fit in ((1, 528, 264), (0, 528, 264), (0, 132, 132)):
    os.environ["LMOT_TRK_CTAS"] = str(trk); os.environ["LMOT_FIT_CTAS"] = str(fit); os.environ["LMOT_COOP"] = str(coop)
    for depth in (1, 2, 4, 8):
        prm = lmot.default_params(); prm.pipeline_depth = depth
        ctx = lmot.Lmot(prm)
        st = torch.cuda.Stream(); torch.cuda.set_stream(st); ctx.set_stream(st.cuda_stream)
        ctx.tracker_reset()
        for i in range(W): ctx.frame_dev(d[i].data_ptr(), n, ts[i])
        torch.cuda.synchronize(); ctx.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter(); e0.record(st)
        for i in range(W, W + K): ctx.frame_dev(d[i].data_ptr(), n, ts[i])
        th = time.perf_counter() - t0
        ctx.flush(); e1.record(st); torch.cuda.synchronize()
        print(json.dumps(dict(coop=coop, trk_ctas=trk, fit_ctas=fit, depth=depth, fps=K / (e0.elapsed_time(e1) * 1e-3), host_submit_us=1e6 * th / K)), flush=True)
        ctx.frame_fetch(); ctx.close()
