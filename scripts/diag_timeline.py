"""Diagnostic: the tracker chain of the frame pipeline, from a torch.profiler trace.

K pipelined lmot_frame_dev steps in production mode (timing events off, frames resident on the device) are traced with CUDA
activities only: every kernel's start and end, nothing added to the streams.  The trace goes to measure_out/<tag>.pt.trace.json.
Printed, as the mean over the K steps in us: TA = imm_predict_gate_kernel, TB = imm_update_kernel, TC = spawn_output_kernel, the
gaps between them (negative: the programmatic dependent's CTAs were resident before its predecessor ended), TA start to the next
TA start (the chain's period, which bounds frames/s), and detection start (ground_fused_kernel) to box_fit_kernel end.  Then the
same loop runs without the profiler, timed with CUDA events: tracing lengthens every step, so the trace gives the chain's shape
and this last line its production length.

    python scripts/diag_timeline.py [tag]        # DIAG_K = steps (default 200)
"""
import importlib, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                     # (sets CUDA_DEVICE_MAX_CONNECTIONS before CUDA initialises)
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

if not torch.cuda.is_available():
    raise SystemExit("diag_timeline.py: no CUDA device -- the timeline is measured on the GPU only")
lmot = importlib.import_module(bench.PKG)
synth = importlib.import_module(bench.PKG + ".synth")
tag = sys.argv[1] if len(sys.argv) > 1 else "timeline"
K, W = int(os.environ.get("DIAG_K", "200")), 20
ts, frames = bench.make_frames(synth, W + K)
n = frames.shape[1]
d = torch.from_numpy(frames).cuda()
ctx = lmot.Lmot(lmot.default_params())
st = torch.cuda.Stream(); torch.cuda.set_stream(st); ctx.set_stream(st.cuda_stream)
clock = bench.ClockSampler(torch.cuda.current_device()); clock.start()


def steps(lo, hi):
    for i in range(lo, hi):
        ctx.frame_dev(d[i].data_ptr(), n, ts[i])
    ctx.flush()


def warm_up():
    ctx.tracker_reset(); steps(0, W); torch.cuda.synchronize()


warm_up()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    steps(W, W + K); torch.cuda.synchronize()
os.makedirs(os.path.join(ROOT, "measure_out"), exist_ok=True)
path = os.path.join(ROOT, "measure_out", f"{tag}.pt.trace.json")
prof.export_chrome_trace(path)
kern = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
span = {k: np.array(sorted((e["ts"], e["ts"] + e["dur"]) for e in kern if k in e["name"])).reshape(-1, 2)
        for k in ("ground_fused_kernel", "box_fit_kernel", "imm_predict_gate_kernel", "imm_update_kernel", "spawn_output_kernel")}
if any(len(v) != K for v in span.values()):
    raise SystemExit(f"diag_timeline.py: expected {K} launches of each kernel in {path}, found {({k: len(v) for k, v in span.items()})}")
ta, tb, tc = span["imm_predict_gate_kernel"], span["imm_update_kernel"], span["spawn_output_kernel"]
det, fit = span["ground_fused_kernel"], span["box_fit_kernel"]

warm_up()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(st); steps(W, W + K); e1.record(st); torch.cuda.synchronize()
ms = e0.elapsed_time(e1)
clk = clock.stop()
ctx.close()

m = lambda x: f"{np.mean(x):.1f}"
print(f"{torch.cuda.get_device_name()}, power limit {clk['power_limit_w']} W, median SM clock {clk['sm_mhz']} MHz; "
      f"{K} pipelined steps, pipeline_depth {lmot.default_params().pipeline_depth}, trace {os.path.relpath(path, ROOT)}")
print(f"tracker chain per step, mean (us): TA {m(ta[:, 1] - ta[:, 0])} | gap {m(tb[:, 0] - ta[:, 1])} | TB {m(tb[:, 1] - tb[:, 0])} | "
      f"gap {m(tc[:, 0] - tb[:, 1])} | TC {m(tc[:, 1] - tc[:, 0])} | gap to the next TA {m(ta[1:, 0] - tc[:-1, 1])}")
print(f"  TA start to next TA start {m(np.diff(ta[:, 0]))} us; detection start -> box_fit_kernel end {m(fit[:, 1] - det[:, 0])} us")
print(f"no profiler: {K / (ms * 1e-3):.0f} frames/s ({1e3 * ms / K:.1f} us/frame), CUDA events around the {K} steps")
