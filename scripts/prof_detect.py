"""Workload for `ncu` captures of the detection kernels: 4 stand-alone ground launches on dense 1 M-point frames, then 3 batched
ticks (8 x 120 k: ground, CCL, counting sort, box fitting) without the tracker.
  ncu --set full --import-source on --clock-control none -k regex:"ground_fused|ccl_|box_fit" --launch-skip 2 -c 8 -o measure_out/r2_detect python scripts/prof_detect.py"""
import importlib, os, sys
os.environ.setdefault("LMOT_FUSE_CCL", "0")     # profile clustering as its own kernel
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = "3d-lidar-multi-object-tracking_b200"
lmot = importlib.import_module(PKG)
synth = importlib.import_module(PKG + ".synth")
SCENE = dict(n_objects=150, lattice_pitch=3.8, ped_fraction=0.65)
fr = [p[:1_000_000] for _, p in synth.frames(synth.dense_config(seed=7, **SCENE), 2)]
d = torch.from_numpy(np.stack(fr)).cuda()
prm = lmot.default_params(); prm.pipeline_depth = 1
ctx = lmot.Lmot(prm)
for i in range(4):
    ctx.ground_remove_dev(d[i % 2].data_ptr(), 1_000_000)
ctx.sync()
F = 8
streams = [[p for _, p in synth.frames(synth.SceneConfig(seed=1 + s, **SCENE), 3)] for s in range(F)]
dev = [[torch.from_numpy(p).cuda() for p in st] for st in streams]
for t in range(3):
    ctx.batch_detect_dev([(dev[s][t].data_ptr(), len(streams[s][t])) for s in range(F)])
    ctx.batch_fetch()
ctx.close()
