#!/bin/bash
# One session on the GPU that measures a build: tests, phase stamps, sweeps, bench lines (default, 20 steps, reference arm),
# tracker timeline, ncu launch list, ncu --set full of the detection kernels and the tracker chain.  Output: measure_out/<tag>_*
#   bash scripts/gpu_measure_all.sh <tag>
T=${1:-run}
mkdir -p measure_out
timeout 900 python -m pytest tests -m gpu -x -q > measure_out/${T}_pytest.log 2>&1; tail -3 measure_out/${T}_pytest.log
timeout 240 python scripts/ground_phases.py > measure_out/${T}_phases.txt 2>&1
timeout 240 python scripts/detect_sweep.py > measure_out/${T}_sweep.txt 2>&1; tail -4 measure_out/${T}_sweep.txt
timeout 600 python bench.py > measure_out/${T}_bench.json 2> measure_out/${T}_bench.err; tail -2 measure_out/${T}_bench.err
timeout 400 python bench.py --steps 20 --warmup 5 > measure_out/${T}_bench_k20.json 2> measure_out/${T}_bench_k20.err
timeout 300 python bench.py --impl reference --steps 20 --warmup 5 > measure_out/${T}_bench_ref.json 2>/dev/null
DIAG_K=200 DIAG_DEPTHS=1,8 timeout 300 python scripts/diag_timeline.py > measure_out/${T}_timeline.txt 2>&1; tail -5 measure_out/${T}_timeline.txt
SMALL="--steps 10 --warmup 3 --cpu-sample 0 --dense-frames 0 --tracker-stress 0 --batch-ticks 0"
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 500 --csv --log-file measure_out/${T}_launches.csv python bench.py $SMALL > /dev/null 2>&1
timeout 300 ncu --set full --import-source on --clock-control none -k regex:ground_fused -s 8 -c 2 -f -o measure_out/${T}_ground_pipeline python bench.py $SMALL > /dev/null 2>&1
LMOT_FUSE_CCL=1 timeout 400 ncu --set full --import-source on --clock-control none -k regex:"ground_fused|tile_hist|scatter|box_fit|concat" --launch-skip 3 -c 6 -f -o measure_out/${T}_detect_fused python scripts/prof_detect.py > measure_out/${T}_ncu.log 2>&1; grep Profiling measure_out/${T}_ncu.log | head
timeout 500 ncu --set full --import-source on --warp-sampling-interval 0 --clock-control none -k regex:"imm_|spawn_output|tracker_gate|publish_kernel" -s 600 -c 10 -f -o measure_out/${T}_tracker python bench.py --steps 200 --warmup 20 --cpu-sample 0 --dense-frames 0 --tracker-stress 0 --batch-ticks 0 > /dev/null 2>&1
ls -la measure_out/${T}*
