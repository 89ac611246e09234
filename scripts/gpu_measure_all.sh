#!/bin/bash
# One session on the GPU that measures a build: tests, sweeps, bench lines (default, 20 steps, reference arm) and the tracker
# timeline from a torch.profiler trace.  Output: measure_out/<tag>_*
#   bash scripts/gpu_measure_all.sh <tag>
T=${1:-run}
mkdir -p measure_out
timeout 900 python -m pytest tests -m gpu -x -q > measure_out/${T}_pytest.log 2>&1; tail -3 measure_out/${T}_pytest.log
timeout 240 python scripts/detect_sweep.py > measure_out/${T}_sweep.txt 2>&1; tail -4 measure_out/${T}_sweep.txt
timeout 600 python bench.py > measure_out/${T}_bench.json 2> measure_out/${T}_bench.err; tail -2 measure_out/${T}_bench.err
timeout 400 python bench.py --steps 20 --warmup 5 > measure_out/${T}_bench_k20.json 2> measure_out/${T}_bench_k20.err
timeout 300 python bench.py --impl reference --steps 20 --warmup 5 > measure_out/${T}_bench_ref.json 2>/dev/null
timeout 600 python scripts/seq_measure.py > measure_out/${T}_seq.txt 2>&1; tail -9 measure_out/${T}_seq.txt
timeout 600 python scripts/seq_rig_measure.py > measure_out/${T}_seq_rig.txt 2>&1; tail -7 measure_out/${T}_seq_rig.txt
timeout 600 python scripts/seq_track_measure.py > measure_out/${T}_seq_track.txt 2>&1; tail -11 measure_out/${T}_seq_track.txt
timeout 600 python scripts/tracker_params_measure.py > measure_out/${T}_tracker_params.txt 2>&1; tail -9 measure_out/${T}_tracker_params.txt
timeout 600 python scripts/seq_detect_params_measure.py > measure_out/${T}_seq_detect_params.txt 2>&1; tail -6 measure_out/${T}_seq_detect_params.txt
timeout 900 python scripts/retire_measure.py > measure_out/${T}_retire.txt 2>&1; tail -30 measure_out/${T}_retire.txt
timeout 900 python scripts/predict_measure.py > measure_out/${T}_predict.txt 2>&1; tail -16 measure_out/${T}_predict.txt
timeout 600 python scripts/seq_tick_measure.py > measure_out/${T}_seq_tick.txt 2>&1; tail -3 measure_out/${T}_seq_tick.txt
timeout 600 python scripts/deskew_measure.py > measure_out/${T}_deskew.txt 2>&1; tail -2 measure_out/${T}_deskew.txt
timeout 600 python scripts/rig_merge_measure.py > measure_out/${T}_rig_merge.txt 2>&1; tail -3 measure_out/${T}_rig_merge.txt
timeout 600 python scripts/box_search_measure.py > measure_out/${T}_box_search.txt 2>&1; tail -3 measure_out/${T}_box_search.txt
timeout 600 python scripts/ground_lines_measure.py > measure_out/${T}_ground_lines.txt 2>&1; tail -3 measure_out/${T}_ground_lines.txt
timeout 900 python scripts/layers_measure.py > measure_out/${T}_layers.txt 2>&1; tail -3 measure_out/${T}_layers.txt
timeout 900 python scripts/obstacles_measure.py > measure_out/${T}_obstacles.txt 2>&1; tail -3 measure_out/${T}_obstacles.txt
timeout 600 python scripts/ego_match_measure.py --out measure_out/${T}_ego_match.json > measure_out/${T}_ego_match.txt 2>&1; tail -3 measure_out/${T}_ego_match.txt
timeout 300 python scripts/diag_timeline.py ${T}_timeline > measure_out/${T}_timeline.txt 2>&1; tail -5 measure_out/${T}_timeline.txt
ls -la measure_out/${T}*
