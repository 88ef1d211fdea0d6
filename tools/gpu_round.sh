#!/bin/bash
# bash tools/gpu_round.sh : the end-to-end verification on one H100 (full GPU test suite, smoke, default bench line, gf4 bench
# line); outputs land in results/.
mkdir -p results
set -x
timeout 900 python -m pytest tests -q -m gpu 2>&1 | grep -v "^# CUDA" > results/pytest_gpu_final.log; tail -3 results/pytest_gpu_final.log
timeout 120 python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" 2>&1 | tail -2
timeout 600 python bench.py > results/bench_final.jsonl 2> results/bench_final.err; cut -c1-1500 results/bench_final.jsonl; tail -2 results/bench_final.err
timeout 400 python bench.py --workload mistral-7b-gf4 > results/bench_gf4_final.jsonl 2> results/bench_gf4_final.err; cut -c1-600 results/bench_gf4_final.jsonl
