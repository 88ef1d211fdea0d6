#!/bin/bash
# bash tools/tp_round.sh N : tensor-parallel parity tests and bench lines on N GPUs of one machine; outputs land in results/
N=${1:-2}
mkdir -p results
set -x
nvidia-smi -L | head -8
KSEL=""
if [ "$N" = "8" ]; then KSEL="tp8-8 or moe-8"; fi   # the world-2 / world-4 cases have their own runs (8 GPUs are charged 8x)
timeout 1200 python -m pytest tests/test_tp_gpu.py -q -rs -x ${KSEL:+-k "$KSEL"} > results/pytest_tp${N}.log 2>&1; tail -12 results/pytest_tp${N}.log
run() { timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $((29500 + RANDOM % 400)) bench.py --gpus $N "$@"; }
run --steps 64 --warmup 8 > results/bench_tp${N}_llama3-8b-fp8.jsonl 2> results/bench_tp${N}_8b.err; tail -c 1500 results/bench_tp${N}_llama3-8b-fp8.jsonl; tail -3 results/bench_tp${N}_8b.err
run --steps 32 --warmup 4 --workload llama3-70b-fp8 > results/bench_tp${N}_llama3-70b-fp8.jsonl 2> results/bench_tp${N}_70b.err; tail -c 1500 results/bench_tp${N}_llama3-70b-fp8.jsonl; tail -3 results/bench_tp${N}_70b.err
if [ "$N" = "2" ] && [ -n "$EXTRA" ]; then
  run --steps 64 --warmup 8 --parallel replicas > results/bench_replicas${N}_llama3-8b-fp8.jsonl 2>> results/bench_tp${N}_8b.err; tail -c 600 results/bench_replicas${N}_llama3-8b-fp8.jsonl
  run --steps 32 --warmup 4 --workload mixtral-8x7b-fp8 > results/bench_tp${N}_mixtral-8x7b-fp8.jsonl 2> results/bench_tp${N}_mx.err; tail -c 800 results/bench_tp${N}_mixtral-8x7b-fp8.jsonl; tail -3 results/bench_tp${N}_mx.err
fi
