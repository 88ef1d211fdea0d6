#!/usr/bin/env python
"""Time calm_b200_decode_sample_queue against the ways a host could run the same requests before it.  Prints one JSON line
(and appends it to the file --out names).

Workload M (mixed lengths): 64 requests, seeded prompt lengths uniform in [64, 512] and max_new uniform in [16, 256], no
stop tokens (random weights make stops arbitrary; the spread of max_new stands in for them).  Arms:
  queue        decode_sample_queue at max_rows 16
  waves        decode_sample_batch in input-order waves of 16, each with n_tokens = the wave's largest max_new, cut after
  sequential   forward_prefill_cuda + decode_sample per request
For each: useful tokens/s (sum of out_len over wall time, prompt passes included) and steps; for the queue also the mean
rows per step and, from one torch.profiler run of an engine without programmatic dependent launch, the device time by
kernel group (prompt pass: k_pf_gemm + k_pf_attn; steps: k_vf_gemm, k_sn_*, the sampler and the rest) and the prompt
pass's share.  outputs_equal: the queue's tokens equal the waves' cut tokens, checked in the same run.
Workload U (uniform): one wave of 16 requests with 256-token prompts and max_new 128: the queue against
decode_sample_batch, its overhead.
Each time is the best of --reps rounds with the arms alternating, after one warm-up of each, host clock around calls that
end in a device synchronise.  The sequential arm takes about half a minute a round and is timed in --seq-reps rounds.
Card name and power limit come from a query-only nvidia-smi in the same run.
  python tools/decode_sample_queue_bench.py [--workload llama3-8b-fp8] [--layers 32] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time
from dataclasses import replace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="llama3-8b-fp8")
ap.add_argument("--layers", type=int, default=None)
ap.add_argument("--seq-len", type=int, default=16384)
ap.add_argument("--t", type=float, default=1.0)
ap.add_argument("--p", type=float, default=0.1)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--seq-reps", type=int, default=2)
ap.add_argument("--nreq", type=int, default=64)
ap.add_argument("--out", default=None, help="a file to append the line to")
a = ap.parse_args()
os.environ.setdefault("CALM_B200_QUIET", "1")
ROWS = 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:  # noqa: BLE001 (no nvidia-smi: the line still carries the timings)
        return None, None


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def best_of(calls, rounds):
    """calls: {name: f}; every call once as warm-up, then rounds alternating (a call in rounds[name] rounds only)."""
    for f in calls.values():
        f()
    best = {k: 1e18 for k in calls}
    for r in range(a.reps):
        for k, f in calls.items():
            if r < rounds.get(k, a.reps):
                best[k] = min(best[k], timed(f)[0])
    return best


def kernel_split(f):
    """Device time of one call of f per kernel group, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        f()
        torch.cuda.synchronize()
    out = {"prompt_pass": 0.0, "k_vf_gemm": 0.0, "attention": 0.0, "sampler": 0.0, "other": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
        if t == 0.0 or e.key.startswith(("Memcpy", "Memset")):
            continue
        key = ("prompt_pass" if "k_pf_gemm" in e.key or "k_pf_attn" in e.key else "k_vf_gemm" if "k_vf_gemm" in e.key
               else "attention" if "k_sn_" in e.key else "sampler" if "k_sample" in e.key or "k_pf_logprob" in e.key else "other")
        out[key] += t
    return {k: round(v, 1) for k, v in out.items()}


spec = mg.SPECS[a.workload] if a.layers is None else replace(mg.SPECS[a.workload], n_layers=a.layers)
tensors = mg.generate(spec, 0, device="cuda")
torch.cuda.synchronize()
rng = np.random.default_rng(0)
seeds = [0x9E3779B97F4A7C15 + 7919 * i for i in range(a.nreq)]
result = {"workload": spec.name, "layers": spec.n_layers, "seq_len": a.seq_len, "temperature": a.t, "minp": a.p, "reps": a.reps, "seq_reps": a.seq_reps}

# ---- M: mixed lengths
lens = rng.integers(64, 513, a.nreq)
max_new = [int(x) for x in rng.integers(16, 257, a.nreq)]
prompts = [rng.integers(0, spec.vocab_size, int(n)).astype(np.int32) for n in lens]
T, P = [a.t] * a.nreq, [a.p] * a.nreq
waves = [range(w, min(w + ROWS, a.nreq)) for w in range(0, a.nreq, ROWS)]


def run_queue(dm):
    return dm.decode_sample_queue(prompts, max_new, T, P, [], ROWS, seeds)


def run_waves(dm):
    return [dm.decode_sample_batch([prompts[i] for i in w], max(max_new[i] for i in w), a.t, a.p, [seeds[i] for i in w])[0] for w in waves]


def run_sequential(dm):
    for p, m, s in zip(prompts, max_new, seeds):
        dm.prefill(p[:-1], 0)
        dm.decode_sample(int(p[-1]), len(p) - 1, m, a.t, a.p, s)


useful = sum(max_new)
with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    toks, _, served, steps = run_queue(dm)
    wt = run_waves(dm)
    cut = [wt[k][r][:max_new[i]] for k, w in enumerate(waves) for r, i in enumerate(w)]
    m = {"served": served, "useful_tokens": useful, "outputs_equal": all(np.array_equal(x, y) for x, y in zip(toks, cut))}
    t = best_of({"queue": lambda: run_queue(dm), "waves": lambda: run_waves(dm), "sequential": lambda: run_sequential(dm)}, {"sequential": a.seq_reps})
wave_steps = sum(max(max_new[i] for i in w) for w in waves)
m["ms"] = {k: round(v, 1) for k, v in t.items()}
m["useful_tps"] = {k: round(useful / v * 1e3, 1) for k, v in t.items()}
m["steps"] = {"queue": steps, "waves": wave_steps}
m["mean_rows_per_step"] = {"queue": round(useful / steps, 2), "waves": round(useful / wave_steps, 2)}
m["speedup_vs_waves"] = round(t["waves"] / t["queue"], 3)
m["speedup_vs_sequential"] = round(t["sequential"] / t["queue"], 3)
# the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its CTAs
# wait for the previous kernel to finish
os.environ["CALM_B200_PDL"] = "0"
try:
    with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
        run_queue(dm)
        split = kernel_split(lambda: run_queue(dm))
    m["split_device_ms_queue"] = split
    m["prompt_pass_share"] = round(split["prompt_pass"] / sum(split.values()), 3)
except Exception as ex:  # noqa: BLE001
    m["split_device_ms_queue"] = {"unavailable": str(ex)[:120]}
del os.environ["CALM_B200_PDL"]
result["M"] = m

# ---- U: one uniform wave
up = [rng.integers(0, spec.vocab_size, 256).astype(np.int32) for _ in range(ROWS)]
with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    q = dm.decode_sample_queue(up, [128] * ROWS, [a.t] * ROWS, [a.p] * ROWS, [], ROWS, seeds[:ROWS])
    b = dm.decode_sample_batch(up, 128, a.t, a.p, seeds[:ROWS])
    u = {"served": q[2], "steps": q[3], "outputs_equal": all(np.array_equal(x, y) for x, y in zip(q[0], b[0])) and q[1] == b[1]}
    t = best_of({"queue": lambda: dm.decode_sample_queue(up, [128] * ROWS, [a.t] * ROWS, [a.p] * ROWS, [], ROWS, seeds[:ROWS]),
                 "batch": lambda: dm.decode_sample_batch(up, 128, a.t, a.p, seeds[:ROWS])}, {})
u["ms"] = {k: round(v, 1) for k, v in t.items()}
u["tps"] = {k: round(ROWS * 128 / v * 1e3, 1) for k, v in t.items()}
u["queue_over_batch"] = round(t["queue"] / t["batch"], 4)
result["U"] = u

name, plim = card()
result.update({"gpu": name, "power_limit_w": plim})
line = json.dumps(result)
print(line)
if a.out:
    with open(a.out, "a") as f:
        f.write(line + "\n")
