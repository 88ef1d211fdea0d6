#!/usr/bin/env python
"""Time calm_b200_decode_sample_queue_truncated: what per-request top-k / top-p truncation costs the request queue.
Prints one JSON line (and appends it to the file --out names).

Workloads M and F are tools/decode_sample_queue_penalties_bench.py's (the queue benches' mixed lengths, and 64 requests
behind one 1024-token context), no stop tokens, max_rows 16, no log-probabilities, penalties or automaton.  Arms, all
the truncated call with every request set the same way: neutral (T --t, minp --p, top_k / top_p NULL, which launches
what decode_sample_queue_constrained launches), top_p_0.9 (T 0.6, minp 0, top_p 0.9: Llama-3-Instruct's generation
config), qwen2 (T 0.7, minp 0, top_k 20, top_p 0.8: Qwen2-Instruct's, without its repetition penalty) and top_k_50
(T --t, minp --p, top_k 50).  No stop tokens, so every arm takes the same steps.  For each: ms, and the overhead over
neutral.  neutral_equal: the neutral arm's tokens, states and steps equal decode_sample_queue_constrained's in the same
run.  split_device_ms: device time per kernel group of one call of each arm, from torch.profiler on an engine without
programmatic dependent launch: classifier (k_vf_gemm's classifier launches), sampler (k_sample_scan_rows and
k_sample_scan_rows_masked), trunc (k_sample_trunc_rows), copies, other; trunc_us_per_step is trunc over the call's
steps.  Each time is the best of --reps rounds with the arms alternating, after one warm-up of each, host clock around
calls that end in a device synchronise.  Card name and power limit come from a query-only nvidia-smi in the same run.
  python tools/decode_sample_queue_truncated_bench.py [--workload llama3-8b-fp8] [--layers 32] [--out FILE]"""
import argparse
import json
import os
import re
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
ap.add_argument("--workloads", default="M,F", help="which of M and F to run")
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


def best_of(calls):
    """calls: {name: f}; every call once as warm-up, then a.reps rounds alternating."""
    for f in calls.values():
        f()
    best = {k: 1e18 for k in calls}
    for _ in range(a.reps):
        for k, f in calls.items():
            best[k] = min(best[k], timed(f)[0])
    return best


def group(key):
    m = re.search(r"k_vf_gemm<(\d+)", key)
    if m and int(m.group(1)) in (5, 7):  # PF_CLS_GREEDY, PF_CLS_SAMPLE
        return "classifier"
    if key.startswith(("Memcpy", "Memset")):
        return "copies"
    if "k_sample_trunc_rows" in key:
        return "trunc"
    if "k_sample_scan_rows" in key:
        return "sampler"
    return "other"


def kernel_split(f):
    """Device time of one call of f per kernel group, from torch.profiler's CUDA activity, and the call's wall time less
    its device time."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        wall, _ = timed(f)
    out = {g: 0.0 for g in ("classifier", "sampler", "trunc", "copies", "other")}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
        if t:
            out[group(e.key)] += t
    out["host_gap_ms"] = wall - sum(out.values())
    return {k: round(v, 2) for k, v in out.items()}


spec = mg.SPECS[a.workload] if a.layers is None else replace(mg.SPECS[a.workload], n_layers=a.layers)
tensors = mg.generate(spec, 0, device="cuda")
torch.cuda.synchronize()
print(f"{spec.name}: weights generated", file=sys.stderr, flush=True)
result = {"workload": spec.name, "layers": spec.n_layers, "seq_len": a.seq_len, "temperature": a.t, "minp": a.p, "reps": a.reps, "max_rows": ROWS}


def measure(contexts, ctx_of, prompts, max_new, seeds):
    """The truncated call's four arms (contexts None: no contexts), and decode_sample_queue_constrained once."""
    n = len(prompts)
    arms_cfg = {"neutral": (a.t, a.p, None, None), "top_p_0.9": (0.6, 0.0, None, 0.9), "qwen2": (0.7, 0.0, 20, 0.8),
                "top_k_50": (a.t, a.p, 50, None)}

    def run(dm, name):
        T, P, K, TP = arms_cfg[name]
        return dm.decode_sample_queue_truncated(contexts, ctx_of, prompts, max_new, [T] * n, [P] * n, [], ROWS, seeds,
                                                top_k=None if K is None else [K] * n, top_p=None if TP is None else [TP] * n)

    arms = {k: (lambda k: lambda dm: run(dm, k))(k) for k in arms_cfg}
    with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
        ref = dm.decode_sample_queue_constrained(contexts, ctx_of, prompts, max_new, [a.t] * n, [a.p] * n, [], ROWS, seeds)
        out = {k: f(dm) for k, f in arms.items()}
        nu = out["neutral"]
        m = {"served": ref[2], "useful_tokens": int(sum(len(x) for x in ref[0])), "steps": ref[3],
             "neutral_equal": nu[1:4] == tuple(ref[1:4]) and all(np.array_equal(x, y) for x, y in zip(nu[0], ref[0])),
             "steps_by_arm": {k: o[3] for k, o in out.items()}}
        t = best_of({k: (lambda f: lambda: f(dm))(f) for k, f in arms.items()})
    m["ms"] = {k: round(v, 1) for k, v in t.items()}
    m["overhead_vs_neutral"] = {k: round(t[k] / t["neutral"] - 1, 4) for k in t if k != "neutral"}
    print(json.dumps(m), file=sys.stderr, flush=True)  # (the profile below takes a while)
    # the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its
    # CTAs wait for the previous kernel to finish
    os.environ["CALM_B200_PDL"] = "0"
    try:
        with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
            split = {}
            for k, f in arms.items():
                f(dm)
                split[k] = kernel_split(lambda: f(dm))
        m["split_device_ms"] = split
        m["trunc_us_per_step"] = {k: round(1e3 * split[k]["trunc"] / max(m["steps_by_arm"][k], 1), 1) for k in split}
    except Exception as ex:  # noqa: BLE001
        m["split_device_ms"] = {"unavailable": str(ex)[:120]}
    del os.environ["CALM_B200_PDL"]
    return m

# ---- M: tools/decode_sample_queue_bench.py's mixed lengths (the same draws in the same order)
if "M" in a.workloads:
    rng = np.random.default_rng(0)
    nreq = 64
    lens = rng.integers(64, 513, nreq)
    mnew = [int(x) for x in rng.integers(16, 257, nreq)]
    prompts = [rng.integers(0, spec.vocab_size, int(n)).astype(np.int32) for n in lens]
    result["M"] = measure(None, None, prompts, mnew, [0x9E3779B97F4A7C15 + 7919 * i for i in range(nreq)])

# ---- F: tools/decode_sample_queue_context_bench.py's few-shot context (the same draws in the same order)
if "F" in a.workloads:
    rng = np.random.default_rng(0)
    nf = 64
    fctx = [rng.integers(0, spec.vocab_size, 1024).astype(np.int32)]
    fown = [rng.integers(0, spec.vocab_size, int(n)).astype(np.int32) for n in rng.integers(16, 129, nf)]
    fnew = [int(x) for x in rng.integers(16, 257, nf)]
    result["F"] = measure(fctx, [0] * nf, fown, fnew, [0x9E3779B97F4A7C15 + 7919 * i for i in range(nf)])

name, plim = card()
result.update({"gpu": name, "power_limit_w": plim})
line = json.dumps(result)
print(line)
if a.out:
    with open(a.out, "a") as f:
        f.write(line + "\n")
