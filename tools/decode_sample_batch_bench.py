#!/usr/bin/env python
"""Time nseq different prompts decoded together against the same prompts run one after another.  Prints one JSON line with,
per workload and nseq:
  batch_ms            calm_b200_decode_sample_batch of --tokens tokens per sequence, end to end (packed prompt pass + steps)
  batch_step_ms       its decode time per step: (batch_ms - the same call for one token) / (--tokens - 1)
  sequential_ms       forward_prefill_cuda + calm_b200_decode_sample for each prompt in turn
  sample_n_ms         (for information) forward_prefill_cuda of one prompt of the same length + calm_b200_decode_sample_n
  aggregate_tps, sequential_tps, speedup = sequential_ms / batch_ms
  outputs_equal       every sequence of the timed batch call equals forward_prefill_cuda + decode_sample_n(nseq = 1) of its
                      prompt alone, checked in the same run (nseq = 16 only: its rows sit at the largest slot bases)
  split_ms_step16     (torch.profiler, an engine launched without programmatic dependent launch) the device time of one
                      16-row step by kernel group: the per-row attention (k_sn_attn + k_sn_fold), k_vf_gemm and the rest;
                      the difference of a 3-token and a 1-token call, halved, so the packed prompt pass drops out
Workloads: A = nseq 1, 2, 4, 8, 16 prompts of 256 different random tokens at seq_len 8192; B = 16 prompts of 1024 tokens at
seq_len 18432.  Each figure is the best of --reps, the calls alternating, after one warm-up of each; CUDA events on the
library's stream.  Card name and power limit come from a query-only nvidia-smi in the same run.
  python tools/decode_sample_batch_bench.py [--workload llama3-8b-fp8] [--layers 32] [--tokens 128]"""
import argparse
import json
import os
import subprocess
import sys
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
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--t", type=float, default=1.0)
ap.add_argument("--p", type=float, default=0.1)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--only", default="A,B", help="workloads to run")
a = ap.parse_args()
os.environ.setdefault("CALM_B200_QUIET", "1")
WORKLOADS = {"A": dict(ns=[1, 2, 4, 8, 16], plen=256, seq_len=8192), "B": dict(ns=[16], plen=1024, seq_len=18432)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:  # noqa: BLE001 (no nvidia-smi: the line still carries the timings)
        return None, None


spec = mg.SPECS[a.workload] if a.layers is None else replace(mg.SPECS[a.workload], n_layers=a.layers)
L = lib.load()
tensors = mg.generate(spec, 0, device="cuda")
torch.cuda.synchronize()
N = a.tokens
seeds = [0x9E3779B97F4A7C15 + 7919 * i for i in range(16)]


def best_of(calls):
    """calls: {name: f}; every call once as warm-up, then --reps rounds alternating; the best time of each in ms."""
    for f in calls.values():
        f()
    best = {k: 1e9 for k in calls}
    for _ in range(a.reps):
        for k, f in calls.items():
            L.calm_b200_timer_start()
            f()
            best[k] = min(best[k], L.calm_b200_timer_stop())
    return best


def kernel_split(f):
    """Device time of one call of f per kernel group, from torch.profiler's CUDA activity (None where it is unavailable)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        f()
        torch.cuda.synchronize()
    out = {"attention": 0.0, "k_vf_gemm": 0.0, "other": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
        if t == 0.0 or e.key.startswith(("Memcpy", "Memset")):
            continue
        key = "attention" if "k_sn_" in e.key else "k_vf_gemm" if "k_vf_gemm" in e.key else "other"
        out[key] += t
    return out


def sequential(dm, prompts):
    for p, s in zip(prompts, seeds):
        dm.prefill(p[:-1], 0)
        dm.decode_sample(int(p[-1]), len(p) - 1, N, a.t, a.p, s)


result = {"workload": spec.name, "layers": spec.n_layers, "temperature": a.t, "minp": a.p, "tokens": N, "reps": a.reps}
rng = np.random.default_rng(0)
for wl in a.only.split(","):
    cfg = WORKLOADS[wl]
    ns, plen = cfg["ns"], cfg["plen"]
    prompts = [rng.integers(0, spec.vocab_size, plen).astype(np.int32) for _ in range(max(ns))]
    r = {"prompt_len": plen, "seq_len": cfg["seq_len"]}
    with lib.DeviceModel(spec, tensors, seq_len=cfg["seq_len"]) as dm:
        r["served"] = {n: int(dm.decode_sample_batch(prompts[:n], 1, a.t, a.p, seeds[:n])[2]) for n in ns}
        calls = {}
        for n in ns:
            calls[f"b{n}"] = lambda n=n: dm.decode_sample_batch(prompts[:n], N, a.t, a.p, seeds[:n])
            calls[f"b1tok{n}"] = lambda n=n: dm.decode_sample_batch(prompts[:n], 1, a.t, a.p, seeds[:n])
            calls[f"seq{n}"] = lambda n=n: sequential(dm, prompts[:n])
            calls[f"sn{n}"] = lambda n=n: (dm.prefill(prompts[0][:-1], 0), dm.decode_sample_n(int(prompts[0][-1]), plen - 1, N, a.t, a.p, seeds[:n]))
        t = best_of(calls)
        n16 = max(ns)
        got = dm.decode_sample_batch(prompts[:n16], N, a.t, a.p, seeds[:n16])[0]
        equal = True
        for b in range(n16):
            dm.prefill(prompts[b][:-1], 0)
            alone = dm.decode_sample_n(int(prompts[b][-1]), plen - 1, N, a.t, a.p, [seeds[b]])[0][0]
            equal &= bool(np.array_equal(alone, got[b]))
        r["outputs_equal"] = equal
    r["batch_ms"] = {n: round(t[f"b{n}"], 2) for n in ns}
    r["batch_step_ms"] = {n: round((t[f"b{n}"] - t[f"b1tok{n}"]) / (N - 1), 3) for n in ns}
    r["sequential_ms"] = {n: round(t[f"seq{n}"], 2) for n in ns}
    r["sample_n_ms"] = {n: round(t[f"sn{n}"], 2) for n in ns}
    r["aggregate_tps"] = {n: round(n * N / t[f"b{n}"] * 1e3, 1) for n in ns}
    r["sequential_tps"] = {n: round(n * N / t[f"seq{n}"] * 1e3, 1) for n in ns}
    r["sample_n_tps"] = {n: round(n * N / t[f"sn{n}"] * 1e3, 1) for n in ns}
    r["speedup"] = {n: round(t[f"seq{n}"] / t[f"b{n}"], 2) for n in ns}
    # the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its
    # CTAs wait for the previous kernel to finish
    os.environ["CALM_B200_PDL"] = "0"
    try:
        with lib.DeviceModel(spec, tensors, seq_len=cfg["seq_len"]) as dm:
            dm.decode_sample_batch(prompts[:16], 3, a.t, a.p, seeds)
            s3 = kernel_split(lambda: dm.decode_sample_batch(prompts[:16], 3, a.t, a.p, seeds))
            s1 = kernel_split(lambda: dm.decode_sample_batch(prompts[:16], 1, a.t, a.p, seeds))
        r["split_ms_step16"] = {k: round((s3[k] - s1[k]) / 2, 3) for k in s3}
    except Exception as ex:  # noqa: BLE001
        r["split_ms_step16"] = {"unavailable": str(ex)[:120]}
    del os.environ["CALM_B200_PDL"]
    result[wl] = r

name, plim = card()
result.update({"gpu": name, "power_limit_w": plim})
print(json.dumps(result))
