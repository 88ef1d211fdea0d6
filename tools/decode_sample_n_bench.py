#!/usr/bin/env python
"""Time n samples of one prompt together against n decode_sample runs.  Prints one JSON line:
  sample_n_ms[n]      calm_b200_decode_sample_n of --tokens tokens for n sequences after position --pos
  sequential_ms[n]    n back-to-back calm_b200_decode_sample runs of the same tokens from the same prefix
  aggregate_tps[n]    n * --tokens over each, and speedup[n] = sequential / sample_n
  split_ms_step16     (torch.profiler, an engine launched without programmatic dependent launch) the device time of one
                      nseq = 16 step by kernel group: the shared-prompt attention (k_sn_attn + k_sn_fold), k_vf_gemm and the
                      rest (norms, embedding, RoPE table, sampler, merges)
Each figure is the best of --reps, the calls alternating, after one warm-up of each; CUDA events on the library's stream.
The cache below --pos is filled with random entries (fill_kv).  Card name and power limit come from a query-only
nvidia-smi in the same run.
  python tools/decode_sample_n_bench.py [--workload llama3-8b-fp8] [--layers 32] [--pos 2048] [--tokens 128]"""
import argparse
import json
import os
import subprocess
import sys
from dataclasses import replace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="llama3-8b-fp8")
ap.add_argument("--layers", type=int, default=None)
ap.add_argument("--pos", type=int, default=2048)
ap.add_argument("--ns", default="1,2,4,8,16")
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--t", type=float, default=1.0)
ap.add_argument("--p", type=float, default=0.1)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--seq-len", type=int, default=4096)
a = ap.parse_args()
os.environ.setdefault("CALM_B200_QUIET", "1")


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
ns = [int(n) for n in a.ns.split(",")]
token0, N = 1234 % spec.vocab_size, a.tokens
seeds = [0x9E3779B97F4A7C15 + 7919 * i for i in range(max(ns))]


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
    try:
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
        return {k: round(v, 3) for k, v in out.items()}
    except Exception as ex:  # noqa: BLE001
        return {"unavailable": str(ex)[:120]}


with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    dm.fill_kv(a.pos, seed=3)
    served = {n: int(dm.decode_sample_n(token0, a.pos, N, a.t, a.p, seeds[:n])[2]) for n in ns}
    calls = {}
    for n in ns:
        calls[f"n{n}"] = lambda n=n: dm.decode_sample_n(token0, a.pos, N, a.t, a.p, seeds[:n])
        calls[f"seq{n}"] = lambda n=n: [dm.decode_sample(token0, a.pos, N, a.t, a.p, s) for s in seeds[:n]]
    t = best_of(calls)

# the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its CTAs
# wait for the previous kernel to finish
os.environ["CALM_B200_PDL"] = "0"
with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    dm.fill_kv(a.pos, seed=3)
    dm.decode_sample_n(token0, a.pos, 1, a.t, a.p, seeds[:16])
    split = kernel_split(lambda: dm.decode_sample_n(token0, a.pos, 1, a.t, a.p, seeds[:16]))

name, plim = card()
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": a.seq_len, "pos": a.pos, "temperature": a.t, "minp": a.p, "tokens": N,
    "served": served, "sample_n_ms": {n: round(t[f"n{n}"], 2) for n in ns}, "sequential_ms": {n: round(t[f"seq{n}"], 2) for n in ns},
    "ms_per_step": {n: round(t[f"n{n}"] / N, 3) for n in ns},
    "aggregate_tps": {n: round(n * N / t[f"n{n}"] * 1e3, 1) for n in ns}, "sequential_tps": {n: round(n * N / t[f"seq{n}"] * 1e3, 1) for n in ns},
    "speedup": {n: round(t[f"seq{n}"] / t[f"n{n}"], 2) for n in ns}, "split_ms_step16": split,
    "reps": a.reps, "gpu": name, "power_limit_w": plim}))
