#!/usr/bin/env python
"""Time sampled draft verification and sampled prompt-lookup decoding.  Prints one JSON line:
  verify_sample_ms[n]     calm_b200_verify_sample of n tokens at pos0 = --pos, temperature --t, min-p --p
  verify_greedy_ms[n]     calm_b200_verify_greedy of the same block
  split_ms_sample16       (torch.profiler, an engine launched without programmatic dependent launch) the device time of
                          one verify_sample(16) and one verify_greedy(16) by kernel group: k_vf_gemm, k_pf_attn, the
                          sampler (k_sample_scan_rows + k_sample_pick_rows, all rows side by side) and the rest
  sampler_row_us          mean over the 16 rows of calm_b200_sample_logits's device time (k_sample_scan + k_sample_pick
                          on one row): what each row would add if the rows were sampled one after another
  decode_sample_tps       calm_b200_decode_sample of --tokens tokens after position --pos, tokens per second
  lookup[name]            calm_b200_decode_lookup_sample of the same tokens from the same generator state: tokens per
                          second, model steps, and whether it returned decode_sample's tokens and final state; full_d{3,7,15}
                          draw from source = prompt ++ decode_sample's stream, no_match from a source that never matches
Each figure is the best of --reps, the calls of a group alternating, after one warm-up of every call; CUDA events on the
library's stream (lookup and decode_sample: wall clock, since the lookup synchronises per step).  The cache below --pos is
filled with random entries.  Random weights give flat logits, so acceptance here says little about real text.  Card name
and power limit come from a query-only nvidia-smi.
  python tools/verify_sample_bench.py [--workload llama3-8b-fp8] [--layers 32] [--pos 2048] [--tokens 256]"""
import argparse
import json
import os
import subprocess
import sys
import time
from dataclasses import replace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="llama3-8b-fp8")
ap.add_argument("--layers", type=int, default=None)
ap.add_argument("--pos", type=int, default=2048)
ap.add_argument("--ns", default="1,2,4,8,16")
ap.add_argument("--tokens", type=int, default=256)
ap.add_argument("--t", type=float, default=1.0)
ap.add_argument("--p", type=float, default=0.1)
ap.add_argument("--seed", type=int, default=12345)
ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()
os.environ.setdefault("CALM_B200_QUIET", "1")
SEQ_LEN = 4096


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
rng = np.random.default_rng(0)
prompt = rng.integers(0, spec.vocab_size, a.pos + 1).astype(np.int32)
ns = [int(n) for n in a.ns.split(",")]


def best_of(calls, timer="events"):
    """calls: {name: f}; every call once as warm-up, then --reps rounds alternating; the best time of each in ms."""
    for f in calls.values():
        f()
    best = {k: 1e9 for k in calls}
    for _ in range(a.reps):
        for k, f in calls.items():
            if timer == "events":
                L.calm_b200_timer_start()
                f()
                best[k] = min(best[k], L.calm_b200_timer_stop())
            else:
                t0 = time.perf_counter()
                f()
                best[k] = min(best[k], 1e3 * (time.perf_counter() - t0))
    return best


def kernel_split(f):
    """Device time of one call of f per kernel group, from torch.profiler's CUDA activity (None where it is unavailable)."""
    try:
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            f()
            torch.cuda.synchronize()
        out = {"k_vf_gemm": 0.0, "k_pf_attn": 0.0, "sampler": 0.0, "other": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
            if t == 0.0 or e.key.startswith(("Memcpy", "Memset")):
                continue
            key = next((k for k, s in (("k_vf_gemm", "k_vf_gemm"), ("k_pf_attn", "k_pf_attn"), ("sampler", "k_sample")) if s in e.key), "other")
            out[key] += t
        return {k: round(v, 3) for k, v in out.items()}
    except Exception as ex:  # noqa: BLE001
        return {"unavailable": str(ex)[:120]}


with lib.DeviceModel(spec, tensors, seq_len=SEQ_LEN) as dm:
    dm.fill_kv(a.pos, seed=3)
    served = {n: int(dm.verify_sample(prompt[a.pos - n + 1:a.pos + 1], a.pos, a.t, a.p, a.seed)[2]) for n in ns}
    calls = {}
    for n in ns:
        blk = prompt[a.pos - n + 1:a.pos + 1]
        calls[f"sample{n}"] = lambda blk=blk: dm.verify_sample(blk, a.pos, a.t, a.p, a.seed)
        calls[f"greedy{n}"] = lambda blk=blk: dm.verify_greedy(blk, a.pos)
    t1 = best_of(calls)

    N = a.tokens
    G, G_state = dm.decode_sample(int(prompt[-1]), a.pos, N, a.t, a.p, a.seed)
    full = np.concatenate([prompt, G]).astype(np.int32)
    absent = np.setdiff1d(np.arange(spec.vocab_size), full)[:2].astype(np.int32)  # tokens neither the prompt nor G holds
    runs = {"decode_sample": lambda: dm.decode_sample(int(prompt[-1]), a.pos, N, a.t, a.p, a.seed)}
    for d in (3, 7, 15):
        runs[f"full_d{d}"] = lambda d=d: dm.decode_lookup_sample(prompt, N, a.t, a.p, a.seed, source=full, max_draft=d)
    runs["no_match"] = lambda: dm.decode_lookup_sample(prompt, N, a.t, a.p, a.seed, source=absent, max_draft=7)
    t2 = best_of(runs, timer="wall")
    lookup = {}
    for k in runs:
        if k == "decode_sample":
            continue
        out, steps, state = runs[k]()
        lookup[k] = {"tps": round(N / t2[k] * 1e3, 1), "ms": round(t2[k], 2), "steps": int(steps),
                     "equals_decode_sample": bool(np.array_equal(out, G) and state == G_state)}

# the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its CTAs
# wait for the previous kernel to finish
os.environ["CALM_B200_PDL"] = "0"
with lib.DeviceModel(spec, tensors, seq_len=SEQ_LEN) as dm:
    dm.fill_kv(a.pos, seed=3)
    blk16 = prompt[a.pos - 15:a.pos + 1]
    dm.verify_sample(blk16, a.pos, a.t, a.p, a.seed)
    dm.verify_greedy(blk16, a.pos)
    split = {"verify_sample": kernel_split(lambda: dm.verify_sample(blk16, a.pos, a.t, a.p, a.seed)),
             "verify_greedy": kernel_split(lambda: dm.verify_greedy(blk16, a.pos))}
    dm.verify_sample(blk16, a.pos, a.t, a.p, a.seed)
    rows = dm.read_state("pf_logits").reshape(16, spec.vocab_size)
row_us = float(np.mean([lib.sample_logits(r, a.t, a.p, a.seed, timed=True)[2] for r in rows]))

name, plim = card()
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": SEQ_LEN, "pos": a.pos, "temperature": a.t, "minp": a.p, "served": served,
    "verify_sample_ms": {n: round(t1[f"sample{n}"], 3) for n in ns}, "verify_greedy_ms": {n: round(t1[f"greedy{n}"], 3) for n in ns},
    "sample_over_greedy": {n: round(t1[f"sample{n}"] / t1[f"greedy{n}"] - 1, 4) for n in ns},
    "split_ms_sample16": split, "sampler_row_us": round(row_us, 1),
    "tokens": N, "decode_sample_tps": round(N / t2["decode_sample"] * 1e3, 1), "decode_sample_ms": round(t2["decode_sample"], 2), "lookup": lookup,
    "reps": a.reps, "gpu": name, "power_limit_w": plim}))
