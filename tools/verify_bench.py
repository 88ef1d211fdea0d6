#!/usr/bin/env python
"""Time draft verification and prompt-lookup decoding.  Prints one JSON line:
  verify_ms[n]            calm_b200_verify_greedy of n tokens at pos0 = --pos
  score_greedy_ms[n]      calm_b200_score_greedy of n + 1 tokens at the same position (the same n greedy tokens)
  forward_argmax_ms       one calm_b200_forward_argmax at that position
  split_ms_verify8        (torch.profiler, an engine launched without programmatic dependent launch) the device time of
                          one verify_greedy(8) by kernel group: k_vf_gemm, k_pf_attn and the rest
  decode_greedy_tps       calm_b200_decode_greedy of --tokens tokens after position --pos, tokens per second
  lookup[name]            calm_b200_decode_lookup of the same tokens: tokens per second, model steps, and whether it
                          returned decode_greedy's tokens; full_d{3,7,15} draw from source = prompt ++ decode_greedy's
                          stream (full acceptance where verification agrees), no_match from a source that never matches
Each figure is the best of --reps, the calls of a group alternating, after one warm-up of every call; CUDA events on the
library's stream (lookup: wall clock, since it synchronises per step).  The cache below --pos is filled with random
entries.  Card name and power limit come from a query-only nvidia-smi.
  python tools/verify_bench.py [--workload llama3-8b-fp8] [--layers 32] [--pos 2048] [--tokens 256]"""
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
        out = {"k_vf_gemm": 0.0, "k_pf_attn": 0.0, "other": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
            if t == 0.0 or e.key.startswith(("Memcpy", "Memset")):
                continue
            key = "k_vf_gemm" if "k_vf_gemm" in e.key else ("k_pf_attn" if "k_pf_attn" in e.key else "other")
            out[key] += t
        return {k: round(v, 3) for k, v in out.items()}
    except Exception as ex:  # noqa: BLE001
        return {"unavailable": str(ex)[:120]}


with lib.DeviceModel(spec, tensors, seq_len=SEQ_LEN) as dm:
    dm.fill_kv(a.pos, seed=3)
    served = {n: int(dm.verify_greedy(prompt[a.pos - n + 1:a.pos + 1], a.pos)[1]) for n in ns}
    calls = {}
    for n in ns:
        blk = prompt[a.pos - n + 1:a.pos + 1]
        calls[f"verify{n}"] = lambda blk=blk: dm.verify_greedy(blk, a.pos)
        calls[f"score_greedy{n}"] = lambda blk=blk: dm.score_greedy(np.concatenate([blk, [0]]), a.pos)
    calls["forward_argmax"] = lambda: dm.forward_argmax(int(prompt[-1]), a.pos)
    t1 = best_of(calls)

    N = a.tokens
    G = dm.decode_greedy(int(prompt[-1]), a.pos, N)
    full = np.concatenate([prompt, G]).astype(np.int32)
    absent = np.setdiff1d(np.arange(spec.vocab_size), full)[:2].astype(np.int32)  # tokens neither the prompt nor G holds
    runs = {"decode_greedy": lambda: dm.decode_greedy(int(prompt[-1]), a.pos, N)}
    for d in (3, 7, 15):
        runs[f"full_d{d}"] = lambda d=d: dm.decode_lookup(prompt, N, source=full, max_draft=d)
    runs["no_match"] = lambda: dm.decode_lookup(prompt, N, source=absent, max_draft=7)
    t2 = best_of(runs, timer="wall")
    lookup = {}
    for k in runs:
        if k == "decode_greedy":
            continue
        out, steps = runs[k]()
        lookup[k] = {"tps": round(N / t2[k] * 1e3, 1), "ms": round(t2[k], 2), "steps": int(steps), "equals_decode_greedy": bool(np.array_equal(out, G))}

# the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its CTAs
# wait for the previous kernel to finish
os.environ["CALM_B200_PDL"] = "0"
with lib.DeviceModel(spec, tensors, seq_len=SEQ_LEN) as dm:
    dm.fill_kv(a.pos, seed=3)
    blk8 = prompt[a.pos - 7:a.pos + 1]
    dm.verify_greedy(blk8, a.pos)
    split = kernel_split(lambda: dm.verify_greedy(blk8, a.pos))

name, plim = card()
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": SEQ_LEN, "pos": a.pos, "served": served,
    "verify_ms": {n: round(t1[f"verify{n}"], 3) for n in ns}, "score_greedy_ms": {n: round(t1[f"score_greedy{n}"], 3) for n in ns},
    "forward_argmax_ms": round(t1["forward_argmax"], 3), "split_ms_verify8": split,
    "tokens": N, "decode_greedy_tps": round(N / t2["decode_greedy"] * 1e3, 1), "decode_greedy_ms": round(t2["decode_greedy"], 2), "lookup": lookup,
    "reps": a.reps, "gpu": name, "power_limit_w": plim}))
