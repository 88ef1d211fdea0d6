#!/usr/bin/env python
"""Time beam search against the same weight passes without selection or ancestry.  Prints one JSON line:
  beam_ms[B]        calm_b200_decode_beam of --tokens steps with B beams after position --pos, no stop list (every call runs
                    --tokens steps)
  sample_n_ms[B]    calm_b200_decode_sample_n of --tokens tokens for nseq = B at temperature 0: the same passes over the
                    weights and the same shared-prompt attention, without the top-K epilogue, the merge's lists, k_bm_select
                    and the ancestry
  greedy_ms         calm_b200_decode_greedy of --tokens tokens (the decode graph, one sequence)
  overhead[B]       beam_ms / sample_n_ms - 1
  split_ms[B]       (torch.profiler, an engine launched without programmatic dependent launch) the device time of a 2-step
                    beam call by kernel group: the attention (k_sn_attn + k_sn_fold), k_vf_gemm, the merge (k_pf_logprob),
                    k_bm_select and the rest (norms, embedding, RoPE table)
Each figure is the best of --reps, the calls alternating, after one warm-up of each; CUDA events on the library's stream.
The cache below --pos is filled with random entries (fill_kv).  Card name and power limit come from a query-only
nvidia-smi in the same run.
  python tools/decode_beam_bench.py [--workload llama3-8b-fp8] [--pos 2048] [--tokens 128] [--beams 1,2,4,8]"""
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
ap.add_argument("--beams", default="1,2,4,8")
ap.add_argument("--tokens", type=int, default=128)
ap.add_argument("--reps", type=int, default=3)
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
beams = [int(b) for b in a.beams.split(",")]
token0, N = 1234 % spec.vocab_size, a.tokens


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
        out = {"attention": 0.0, "k_vf_gemm": 0.0, "merge": 0.0, "k_bm_select": 0.0, "other": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
            if t == 0.0 or e.key.startswith(("Memcpy", "Memset")):
                continue
            key = ("attention" if "k_sn_" in e.key else "k_vf_gemm" if "k_vf_gemm" in e.key else "merge" if "k_pf_logprob" in e.key
                   else "k_bm_select" if "k_bm_select" in e.key else "other")
            out[key] += t
        return {k: round(v, 3) for k, v in out.items()}
    except Exception as ex:  # noqa: BLE001
        return {"unavailable": str(ex)[:120]}


with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    dm.fill_kv(a.pos, seed=3)
    served = {B: int(dm.decode_beam(token0, a.pos, N, B)[1]) for B in beams}
    calls = {"greedy": lambda: dm.decode_greedy(token0, a.pos, N)}
    for B in beams:
        calls[f"beam{B}"] = lambda B=B: dm.decode_beam(token0, a.pos, N, B)
        calls[f"n{B}"] = lambda B=B: dm.decode_sample_n(token0, a.pos, N, 0.0, 0.1, [1] * B)
    t = best_of(calls)

os.environ["CALM_B200_PDL"] = "0"  # with programmatic dependent launch a kernel's span includes its wait for the one before
with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    dm.fill_kv(a.pos, seed=3)
    split = {}
    for B in beams:
        dm.decode_beam(token0, a.pos, 2, B)
        split[B] = kernel_split(lambda B=B: dm.decode_beam(token0, a.pos, 2, B))

name, plim = card()
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": a.seq_len, "pos": a.pos, "tokens": N, "served": served,
    "beam_ms": {B: round(t[f"beam{B}"], 2) for B in beams}, "sample_n_ms": {B: round(t[f"n{B}"], 2) for B in beams},
    "greedy_ms": round(t["greedy"], 2), "ms_per_step": {B: round(t[f"beam{B}"] / N, 3) for B in beams},
    "overhead": {B: round(t[f"beam{B}"] / t[f"n{B}"] - 1, 4) for B in beams}, "split_ms_2steps": split,
    "reps": a.reps, "gpu": name, "power_limit_w": plim}))
