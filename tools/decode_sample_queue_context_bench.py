#!/usr/bin/env python
"""Time calm_b200_decode_sample_queue_context against the queue over the concatenated prompts.  Prints one JSON line (and
appends it to the file --out names).

Workload F (few-shot): 64 requests behind one 1024-token context, seeded own lengths uniform in [16, 128] and max_new
uniform in [16, 256].  Workload N (samples): 4 prompts of 512 tokens x 16 samples of 128 tokens, each sample a request
with context = prompt[:-1] and own = prompt[-1:].  No stop tokens (random weights make stops arbitrary).  Arms:
  context      decode_sample_queue_context at max_rows 16
  queue        decode_sample_queue over the concatenated prompts at max_rows 16
  sample_n     (N only) forward_prefill_cuda + decode_sample_n(nseq = 16) per prompt
For each: useful tokens/s (sum of out_len over wall time, prompt passes included), steps and prompt_rows; for the two queue
arms the device time by kernel group from one torch.profiler run of an engine without programmatic dependent launch
(prompt pass: k_pf_gemm + k_pf_attn; k_sn_*; k_vf_gemm; the rest).  outputs_equal: the context call's tokens and states
equal the concatenated queue's (and, for N, decode_sample_n's), checked in the same run.
Each time is the best of --reps rounds with the arms alternating, after one warm-up of each, host clock around calls that
end in a device synchronise.  Card name and power limit come from a query-only nvidia-smi in the same run.
  python tools/decode_sample_queue_context_bench.py [--workload llama3-8b-fp8] [--layers 32] [--out FILE]"""
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
ap.add_argument("--workloads", default="F,N", help="which of F and N to run")
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


def kernel_split(f):
    """Device time of one call of f per kernel group, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        f()
        torch.cuda.synchronize()
    out = {"prompt_pass": 0.0, "k_sn": 0.0, "k_vf_gemm": 0.0, "rest": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
        if t == 0.0 or e.key.startswith(("Memcpy", "Memset")):
            continue
        key = ("prompt_pass" if "k_pf_gemm" in e.key or "k_pf_attn" in e.key else "k_sn" if "k_sn_" in e.key
               else "k_vf_gemm" if "k_vf_gemm" in e.key else "rest")
        out[key] += t
    return {k: round(v, 1) for k, v in out.items()}


spec = mg.SPECS[a.workload] if a.layers is None else replace(mg.SPECS[a.workload], n_layers=a.layers)
tensors = mg.generate(spec, 0, device="cuda")
torch.cuda.synchronize()
print(f"{spec.name}: weights generated", file=sys.stderr, flush=True)
rng = np.random.default_rng(0)
result = {"workload": spec.name, "layers": spec.n_layers, "seq_len": a.seq_len, "temperature": a.t, "minp": a.p, "reps": a.reps}


def measure(contexts, ctx_of, prompts, max_new, seeds, extra=None):
    """The context call against the queue over ctx ++ prompt (and `extra`: {name: (f, check)})."""
    n = len(prompts)
    T, P = [a.t] * n, [a.p] * n
    cat = [np.concatenate([contexts[c], p]).astype(np.int32) if c >= 0 else p for c, p in zip(ctx_of, prompts)]

    def run_context(dm):
        return dm.decode_sample_queue_context(contexts, ctx_of, prompts, max_new, T, P, [], ROWS, seeds)

    def run_queue(dm):
        return dm.decode_sample_queue(cat, max_new, T, P, [], ROWS, seeds)

    useful = sum(max_new)
    with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
        c = run_context(dm)
        q = run_queue(dm)
        m = {"served": [c[2], q[2]], "useful_tokens": useful,
             "outputs_equal": c[1] == q[1] and all(np.array_equal(x, y) for x, y in zip(c[0], q[0]))}
        calls = {"context": lambda: run_context(dm), "queue": lambda: run_queue(dm)}
        for k, (f, check) in (extra or {}).items():
            m[f"outputs_equal_{k}"] = check(f(dm), c)
            calls[k] = (lambda f: lambda: f(dm))(f)
        t = best_of(calls)
    m["ms"] = {k: round(v, 1) for k, v in t.items()}
    m["useful_tps"] = {k: round(useful / v * 1e3, 1) for k, v in t.items()}
    m["steps"] = {"context": c[3], "queue": q[3]}
    m["prompt_rows"] = {"context": c[4], "queue": sum(-(-(len(x) - 1) // 8) * 8 for x, mn in zip(cat, max_new) if mn)}
    m["speedup_vs_queue"] = round(t["queue"] / t["context"], 3)
    print(json.dumps(m), file=sys.stderr, flush=True)  # (the profile below takes a while)
    # the split comes from an engine without programmatic dependent launch: with it, a kernel's span includes the time its
    # CTAs wait for the previous kernel to finish
    os.environ["CALM_B200_PDL"] = "0"
    try:
        with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
            m["split_device_ms"] = {}
            for k, f in (("context", run_context), ("queue", run_queue)):
                f(dm)
                m["split_device_ms"][k] = kernel_split(lambda: f(dm))
    except Exception as ex:  # noqa: BLE001
        m["split_device_ms"] = {"unavailable": str(ex)[:120]}
    del os.environ["CALM_B200_PDL"]
    return m


# ---- F: one few-shot context
nf = 64
fctx = [rng.integers(0, spec.vocab_size, 1024).astype(np.int32)]
fown = [rng.integers(0, spec.vocab_size, int(n)).astype(np.int32) for n in rng.integers(16, 129, nf)]
fnew = [int(x) for x in rng.integers(16, 257, nf)]
if "F" in a.workloads:
    result["F"] = measure(fctx, [0] * nf, fown, fnew, [0x9E3779B97F4A7C15 + 7919 * i for i in range(nf)])

# ---- N: 4 prompts x 16 samples
nprompt, nsamp, ntok = 4, 16, 128
nprompts = [rng.integers(0, spec.vocab_size, 512).astype(np.int32) for _ in range(nprompt)]
nseeds = [0x9E3779B97F4A7C15 + 104729 * i for i in range(nprompt * nsamp)]


def run_sample_n(dm):
    toks, states = [], []
    for k, p in enumerate(nprompts):
        dm.prefill(p[:-1], 0)
        t, s, _ = dm.decode_sample_n(int(p[-1]), len(p) - 1, ntok, a.t, a.p, nseeds[k * nsamp:(k + 1) * nsamp])
        toks += list(t)
        states += s
    return toks, states


def same_as_context(sn, c):
    return sn[1] == c[1] and all(np.array_equal(x, y) for x, y in zip(sn[0], c[0]))


if "N" in a.workloads:
    result["N"] = measure([p[:-1] for p in nprompts], [k // nsamp for k in range(nprompt * nsamp)], [nprompts[k // nsamp][-1:] for k in range(nprompt * nsamp)],
                      [ntok] * (nprompt * nsamp), nseeds, {"sample_n": (run_sample_n, same_as_context)})

name, plim = card()
result.update({"gpu": name, "power_limit_w": plim})
line = json.dumps(result)
print(line)
if a.out:
    with open(a.out, "a") as f:
        f.write(line + "\n")
