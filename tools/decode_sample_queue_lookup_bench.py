#!/usr/bin/env python
"""Time calm_b200_decode_sample_queue_lookup: what prompt-lookup drafts in the request queue's free rows buy and cost.
Prints one JSON line (and appends it to the file --out names).

1. rows: the queue's step time against the rows in flight (1, 2, 4, 8, 16 requests of 512-token prompts, max_rows = the
   requests, greedy, the _truncated call), from two calls of 8 and 72 new tokens: (t72 - t8) / 64 steps, so the prompt
   pass cancels.  sync_ms: the same difference for calls with a stop token that never fires, which copy each step's
   tokens back and synchronise as the lookup call does; sync_ms - ms is that readback's cost per step.
2. greedy: 512-token random prompts, 256 new tokens, greedy, at max_rows 1 (4 requests) and 4 (16 requests): tokens/s,
   steps, drafted and accepted of the lookup call at max_draft 7 against the _truncated call, tokens compared in the same
   run.  At max_rows 1 also calm_b200_decode_greedy and calm_b200_decode_lookup (max_draft 7) over each request in turn.
3. sampled: the same at T 1.0, min-p 0.1.  Random weights give flat logits, so few drafts are accepted: this measures the
   overhead.  forced: the same requests constrained to a 7-token cycle (an automaton that allows one token per state),
   so that every draft is accepted once a request's own tokens hold the cycle: what accepted drafts buy, at most.
4. M: workload M of tools/decode_sample_queue_truncated_bench.py (64 requests, max_rows 16, T --t, min-p --p), the
   lookup call at max_draft 7 against _truncated.  Its rows are mostly full, so drafts land only in the tail.
Acceptance on random weights is not acceptance on text: a greedy random model falls into short cycles that lookup
predicts well, and a sampled one draws from nearly flat logits that no draft predicts.  Every time is the best of --reps
rounds with the arms alternating, after one warm-up of each, host clock around calls that end in a device synchronise.
Card name and power limit come from a query-only nvidia-smi in the same run.
  python tools/decode_sample_queue_lookup_bench.py [--workload llama3-8b-fp8] [--layers 32] [--out FILE]"""
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
ap.add_argument("--max-draft", type=int, default=7)
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--sections", default="rows,greedy,sampled,forced,M")
ap.add_argument("--out", default=None, help="a file to append the line to")
a = ap.parse_args()
os.environ.setdefault("CALM_B200_QUIET", "1")
SEEDS = [0x9E3779B97F4A7C15 + 7919 * i for i in range(64)]


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
    """calls: {name: f}; every call once as warm-up, then a.reps rounds alternating.  Returns ({name: best ms}, {name:
    the warm-up's result})."""
    res = {k: f() for k, f in calls.items()}
    best = {k: 1e18 for k in calls}
    for _ in range(a.reps):
        for k, f in calls.items():
            best[k] = min(best[k], timed(f)[0])
    return best, res


def same(x, y):
    """Tokens, states, served and prompt_rows of two queue tuples equal."""
    return x[1:3] == y[1:3] and x[4] == y[4] and all(np.array_equal(u, v) for u, v in zip(x[0], y[0]))


spec = mg.SPECS[a.workload] if a.layers is None else replace(mg.SPECS[a.workload], n_layers=a.layers)
tensors = mg.generate(spec, 0, device="cuda")
torch.cuda.synchronize()
print(f"{spec.name}: weights generated", file=sys.stderr, flush=True)
V = spec.vocab_size
result = {"workload": spec.name, "layers": spec.n_layers, "seq_len": a.seq_len, "max_draft": a.max_draft, "reps": a.reps}
sections = a.sections.split(",")


def alone(p, decode):
    dm.prefill(p[:-1])
    return decode(p)


def trunc(dm, prompts, max_new, T, P, rows, stop=(), **kw):
    n = len(prompts)
    return dm.decode_sample_queue_truncated(None, None, prompts, max_new, [T] * n, [P] * n, list(stop), rows, SEEDS[:n], **kw)


def look(dm, prompts, max_new, T, P, rows, **kw):
    n = len(prompts)
    return dm.decode_sample_queue_lookup(None, None, prompts, max_new, [T] * n, [P] * n, [], rows, SEEDS[:n], max_draft=a.max_draft, **kw)


with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
    rng = np.random.default_rng(1)
    prompts16 = [rng.integers(0, V, 512).astype(np.int32) for _ in range(16)]

    # ---- 1. step time against rows in flight
    if "rows" in sections:
        curve = {}
        for n in (1, 2, 4, 8, 16):
            ps = prompts16[:n]
            first = trunc(dm, ps, [72] * n, 0.0, 0.0, n)
            unused = int(np.setdiff1d(np.arange(V), np.concatenate(first[0]))[0])  # a stop token the run never emits
            t, _ = best_of({"s8": lambda: trunc(dm, ps, [8] * n, 0.0, 0.0, n), "s72": lambda: trunc(dm, ps, [72] * n, 0.0, 0.0, n),
                            "y8": lambda: trunc(dm, ps, [8] * n, 0.0, 0.0, n, [unused]), "y72": lambda: trunc(dm, ps, [72] * n, 0.0, 0.0, n, [unused])})
            curve[n] = {"ms": round((t["s72"] - t["s8"]) / 64, 3), "sync_ms": round((t["y72"] - t["y8"]) / 64, 3)}
        result["rows"] = curve
        print(json.dumps(curve), file=sys.stderr, flush=True)

    # ---- 2, 3. few rows in flight, greedy and sampled
    cyc = list(range(100, 107))  # (forced) state s allows cyc[s] alone and moves to s + 1 mod 7
    allow = np.zeros((len(cyc), V), bool)
    allow[np.arange(len(cyc)), cyc] = True
    cycle = lib.TokenAutomaton(V, allow, (np.arange(len(cyc)) + 1) % len(cyc), None)
    for sec, (T, P) in (("greedy", (0.0, 0.0)), ("sampled", (1.0, 0.1)), ("forced", (1.0, 0.1))):
        if sec not in sections:
            continue
        out = {}
        for rows, nreq in ((1, 4), (4, 16)):
            ps, mn = prompts16[:nreq], [256] * nreq
            kw = dict(automaton=cycle, start=[i % len(cyc) for i in range(nreq)]) if sec == "forced" else {}
            calls = {"truncated": lambda: trunc(dm, ps, mn, T, P, rows, **kw), "lookup": lambda: look(dm, ps, mn, T, P, rows, **kw)}
            if rows == 1 and T == 0.0:  # the single-sequence decode path, each request in turn after its prompt pass
                calls["decode_greedy"] = lambda: [alone(p, lambda p: dm.decode_greedy(int(p[-1]), len(p) - 1, 256)) for p in ps]
                calls["decode_lookup"] = lambda: [alone(p, lambda p: dm.decode_lookup(p, 256, max_draft=a.max_draft)[0]) for p in ps]
            t, res = best_of(calls)
            tr, lk = res["truncated"], res["lookup"]
            m = {"requests": nreq, "tokens": int(sum(len(x) for x in tr[0])), "served": lk[2], "equal": same(lk, tr), "steps": {"truncated": tr[3], "lookup": lk[3]},
                 "drafted": lk[-2], "accepted": lk[-1], "ms": {k: round(v, 1) for k, v in t.items()}}
            m["tokens_per_s"] = {k: round(m["tokens"] / (v / 1e3), 1) for k, v in t.items()}
            m["speedup_vs_truncated"] = {k: round(t["truncated"] / v, 3) for k, v in t.items() if k != "truncated"}
            if "decode_greedy" in res:  # (the decode path differs from the queue's in the last bits, so its tokens may part)
                for k in ("decode_greedy", "decode_lookup"):
                    m[f"{k}_same_tokens"] = sum(bool(np.array_equal(g, x)) for g, x in zip(res[k], tr[0]))
            out[f"max_rows_{rows}"] = m
            print(json.dumps({sec: m}), file=sys.stderr, flush=True)
        result[sec] = out

# ---- 4. workload M (tools/decode_sample_queue_truncated_bench.py's draws, in the same order)
if "M" in sections:
    rng = np.random.default_rng(0)
    nreq = 64
    lens = rng.integers(64, 513, nreq)
    mnew = [int(x) for x in rng.integers(16, 257, nreq)]
    prompts = [rng.integers(0, V, int(n)).astype(np.int32) for n in lens]
    with lib.DeviceModel(spec, tensors, seq_len=a.seq_len) as dm:
        t, res = best_of({"truncated": lambda: trunc(dm, prompts, mnew, a.t, a.p, 16), "lookup": lambda: look(dm, prompts, mnew, a.t, a.p, 16)})
    tr, lk = res["truncated"], res["lookup"]
    result["M"] = {"temperature": a.t, "minp": a.p, "useful_tokens": int(sum(len(x) for x in tr[0])), "equal": same(lk, tr),
                   "steps": {"truncated": tr[3], "lookup": lk[3]}, "drafted": lk[-2], "accepted": lk[-1], "ms": {k: round(v, 1) for k, v in t.items()},
                   "overhead_vs_truncated": round(t["lookup"] / t["truncated"] - 1, 4)}

name, plim = card()
result.update({"gpu": name, "power_limit_w": plim})
line = json.dumps(result)
print(line)
if a.out:
    with open(a.out, "a") as f:
        f.write(line + "\n")
