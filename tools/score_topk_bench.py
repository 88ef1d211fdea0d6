#!/usr/bin/env python
"""Time the top-k scoring calls against their plain siblings on the same inputs.  Prints one JSON line:
  score_ms / score_topk_ms[k]              calm_b200_score vs calm_b200_score_topk on one --n-token sequence, k in --ks
  batch_ms / batch_topk_ms                 calm_b200_score_batch vs calm_b200_score_batch_topk at k = --batch-k on --nseq
                                           sequences of --seqlen tokens (the workload of profiles/h100_score_batch_llama3-8b-fp8.jsonl)
  *_extra_pct                              (top-k - plain) / plain in percent
Each figure is the best of --reps, the calls of a group alternating, after one warm-up of every call; CUDA events on the
library's stream.  Card name and power limit come from a query-only nvidia-smi.
  python tools/score_topk_bench.py [--workload llama3-8b-fp8] [--layers 32] [--n 2049] [--ks 1,5,20] [--nseq 256] [--seqlen 64]"""
import argparse
import json
import os
import subprocess
import sys
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
ap.add_argument("--n", type=int, default=2049)
ap.add_argument("--ks", default="1,5,20")
ap.add_argument("--nseq", type=int, default=256)
ap.add_argument("--seqlen", type=int, default=64)
ap.add_argument("--batch-k", type=int, default=20)
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
one = rng.integers(0, spec.vocab_size, a.n).astype(np.int32)
packed = rng.integers(0, spec.vocab_size, a.nseq * a.seqlen).astype(np.int32)
off = np.arange(0, len(packed), a.seqlen, dtype=np.int32)
ln = np.full(a.nseq, a.seqlen, np.int32)
ks = [int(k) for k in a.ks.split(",")]
bk = a.batch_k


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


with lib.DeviceModel(spec, tensors, seq_len=SEQ_LEN) as dm:
    lp, _ = dm.score(one, 0)
    _, g, _ = dm.score_greedy(one, 0)
    same, served = True, []
    for k in ks:
        lpk, ids, _, s = dm.score_topk(one, k, 0)
        same = same and bool(np.array_equal(lp, lpk)) and bool(np.array_equal(ids[:, 0], g))
        served.append(s)
    n = len(packed)
    out_b, out_bk = np.zeros(n, np.float32), np.zeros(n, np.float32)
    top = (np.zeros((n, bk), np.int32), np.zeros((n, bk), np.float32))
    served.append(dm.score_batch_topk(packed, off, ln, bk, out_bk, top)[3])
    dm.score_batch(packed, off, ln, out_b)
    same = same and bool(np.array_equal(out_b, out_bk))
    calls = {"score": lambda: dm.score(one, 0)}
    calls.update({f"k{k}": (lambda k=k: dm.score_topk(one, k, 0)) for k in ks})
    t1 = best_of(calls)
    t2 = best_of({"batch": lambda: dm.score_batch(packed, off, ln, out_b), "batch_topk": lambda: dm.score_batch_topk(packed, off, ln, bk, out_bk, top)})

name, plim = card()
pct = lambda x, p: round(100.0 * (x - p) / p, 2)  # noqa: E731
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": SEQ_LEN, "n": a.n, "nseq": a.nseq, "seqlen": a.seqlen,
    "served": served, "logprobs_bit_identical": same,
    "score_ms": round(t1["score"], 3), "score_topk_ms": {f"k{k}": round(t1[f"k{k}"], 3) for k in ks},
    "score_extra_pct": {f"k{k}": pct(t1[f"k{k}"], t1["score"]) for k in ks},
    "batch_k": bk, "batch_ms": round(t2["batch"], 3), "batch_topk_ms": round(t2["batch_topk"], 3), "batch_extra_pct": pct(t2["batch_topk"], t2["batch"]),
    "reps": a.reps, "gpu": name, "power_limit_w": plim}))
