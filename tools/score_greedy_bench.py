#!/usr/bin/env python
"""Time the greedy scoring calls against their plain siblings on the same inputs, and record what a draft-verification
pass costs.  Prints one JSON line:
  score_ms / score_greedy_ms               calm_b200_score vs calm_b200_score_greedy on one --n-token sequence
  batch_ms / batch_greedy_ms               calm_b200_score_batch vs calm_b200_score_batch_greedy on --nseq sequences of
                                           --seqlen tokens (the workload of profiles/h100_score_batch_llama3-8b-fp8.jsonl)
  *_extra_pct                              (greedy - plain) / plain in percent
  verify_ms[k] / forward_argmax_ms         (information only) calm_b200_score_greedy of k + 2 tokens at pos0 = --pos, beside
                                           one calm_b200_forward_argmax at that position
Each figure is the best of --reps, the calls of a pair alternating, after one warm-up of every shape; CUDA events on the
library's stream.  Card name and power limit come from a query-only nvidia-smi.
  python tools/score_greedy_bench.py [--workload llama3-8b-fp8] [--layers 32] [--n 2049] [--nseq 256] [--seqlen 64]"""
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
ap.add_argument("--nseq", type=int, default=256)
ap.add_argument("--seqlen", type=int, default=64)
ap.add_argument("--pos", type=int, default=2048)
ap.add_argument("--drafts", default="1,3,7,15")
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
drafts = [int(k) for k in a.drafts.split(",")]


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
    lpg, g, served_one = dm.score_greedy(one, 0)
    same = bool(np.array_equal(lp, lpg))
    out_b, out_bg, g_b = np.zeros(len(packed), np.float32), np.zeros(len(packed), np.float32), np.zeros(len(packed), np.int32)
    served_batch = dm.score_batch_greedy(packed, off, ln, out_bg, g_b)[2]
    dm.score_batch(packed, off, ln, out_b)
    same = same and bool(np.array_equal(out_b, out_bg))
    t1 = best_of({"score": lambda: dm.score(one, 0), "score_greedy": lambda: dm.score_greedy(one, 0)})
    t2 = best_of({"batch": lambda: dm.score_batch(packed, off, ln, out_b), "batch_greedy": lambda: dm.score_batch_greedy(packed, off, ln, out_bg, g_b)})
    # draft verification at pos0 = --pos on a cache the --n-token score left (its first --pos slots are that sequence's)
    verify = {f"k{k}": (lambda k=k: dm.score_greedy(one[:k + 2], a.pos)) for k in drafts}
    verify["forward_argmax"] = lambda: dm.forward_argmax(int(one[0]), a.pos)
    t3 = best_of(verify)

name, plim = card()
pct = lambda g, p: round(100.0 * (g - p) / p, 2)  # noqa: E731
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": SEQ_LEN, "n": a.n, "nseq": a.nseq, "seqlen": a.seqlen,
    "served": [served_one, served_batch], "logprobs_bit_identical": same,
    "score_ms": round(t1["score"], 3), "score_greedy_ms": round(t1["score_greedy"], 3), "score_extra_pct": pct(t1["score_greedy"], t1["score"]),
    "batch_ms": round(t2["batch"], 3), "batch_greedy_ms": round(t2["batch_greedy"], 3), "batch_extra_pct": pct(t2["batch_greedy"], t2["batch"]),
    "verify_pos0": a.pos, "verify_ms": {k: round(v, 3) for k, v in t3.items() if k != "forward_argmax"},
    "forward_argmax_ms": round(t3["forward_argmax"], 3), "reps": a.reps, "gpu": name, "power_limit_w": plim}))
