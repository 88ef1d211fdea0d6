#!/usr/bin/env python
"""Time calm_b200_score_context (continuations packed after one copy of their context per block) against
calm_b200_score_batch over the same context ++ continuation concatenations, on a multiple-choice workload: --items
contexts of --ctx tokens, each with --choices continuations of --cont tokens, scored as ln p(continuation | context)
(INTEGRATION.md: the context's last token moves into each sequence).  Prints one JSON line:
  rows_context / rows_batch      prompt-pass rows each call computes (counted from the packing), and their blocks
  context_ms / batch_ms          best of --reps, the two calls alternating, after one warm-up of each
  context_pos_s / batch_pos_s    scored continuation positions per second
  speedup                        batch_ms / context_ms
CUDA events on the library's stream; a position is one scored token.  Card name and power limit come from a query-only
nvidia-smi.
  python tools/score_context_bench.py [--workload llama3-8b-fp8] [--layers 32] [--items 64] [--ctx 512] [--choices 4] [--cont 16]"""
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
ap.add_argument("--items", type=int, default=64)
ap.add_argument("--ctx", type=int, default=512)
ap.add_argument("--choices", type=int, default=4)
ap.add_argument("--cont", type=int, default=16)
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


def ceil8(x):
    return -(-x // 8) * 8


def packed_rows(units, cap=min(2048, SEQ_LEN // 8 * 8)):
    """(rows, blocks) of the library's next-fit packing; units: [(context key or None, context rows, sequence rows)]."""
    rows, blocks, used, placed = 0, 0, 0, set()
    for key, rc, r in units:
        need = r + (0 if key in placed else rc)
        if used + need > cap:
            blocks, used, placed = blocks + 1, 0, set()
            need = r + rc
        used, rows = used + need, rows + need
        if key is not None:
            placed.add(key)
    return rows, blocks + (used > 0)


spec = mg.SPECS[a.workload] if a.layers is None else replace(mg.SPECS[a.workload], n_layers=a.layers)
L = lib.load()
tensors = mg.generate(spec, 0, device="cuda")
torch.cuda.synchronize()

# The buffer: item k's context, then its continuations.  score_context: context ctx[:-1], sequence ctx[-1:] ++ continuation.
# score_batch: the same ln p(continuation | context) from each ctx ++ continuation, built in a buffer of its own.
rng = np.random.default_rng(0)
toks, co, cl, off, ln, cat, boff, units_ctx, units_batch = [], [], [], [], [], [], [], [], []
for k in range(a.items):
    ctx = rng.integers(0, spec.vocab_size, a.ctx)
    base = len(toks)
    toks += ctx.tolist()
    for _ in range(a.choices):
        cont = rng.integers(0, spec.vocab_size, a.cont).tolist()
        co.append(base), cl.append(a.ctx - 1), off.append(len(toks)), ln.append(a.cont + 1)
        toks += [int(ctx[-1])] + cont
        boff.append(len(cat)), cat.extend(ctx.tolist() + cont)
        units_ctx.append((k, ceil8(a.ctx - 1), ceil8(a.cont)))
        units_batch.append((None, 0, ceil8(a.ctx + a.cont - 1)))
i32 = lambda x: np.asarray(x, np.int32)  # noqa: E731
toks, co, cl, off, ln, cat, boff = i32(toks), i32(co), i32(cl), i32(off), i32(ln), i32(cat), i32(boff)
blen = np.full(len(boff), a.ctx + a.cont, np.int32)
positions = a.items * a.choices * a.cont
rows_ctx, blocks_ctx = packed_rows(units_ctx)
rows_batch, blocks_batch = packed_rows(units_batch)

with lib.DeviceModel(spec, tensors, seq_len=SEQ_LEN) as dm:
    out_c, out_b = np.zeros(len(toks), np.float32), np.zeros(len(cat), np.float32)
    calls = {"context": lambda: dm.score_context(toks, co, cl, off, ln, out_c)[1],
             "batch": lambda: dm.score_batch(cat, boff, blen, out_b)[1]}
    served = {k: f() for k, f in calls.items()}  # warm-up at the timed size
    # the two calls give the same ln p(continuation | context)
    same = all(np.array_equal(out_c[o:o + a.cont], out_b[b + a.ctx - 1:b + a.ctx - 1 + a.cont]) for o, b in zip(off, boff))
    best = {k: 1e9 for k in calls}
    for _ in range(a.reps):  # alternate, so that clock and thermal drift hits both alike
        for k, f in calls.items():
            L.calm_b200_timer_start()
            f()
            best[k] = min(best[k], L.calm_b200_timer_stop())

name, plim = card()
print(json.dumps({
    "workload": spec.name, "layers": spec.n_layers, "seq_len": SEQ_LEN, "items": a.items, "ctx_tokens": a.ctx,
    "choices": a.choices, "cont_tokens": a.cont, "positions": positions, "served": [served["context"], served["batch"]],
    "bit_identical": bool(same), "rows_context": rows_ctx, "blocks_context": blocks_ctx, "rows_batch": rows_batch,
    "blocks_batch": blocks_batch, "row_ratio": round(rows_batch / rows_ctx, 2),
    "context_ms": round(best["context"], 2), "context_pos_s": round(positions / best["context"] * 1e3, 1),
    "batch_ms": round(best["batch"], 2), "batch_pos_s": round(positions / best["batch"] * 1e3, 1),
    "speedup": round(best["batch"] / best["context"], 2), "reps": a.reps, "gpu": name, "power_limit_w": plim}))
