#!/usr/bin/env python
"""Time calm_b200_score (perplexity scoring in the batched prompt pass) against the serial way of scoring, one
forward_cuda per position plus a log-softmax on the host (the reference's study(), run.c:291-308).  Prints one JSON line:
  score_ms / score_tok_s   calm_b200_score over --tokens tokens (tokens - 1 scored positions), CUDA events on the library's
                           stream, best of --reps after a warm-up at the timed size
  prefill_ms               forward_prefill_cuda over the same tokens - 1 rows, same run
  cls_ms / cls_tflops      the classifier leg: score_ms - prefill_ms, and 2 n vocab dim over it
  serial_ms_per_pos        forward_cuda + float64 log-softmax of the logits on the host, mean over --serial positions
  speedup                  serial_ms_per_pos * (tokens - 1) / score_ms
  gpu, power_limit_w       from a query-only nvidia-smi
  python tools/score_bench.py [--workload llama3-8b-fp8] [--layers 32] [--tokens 2049] [--serial 256]"""
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
ap.add_argument("--tokens", type=int, default=2049)
ap.add_argument("--serial", type=int, default=256)
ap.add_argument("--reps", type=int, default=3)
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
toks = np.array(mg.teacher_tokens(spec.vocab_size, a.tokens), np.int32)
n = a.tokens - 1
with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
    def timed(fn):
        fn()  # warm-up at the timed size
        best = 1e9
        for _ in range(a.reps):
            L.calm_b200_timer_start()
            fn()
            best = min(best, L.calm_b200_timer_stop())
        return best

    served = dm.score(toks, 0)[1]
    score_ms = timed(lambda: dm.score(toks, 0))
    prefill_ms = timed(lambda: dm.prefill(toks[:-1], 0))
    dm.forward(int(toks[0]), 0)  # the decode graph is captured before the serial timing
    t0 = time.perf_counter()
    for p in range(a.serial):
        lg = dm.forward(int(toks[p]), p).astype(np.float64)
        mx = lg.max()
        _ = lg[toks[p + 1]] - mx - np.log(np.exp(lg - mx).sum())
    serial_ms = (time.perf_counter() - t0) * 1e3 / a.serial
name, plim = card()
cls_ms = score_ms - prefill_ms
print(json.dumps({"workload": spec.name, "layers": spec.n_layers, "tokens": a.tokens, "positions": n, "served": served,
                  "score_ms": round(score_ms, 2), "score_tok_s": round(n / score_ms * 1e3, 1), "prefill_ms": round(prefill_ms, 2),
                  "cls_ms": round(cls_ms, 2), "cls_tflops": round(2.0 * n * spec.vocab_size * spec.dim / cls_ms / 1e9, 1),
                  "serial_ms_per_pos": round(serial_ms, 3), "serial_positions": a.serial, "speedup": round(serial_ms * n / score_ms, 1),
                  "gpu": name, "power_limit_w": plim}))
