#!/usr/bin/env python
"""Time calm_b200_score_batch (many independent sequences packed into shared prompt-pass blocks) against one
calm_b200_score call per sequence, on two workloads.  Prints one JSON line:
  study_*   an --text-token text in study() chunks of --steps positions (chunk c: off = c * steps, len = steps + 1)
  short_*   --nseq sequences of --seqlen tokens each
  *_loop_ms / *_loop_pos_s     one calm_b200_score per sequence (pos0 = 0), back to back
  *_batch_ms / *_batch_pos_s   one calm_b200_score_batch over all of them
  *_speedup                    loop_ms / batch_ms
CUDA events on the library's stream, best of --reps after a warm-up at the timed size; a position is one scored token.
Card name and power limit come from a query-only nvidia-smi.
  python tools/score_batch_bench.py [--workload llama3-8b-fp8] [--layers 32] [--text 8193] [--steps 256] [--nseq 256] [--seqlen 64]"""
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
ap.add_argument("--text", type=int, default=8193)
ap.add_argument("--steps", type=int, default=256)
ap.add_argument("--nseq", type=int, default=256)
ap.add_argument("--seqlen", type=int, default=64)
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

off_study = np.arange(0, a.text - 1, a.steps, dtype=np.int32)
workloads = {
    "study": (np.array(mg.teacher_tokens(spec.vocab_size, a.text), np.int32), off_study,
              np.minimum(a.steps + 1, a.text - off_study).astype(np.int32)),
    "short": (np.array(mg.teacher_tokens(spec.vocab_size, a.nseq * a.seqlen, start=a.text), np.int32),
              np.arange(0, a.nseq * a.seqlen, a.seqlen, dtype=np.int32), np.full(a.nseq, a.seqlen, np.int32)),
}
res = {"workload": spec.name, "layers": spec.n_layers, "seq_len": 4096}
with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
    def timed(fn):
        fn()  # warm-up at the timed size
        best = 1e9
        for _ in range(a.reps):
            L.calm_b200_timer_start()
            fn()
            best = min(best, L.calm_b200_timer_stop())
        return best

    for name, (toks, off, lens) in workloads.items():
        positions = int((lens - 1).sum())
        out = np.zeros(len(toks), np.float32)

        def loop():
            served = 1
            for o, n in zip(off, lens):
                served &= dm.score(toks[o:o + n], 0)[1]
            return served

        served_loop = loop()
        served_batch = dm.score_batch(toks, off, lens, out)[1]
        loop_ms = timed(loop)
        batch_ms = timed(lambda: dm.score_batch(toks, off, lens, out))
        res.update({f"{name}_sequences": len(off), f"{name}_seq_tokens": int(lens.max()), f"{name}_positions": positions,
                    f"{name}_served": [served_loop, served_batch],
                    f"{name}_loop_ms": round(loop_ms, 2), f"{name}_loop_pos_s": round(positions / loop_ms * 1e3, 1),
                    f"{name}_batch_ms": round(batch_ms, 2), f"{name}_batch_pos_s": round(positions / batch_ms * 1e3, 1),
                    f"{name}_speedup": round(loop_ms / batch_ms, 2)})
name, plim = card()
res.update({"gpu": name, "power_limit_w": plim})
print(json.dumps(res))
