#!/usr/bin/env python
"""A/B sweeps of engine knobs in ONE process (one model generation, one box): for every environment setting in the list,
prepare the model, time a device-resident greedy run at the end of the context, and print the in-kernel per-stage table.

  python tools/sweep.py [--workload llama3-8b-fp8] [--steps 64] [--set NAME=VAL,NAME=VAL ...]...

Each --set is one configuration (comma-separated env assignments; "base" = no overrides)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="llama3-8b-fp8")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--set", action="append", default=[])
    ap.add_argument("--kvbits", type=int, default=16)
    a = ap.parse_args()
    from dataclasses import replace

    spec = mg.SPECS[a.workload]
    if a.layers:
        spec = replace(spec, n_layers=a.layers)
    os.environ.setdefault("CALM_B200_QUIET", "1")
    L = lib.load()
    tensors = mg.generate(spec, 0, device="cuda")
    torch.cuda.synchronize()
    seq_len = 4096
    K, W = a.steps, 8
    pos0 = seq_len - K - W
    for cfg in (a.set or ["base"]):
        env = {} if cfg == "base" else dict(kv.split("=", 1) for kv in cfg.split(";"))
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            dm = lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=a.kvbits)
            dm.fill_kv(pos0, seed=1)
            dm.decode_greedy(17, pos0, W)
            best = 1e9
            for rep in range(3):
                L.calm_b200_timer_start()
                dm.decode_greedy(23, pos0 + W, K)
                best = min(best, L.calm_b200_timer_stop() / K)
            stats, span = dm.profile(23, seq_len - 16, 8)
            import ctypes as C
            dbg = (C.c_ulonglong * 16)()
            L.calm_b200_debug_stamps(dbg)
            d = [int(x) for x in dbg]
            attn_dbg = {"entry->wait": d[1] - d[0], "wait->q": d[2] - d[1], "q->first_block": d[3] - d[2], "loop": d[4] - d[3], "q->all_blocks_landed": d[8] - d[2], "loop_after_all_blocks": d[4] - d[8],
                        "loop_scores_softmax": d[11] - d[3], "loop_values": d[4] - d[11], "tail": d[7] - d[4], "tail_publish_wait_ml_coef": d[6] - d[4], "tail_outputs": d[7] - d[6],
                        "first_start->last_end": d[9] - d[10], "cta0_start_after_first": d[1] - d[10]} if d[1] else None
            dm.close()
            row = {k: round(v[0] / max(v[2], 1) * 1e3, 2) for k, v in stats.items() if v[2]}
            print(json.dumps({"cfg": cfg, "ms_per_token": round(best, 4), "tok_s": round(1e3 / best, 1), "span_us_profiled": round(span * 1e3, 1), "us_per_launch": row, "attn_dbg_ns": attn_dbg}), flush=True)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v


if __name__ == "__main__":
    main()
