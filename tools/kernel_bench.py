#!/usr/bin/env python
"""Per-kernel roofline of the stand-alone matvec kernel (calm_b200_matvec) on matrices larger than L2.

  python tools/kernel_bench.py [--iters 20]            # prints one JSON line per (format, shape)
Timed with CUDA events around the kernel over many launches."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--formats", default="8,16,4")
    ap.add_argument("--shapes", default="4096x65536,14336x16384")  # n x d; >= 256 MB in fp8
    args = ap.parse_args()
    peak = 6583.5
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    g = torch.Generator(device="cuda").manual_seed(0)
    for dbits in [int(x) for x in args.formats.split(",")]:
        for shp in args.shapes.split(","):
            n, d = [int(x) for x in shp.split("x")]
            dtype = {16: "fp16", 8: "fp8", 4: "gf4"}[dbits]
            w = torch.empty((d, n * dbits // 8), dtype=torch.uint8, device="cuda")
            for r0 in range(0, d, 8192):
                blk = 0.02 * torch.randn((min(8192, d - r0), n), generator=g, device="cuda")
                w[r0:r0 + blk.shape[0]] = mg.quantize(blk, dtype).view(torch.uint8).reshape(blk.shape[0], -1)
            x = np.random.default_rng(0).standard_normal(n).astype(np.float32)
            y, ms = lib.matvec(dbits, w.data_ptr(), x, n, d, args.warmup, args.iters)
            nbytes = d * n * dbits / 8
            print(json.dumps({"kernel": f"k_matvec<{dbits}>", "n": n, "d": d, "mbytes": nbytes / 1e6, "us": ms * 1e3,
                              "gbs": nbytes / 1e9 / (ms / 1e3), "frac_of_measured_peak": nbytes / 1e9 / (ms / 1e3) / peak,
                              "checksum": float(np.abs(y).sum())}), flush=True)
            del w


if __name__ == "__main__":
    main()
