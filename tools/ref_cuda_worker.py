#!/usr/bin/env python
"""Run the UNMODIFIED reference CUDA backend (oracle/_ref/libcalm_ref_cuda.so = reference src/infer.cu compiled for
sm_90a by oracle/Makefile) on a seeded synthetic model and save its logits: the at-scale oracle of the GPU parity
tests (tests/test_scale_gpu.py).  TEST INFRASTRUCTURE ONLY; runs in its own process because the reference keeps global
state and abort()s on errors.

  python tools/ref_cuda_worker.py --spec llama3-8b-fp8 --seq-len 4096 --kvbits 16 --tokens 4096 --keep 63,1023,2047,4095 --out ref.npz
  [--layers N] [--fill-pos P --fill-seed S]   (teacher forcing starts at P on a cache pre-filled by the numpy pattern)

Feeds tok_i = (7919 i + 13) mod vocab at positions start..start+tokens-1 (FF_UPDATE_KV_ONLY except at kept steps) and
stores logits[keep].  Mirrors what reference run.c does around its backend (upload -> prepare_cuda -> forward)."""
import argparse
import ctypes as C
import os
import sys
from dataclasses import replace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY, Transformer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spec", required=True)
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--seq-len", type=int, default=None)
    ap.add_argument("--kvbits", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--tokens", type=int, default=0)
    ap.add_argument("--keep", default="")
    ap.add_argument("--out", default="")
    ap.add_argument("--bench", default="", help="pos0,warmup,steps: time forward_cuda (host token in, host logits out, host argmax) and print one JSON line")
    a = ap.parse_args()
    import torch

    spec = mg.SPECS[a.spec]
    if a.layers:
        spec = replace(spec, n_layers=a.layers)
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libcalm_ref_cuda.so"))
    T = C.POINTER(Transformer)
    lib.prepare_cuda.argtypes, lib.prepare_cuda.restype = [T], None
    lib.forward_cuda.argtypes, lib.forward_cuda.restype = [T, C.c_int, C.c_int, C.c_uint], C.POINTER(C.c_float)
    tensors = mg.generate(spec, a.seed, device="cuda")  # struct Weights carries device pointers after upload_cuda anyway
    torch.cuda.synchronize()
    t = mg.fill_transformer(spec, lambda n: tensors[n].data_ptr() if n in tensors else 0, a.seq_len, a.kvbits)
    lib.prepare_cuda(C.byref(t))
    if a.bench:
        import json
        import time

        pos0, W, K = (int(x) for x in a.bench.split(","))
        tok = 23
        for i in range(W):
            p = lib.forward_cuda(C.byref(t), tok, pos0 + i, 0)
            tok = int(np.argmax(np.ctypeslib.as_array(p, shape=(spec.vocab_size,))))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(K):
            p = lib.forward_cuda(C.byref(t), tok, pos0 + W + i, 0)  # synchronises itself (infer.cu:734)
            tok = int(np.argmax(np.ctypeslib.as_array(p, shape=(spec.vocab_size,))))
        dt = time.perf_counter() - t0
        print(json.dumps({"tok_s": K / dt, "ms_per_step": dt / K * 1e3, "steps": K, "pos0": pos0 + W}), flush=True)
        os._exit(0)
    keep = [int(x) for x in a.keep.split(",")]
    toks = mg.teacher_tokens(spec.vocab_size, a.tokens)
    out = {}
    for i, tok in enumerate(toks):
        p = lib.forward_cuda(C.byref(t), tok, i, 0 if i in keep else FF_UPDATE_KV_ONLY)
        if i in keep:
            out[i] = np.ctypeslib.as_array(p, shape=(spec.vocab_size,)).copy()
    np.savez(a.out, keep=np.array(keep, np.int32), logits=np.stack([out[i] for i in keep]))
    os._exit(0)  # the reference never frees (run.c:636); skip interpreter teardown of its statics


if __name__ == "__main__":
    main()
