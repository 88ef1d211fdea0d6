#!/usr/bin/env python
"""Store what the tests that compare against the reference project compared against, so that they run anywhere.

  python tools/make_reference_golden.py                 -> tests/golden/reference-cpu.npz
      the reference CPU backend (oracle/_ref/libcalm_ref_cpu.so) teacher-forced on the cases of
      test_oracle.py and test_parity_gpu.py, and the reference program (oracle/_ref/run_ref, its CPU path) decoding
      .calm files written by modelgen.write_calm (test_oracle.py, test_dropin_gpu.py)
  python tools/make_reference_golden.py --cuda DIR      -> tests/golden/reference-cuda.npz
      a seeded sample of the logits tools/ref_cuda_worker.py saved in DIR (the reference CUDA backend on an H100, the
      runs test_scale_gpu.py lists in REF_CUDA_RUNS); the full vocabulary of the 8B shape does not fit the 1 MB file limit

Needs oracle/_ref, i.e. `build()` on a machine where the reference sources are present.
"""
import hashlib
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
# (key, spec, seed, n_tokens, first token index, seq_len)
CPU_RUNS = [("live-" + n, n, 3, 12, 100, None) for n in ("tiny-fp8", "tiny-gf4", "tiny-qwen", "tiny-moe")] + \
           [("rolling-tiny-fp8", "tiny-fp8", 1, 40, 0, 16)] + \
           [("parity-" + n, n, 5, 20, 50, None) for n in ("tiny-llama", "tiny-moe", "tiny-gf4")]
# (key, spec, tokens to generate): the reference program on a written .calm file, prompt <|t7|><|t8|>, greedy
DRIVER_RUNS = [("driver-tiny-fp8", "tiny-fp8", 8)] + [("dropin-" + n, n, 12) for n in ("tiny-llama", "tiny-gf4", "tiny-moe")]
SAMPLE = 4096  # logits kept per position of a reference CUDA run


def calm_file(spec, path):
    mg.write_calm(path, spec, mg.HostModel(spec, seed=0).tensors)
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def driver_tokens(path, n):
    exe = os.path.join(ROOT, "oracle", "_ref", "run_ref")
    r = subprocess.run([exe, path, "-n", str(n), "-t", "0", "-i", "<|t7|><|t8|>"], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CALM_CPU="1", OMP_NUM_THREADS="2"), check=True)
    assert "tok/s" in r.stderr
    return np.array([int(t) for t in re.findall(r"<\|t(\d+)\|>", r.stdout.rstrip("\n").split("\n")[-1])], np.int32)


def make_cpu():
    oracle.build(ref=True)
    out = {}
    for key, name, seed, n, start, seq_len in CPU_RUNS:
        spec = mg.SPECS[name]
        model = mg.HostModel(spec, seed=seed, seq_len=seq_len)
        out[key] = oracle.teacher_forced(oracle.Checker("reference"), model, mg.teacher_tokens(spec.vocab_size, n, start=start)).astype(np.float32)
    with tempfile.TemporaryDirectory() as d:
        for key, name, n in DRIVER_RUNS:
            path = os.path.join(d, name + ".calm")
            out[key + "-sha256"] = np.array(calm_file(mg.SPECS[name], path))
            out[key + "-tokens"] = driver_tokens(path, n)
    np.savez_compressed(os.path.join(GOLDEN, "reference-cpu.npz"), **out)


def make_cuda(src):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_scale_gpu import REF_CUDA_RUNS

    out = {}
    for key, spec_name, *_ in REF_CUDA_RUNS:
        logits = np.load(os.path.join(src, key + ".npz"))["logits"]
        idx = np.sort(np.random.default_rng(0).choice(logits.shape[1], min(SAMPLE, logits.shape[1]), replace=False))
        srt = np.sort(logits, axis=1)
        out[key + "-idx"] = idx.astype(np.int32)
        out[key + "-logits"] = logits[:, idx].astype(np.float32)
        out[key + "-std"] = logits.std(axis=1).astype(np.float64)
        out[key + "-argmax"] = logits.argmax(1).astype(np.int32)
        out[key + "-margin"] = (srt[:, -1] - srt[:, -2]).astype(np.float32)
    np.savez_compressed(os.path.join(GOLDEN, "reference-cuda.npz"), **out)


if __name__ == "__main__":
    if "--cuda" in sys.argv:
        make_cuda(sys.argv[sys.argv.index("--cuda") + 1])
    else:
        make_cpu()
