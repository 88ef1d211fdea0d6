#!/usr/bin/env python
"""Same-box comparison through the REFERENCE DRIVER (unmodified run.c + tensors.c + tokenizer.c + sampler.c):

  oracle/_ref/run_ref   reference program with its own CUDA backend (src/infer.cu, compiled for sm_90a)
  oracle/_ref/run_b200  the same reference program linked against libcalm_b200.so (the drop-in)

Writes the synthetic model as a .calm file (calm_b200.modelgen.write_calm) into /dev/shm, runs both binaries with
the reference's own protocol (README.md:86: first tokens at pos 0.., last tokens with CALM_POSO) and prints the
reference's stats lines (run.c:249-253).  Usage: python tools/ref_cuda_bench.py [workload] [n_tokens]"""
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from calm_b200 import modelgen as mg  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "llama3-8b-fp8"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 64
spec = mg.SPECS[name]
path = f"/dev/shm/{name}.calm"
t0 = time.time()
dev = "cuda" if torch.cuda.is_available() else "cpu"
tensors = mg.generate(spec, 0, device=dev)
tensors = {k: v.cpu() for k, v in tensors.items()}
mg.write_calm(path, spec, tensors)
del tensors
print(f"# wrote {path} ({os.path.getsize(path) / 1e9:.2f} GB) in {time.time() - t0:.1f} s", flush=True)

out = {}
for binary in ("run_ref", "run_b200"):
    exe = os.path.join(ROOT, "oracle", "_ref", binary)
    if not os.path.exists(exe):
        print(f"# {binary}: not built", flush=True)
        continue
    for label, poso in (("first", None), ("last", str(4096 - n - 8))):
        env = dict(os.environ, CALM_B200_QUIET="1")
        env.pop("CALM_CPU", None)
        if poso:
            env["CALM_POSO"] = poso
        r = subprocess.run([exe, path, "-n", str(n), "-t", "0", "-i", "<|t5|>"], capture_output=True, text=True, env=env, timeout=600)
        m = re.search(r"throughput: ([0-9.]+) tok/s; latency: ([0-9.]+) ms/tok; bandwidth: ([0-9.]+) GB/s.*#([0-9a-f]+)", r.stderr)
        key = f"{binary} {label}"
        if m:
            out[key] = {"tok_s": float(m.group(1)), "ms_tok": float(m.group(2)), "gbs": float(m.group(3)), "hash": m.group(4)}
            print(f"{key:34s} {m.group(1):>8s} tok/s  {m.group(2):>7s} ms/tok  {m.group(3):>8s} GB/s  #{m.group(4)}  tokens: {r.stdout.strip()[:60]}", flush=True)
        else:
            print(f"{key}: rc={r.returncode} stderr tail: {r.stderr[-300:]}", flush=True)
os.remove(path)
print(json.dumps(out))
