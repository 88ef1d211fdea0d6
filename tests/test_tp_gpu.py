"""Tensor parallelism on 2 / 4 / 8 GPUs (SURVEY.md s.8e): one process per GPU, each given the FULL model through the
reference boundary plus calm_b200_tp_init; every rank must return the full logits, equal to the single-device reference
fixtures within the stated tolerance, and all ranks must agree bit for bit (they sample independently).  Covers the fused
matvec -> all-reduce inside k_matres, the vocabulary-split classifier with its NVLink gather, and MoE expert slices.
Cases whose world size exceeds the visible GPUs are skipped (tools/tp_round.sh N runs them on N GPUs)."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT, TOL_SIGMA, golden  # noqa: E402

from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu


def _gpus():
    import torch

    return torch.cuda.device_count()


def _run_world(tmp_path, name, world, fused, tokens, greedy=12):
    out = str(tmp_path / "tp")
    idfile = str(tmp_path / "nccl.id")
    env = dict(os.environ, PYTHONPATH=ROOT, CALM_B200_QUIET="1", CALM_B200_TP_FUSED=str(fused))
    procs = [subprocess.Popen([sys.executable, "-m", "calm_b200.tp", "--spec", name, "--rank", str(r), "--world", str(world), "--idfile", idfile,
                               "--tokens", str(tokens), "--out", out, "--greedy", str(greedy)], cwd=ROOT, env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(world)]
    logs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=300)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            pytest.fail("tensor-parallel worker hung")
        logs.append(o)
    assert all(p.returncode == 0 for p in procs), "\n".join(l[-1500:] for l in logs)
    return [np.load(f"{out}.rank{r}.npz") for r in range(world)]


CASES = [("tiny-fp8", 2, 1), ("tiny-gf4", 2, 1), ("tiny-bias2", 2, 1), ("tiny-lnpar", 2, 1), ("tiny-mha", 2, 1), ("tiny-fp8", 2, 0), ("tiny-bias2", 2, 0),
         ("tiny-moe", 2, 1), ("ring-tp", 2, 1), ("tiny-tp8", 2, 1), ("ring-tp", 4, 1), ("tiny-tp8", 4, 1), ("tiny-tp8-moe", 4, 1), ("tiny-tp8", 4, 0), ("tiny-tp8", 8, 1), ("tiny-tp8-moe", 8, 1), ("tiny-tp8", 8, 0)]


@pytest.mark.parametrize("name,world,fused", CASES)
def test_ranks_match_single_device_reference(tmp_path, name, world, fused):
    """fused=1: partial sums exchanged inside k_matres over peer memory, classifier split by vocabulary;
    fused=0: ncclAllReduce between kernels, replicated classifier."""
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    spec = mg.SPECS[name]
    g = golden(name)
    res = _run_world(tmp_path, name, world, fused, len(g["tokens"]))
    r0 = res[0]
    assert int(r0["world"]) == world
    for r in res:
        assert int(r["mode"]) == (2 if fused else 1), "peer-memory exchange not in use"
        assert np.array_equal(r0["logits"], r["logits"])      # every rank holds the same full logits
        assert np.array_equal(r0["greedy"], r["greedy"])      # so independent greedy sampling stays in lock step
    steps = list(g["steps"])
    ref = g["logits"]
    sigma = float(ref.std())
    err = float(np.abs(r0["logits"][steps] - ref).max())
    print(f"{name} tp{world} fused={fused}: |tp - reference| {err:.2e} = {err / sigma:.1e} sigma")
    assert err <= TOL_SIGMA * sigma, (err, sigma)
    clear = g["margin"] > 2 * TOL_SIGMA * sigma
    assert np.array_equal(r0["logits"].argmax(1)[clear], g["argmax"][clear])
    assert spec.vocab_size == r0["logits"].shape[1]
