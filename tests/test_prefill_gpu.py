"""The batched prompt pass (forward_prefill_cuda: wgmma GEMMs + block-causal attention, SURVEY.md s.8f row 1) against
the path it replaces: n serial forward(FF_UPDATE_KV_ONLY) calls (reference run.c:206-209).  The parity contract is the
KV cache -- every layer, positions across the block -- and the logits of the token that follows, also against the CPU
oracle.  Shapes: the smallest the pass serves, all three weight formats, both cache types, a bias / wide-head variant,
partial token tiles, a block that starts in the middle of a context, and Llama-3-8B's own widths."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import KV_ATOL, KV_RTOL, TOL_SIGMA  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY  # noqa: E402

pytestmark = pytest.mark.gpu


def _both(spec, tensors, toks, pos0, seq_len, kvbits, warm=()):
    """(serial, batched): logits of the token after the block and a sample of cache entries."""
    out = []
    nxt = int(toks[-1])
    for batched in (False, True):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
            for i, t in enumerate(warm):
                dm.forward(int(t), i, FF_UPDATE_KV_ONLY)
            if batched:
                assert dm.prefill(toks[:-1], pos0) == 1, "the tensor-core pass did not serve this shape"
            else:
                for i, t in enumerate(toks[:-1]):
                    dm.forward(int(t), pos0 + i, FF_UPDATE_KV_ONLY)
            logits = dm.forward(nxt, pos0 + len(toks) - 1)
            n = len(toks) - 1
            kv = [dm.read_kv(l, p) for l in range(spec.n_layers) for p in sorted({pos0, pos0 + n // 3, pos0 + n // 2, pos0 + n - 1})]
        out.append((logits, kv))
    return out


def _check(spec, serial, batched, kvbits, label):
    (ls, kvs), (lb, kvb) = serial, batched
    sigma = float(ls.std())
    err = float(np.abs(lb - ls).max())
    tol = TOL_SIGMA if kvbits == 16 else 4e-2
    print(f"{label}: next-token |batched - serial| {err:.2e} = {err / sigma:.1e} sigma")
    assert err <= tol * sigma
    for (ks, vs), (kb, vb) in zip(kvs, kvb):
        if kvbits == 16:
            # entries are fp16 roundings of sums whose noise scales with the vector, not with the entry: two orders of summation may land
            # one fp16 ulp of the LARGEST entries apart on a small entry of a deeper layer (KV_ATOL was sized for sigma ~ 0.3 models)
            np.testing.assert_allclose(kb, ks, rtol=KV_RTOL, atol=max(KV_ATOL, 5e-4 * float(np.abs(ks).max())))
            np.testing.assert_allclose(vb, vs, rtol=KV_RTOL, atol=max(KV_ATOL, 5e-4 * float(np.abs(vs).max())))
        else:  # e5m2 entries: equal or neighbouring values
            for a, b in ((kb, ks), (vb, vs)):
                assert (np.abs(a - b) <= 0.26 * np.maximum(np.abs(a), np.abs(b)) + 2e-5).all() and (a == b).mean() > 0.95


@pytest.mark.parametrize("name,dtype,kvbits,n", [("pf-tiny", "fp8", 16, 40), ("pf-tiny", "fp16", 16, 129), ("pf-tiny", "gf4", 16, 300), ("pf-tiny", "fp8", 8, 131),
                                                  ("pf-tiny-hd128", "fp8", 16, 257), ("pf-tiny-hd128", "gf4", 8, 64)])
def test_prefill_matches_serial_prompt_and_oracle(oracle_pkg, name, dtype, kvbits, n):
    spec = replace(mg.SPECS[name], dtype=dtype)
    host = mg.HostModel(spec, seed=3, kvbits=kvbits)
    toks = mg.teacher_tokens(spec.vocab_size, n + 1)
    serial, batched = _both(spec, host.tensors, toks, 0, None, kvbits)
    _check(spec, serial, batched, kvbits, f"{name}/{dtype}/kv{kvbits}/n{n}")
    ck = oracle_pkg.Checker("port")
    ck.prepare(host)
    for i, t in enumerate(toks[:-1]):
        ck.forward(host, int(t), i, FF_UPDATE_KV_ONLY)
    want = ck.forward(host, int(toks[-1]), n)
    ck.release(host)
    tol = TOL_SIGMA if kvbits == 16 else 4e-2
    assert np.abs(batched[0] - want).max() <= tol * want.std()


def test_prefill_in_the_middle_of_a_context():
    """pos0 > 0: the block attends to what is already cached (a chat's second turn, run.c:349-419)."""
    spec = mg.SPECS["pf-tiny"]
    host = mg.HostModel(spec, seed=4)
    warm = mg.teacher_tokens(spec.vocab_size, 37, start=500)
    toks = mg.teacher_tokens(spec.vocab_size, 150)
    serial, batched = _both(spec, host.tensors, toks, len(warm), None, 16, warm=warm)
    _check(spec, serial, batched, 16, "pf-tiny, pos0 = 37")


def test_prefill_falls_back_for_unsupported_shapes():
    """head_dim 32 (tiny-fp8), MoE: forward_prefill_cuda returns 0 and feeds the tokens one by one -- identical to the serial path."""
    for name in ("tiny-fp8", "tiny-moe"):
        spec = mg.SPECS[name]
        host = mg.HostModel(spec, seed=0)
        toks = mg.teacher_tokens(spec.vocab_size, 20)
        with lib.DeviceModel(spec, host.tensors) as dm:
            assert dm.prefill(toks[:-1], 0) == 0
            a = dm.forward(int(toks[-1]), len(toks) - 1)
        with lib.DeviceModel(spec, host.tensors) as dm:
            for i, t in enumerate(toks[:-1]):
                dm.forward(int(t), i, FF_UPDATE_KV_ONLY)
            b = dm.forward(int(toks[-1]), len(toks) - 1)
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("workload,n", [("llama3-8b-fp8", 300), ("mistral-7b-gf4", 200)])
def test_prefill_at_reference_widths(workload, n):
    """Llama-3-8B / Mistral-7B widths (dim 4096, hidden 14336, 32/8 heads of 128) at two layers, a block with a partial tile."""
    spec = replace(mg.SPECS[workload], n_layers=2, vocab_size=4096)
    tensors = mg.generate(spec, 0, device="cuda")
    torch.cuda.synchronize()
    toks = mg.teacher_tokens(spec.vocab_size, n + 1)
    serial, batched = _both(spec, tensors, toks, 0, 1024, 16)
    _check(spec, serial, batched, 16, f"{workload} widths, 2 layers, n = {n}")
