"""calm_b200_score: per-position log-probabilities of a token sequence (the reference's study(), run.c:291-308) from the
batched prompt pass, the classifier as a wgmma GEMM (k_pf_gemm PF_CLS) with its log-softmax fused into the epilogue, and
k_pf_logprob merging each token's per-tile records.

- The stage on its own: the device's own classifier input (the pass's residual rows, read back after the call) through a
  float64 final norm, classifier and log-softmax, at real widths and vocabularies, one layer each.
- Against the path it replaces: one forward_cuda per position and a float64 log-softmax of its logits, plus the KV cache,
  which must be bit for bit what forward_prefill_cuda(tokens[:-1]) leaves; once against the CPU oracle too.
- A 2100-token sequence across the 2048-row block boundary, the decode-path fallback, determinism and the n < 2 edges."""
import ctypes as C
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_stages_gpu import DECODE, make_model, pf_tol  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY  # noqa: E402

pytestmark = pytest.mark.gpu

# Stage bound per position: 2 pf_tol(dim) max |logits of the row| + MERGE_C max(1, |ln sum exp(logits)|).  The logits'
# own error (the GEMM's 22-bit inputs, pf_tol) enters the target's logit and the log-sum-exp once each.  MERGE_C is the
# merge's share: fp32 (max, sum) records of a tile (32 expf terms per lane, two shuffles), their merge over the tiles
# (expf rescaling, lane-strided, then a butterfly) and tgt - M - logf(S) in fp32, a few u of |LSE| and some 32 u of the
# sum.  On an H100 80GB HBM3 (700 W limit) no position of the five cases below erred beyond the GEMM term (measured 0), so,
# as with the sinks of test_stages_gpu.py, MERGE_C is the arithmetic's bound and cannot be tied to a measurement.  The
# largest error was 0.07 of the whole bound (switch-layernorm-par; Llama-3-8B widths 4.0e-5 absolute, 0.06).
MERGE_C = 2e-6


def stage_bound(dim, amax, lse):
    """The bound above per position: amax = max |logits of the row|, lse = ln sum exp(logits)."""
    return 2 * pf_tol(dim) * amax + MERGE_C * np.maximum(1.0, np.abs(lse))


def log_softmax_at(logits, targets):
    """float64 ln softmax(logits[i])[targets[i]] and the row's log-sum-exp; logits[n, vocab] (numpy or torch, any float)."""
    L = torch.as_tensor(logits).to(torch.float64)
    lse = torch.logsumexp(L, dim=1)
    t = torch.as_tensor(np.asarray(targets, np.int64), device=L.device)
    return (L.gather(1, t[:, None])[:, 0] - lse).cpu().numpy(), lse.cpu().numpy()


def serial_logprobs(dm, toks, pos0):
    """One forward_cuda per position (the decode path) and the float64 log-softmax of its logits at the next token."""
    logits = np.stack([dm.forward(int(t), pos0 + i) for i, t in enumerate(toks[:-1])])
    lp, _ = log_softmax_at(logits, toks[1:])
    return lp, logits.std(1)


# ---- 1. the stage, from the device's own input: (spec, kvbits, tokens)
STAGE = {
    "llama3-8b fp8 vocab 128256 n300": (replace(mg.SPECS["llama3-8b-fp8"], n_layers=1), 16, 301),  # 1002 vocabulary tiles, a partial token tile
    "qwen2-0.5b fp16 tied vocab 151936": (replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=1), 16, 200),  # QKV bias, classifier = embedding
    "mistral gf4 vocab 32000 kv8": (replace(mg.SPECS["mistral-7b-gf4"], n_layers=1), 8, 200),
    "pf-tiny vocab 1000": (replace(mg.SPECS["pf-tiny"], n_layers=1, vocab_size=1000), 16, 150),  # a partial vocabulary tile
    "switch-layernorm-par": (DECODE["switch-layernorm-par"][0], 16, 150),  # a LayerNorm final norm
}
worst = {}


@pytest.mark.parametrize("case", sorted(STAGE))
def test_score_stage_against_float64(case):
    spec, kvbits, n = STAGE[case]
    tensors, w = make_model(spec, 7)
    toks = mg.teacher_tokens(spec.vocab_size, n)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        lp, served = dm.score(toks, 0)
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n - 1]
    assert served == 1, f"{case}: the tensor-core pass did not serve this shape"
    xn = torch.as_tensor(sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, spec.norm_type != "rmsnorm"), device="cuda")
    W = w.classifier()
    logits = torch.empty((n - 1, spec.vocab_size), dtype=torch.float64, device="cuda")
    for r in range(0, W.shape[0], 16384):  # float64 on the device, 16384 classifier rows at a time
        logits[:, r:r + 16384] = xn @ torch.as_tensor(W[r:r + 16384], device="cuda").to(torch.float64).T
    ref, lse = log_softmax_at(logits, toks[1:])
    amax = logits.abs().amax(1).cpu().numpy()
    err = np.abs(lp.astype(np.float64) - ref)
    gemm = 2 * pf_tol(spec.dim) * amax
    bound = stage_bound(spec.dim, amax, lse)
    i = int(np.argmax(err / bound))
    excess = float(((err - gemm) / np.maximum(1.0, np.abs(lse))).max())
    worst[case] = (float(err[i] / bound[i]), excess)
    print(f"\n  {case}: max |logprob - float64| {err.max():.2e}; worst {err[i]:.2e} = {err[i] / bound[i]:.2f} of its bound at position {i}"
          f" (max |logit| {amax[i]:.2f}, lse {lse[i]:.2f}); beyond the GEMM term {max(excess, 0):.2e} of max(1, |lse|) (MERGE_C {MERGE_C:.0e})")
    assert np.isfinite(lp).all() and (err <= bound).all(), f"{case}: position {i}: device {lp[i]!r} vs float64 {ref[i]!r}"


# ---- 2. against the serial path and the cache forward_prefill_cuda leaves
SERIAL = [("pf-tiny", "fp8", 16, 40), ("pf-tiny", "fp16", 16, 129), ("pf-tiny", "gf4", 16, 300), ("pf-tiny", "fp8", 8, 300),
          ("pf-tiny", "gf4", 8, 129), ("pf-tiny-hd128", "fp8", 16, 300), ("pf-tiny-hd128", "fp16", 8, 40), ("pf-tiny-hd128", "gf4", 16, 129)]


def _score_vs_serial(spec, tensors, toks, pos0, kvbits, warm, label):
    n = len(toks) - 1
    positions = sorted({pos0, pos0 + n // 3, pos0 + n // 2, pos0 + n - 1})
    runs = []
    for mode in ("serial", "score", "prefill"):
        with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
            for i, t in enumerate(warm):
                dm.forward(int(t), i, FF_UPDATE_KV_ONLY)
            if mode == "serial":
                runs.append(serial_logprobs(dm, toks, pos0))
                continue
            if mode == "score":
                lp, served = dm.score(toks, pos0)
                assert served == 1, f"{label}: the tensor-core pass did not serve this shape"
                runs.append(lp)
            else:
                assert dm.prefill(toks[:-1], pos0) == 1
            runs.append([dm.read_kv(l, p) for l in range(spec.n_layers) for p in positions])
    (want, sigma), lp, kv_score, kv_prefill = runs
    tol = 2 * (TOL_SIGMA if kvbits == 16 else 4e-2) * sigma
    err = np.abs(lp - want)
    i = int(np.argmax(err / tol))
    print(f"  {label}: max |score - serial| {err.max():.2e}; worst {err[i] / tol[i]:.2f} of its bound at position {pos0 + i}")
    assert (err <= tol).all(), f"{label}: position {pos0 + i}: {lp[i]!r} vs serial {want[i]!r}"
    for (ks, vs), (kp, vp) in zip(kv_score, kv_prefill):
        assert np.array_equal(ks, kp) and np.array_equal(vs, vp), f"{label}: the cache after score differs from the prompt pass's"
    return lp


@pytest.mark.parametrize("name,dtype,kvbits,n", SERIAL)
def test_score_matches_serial_and_prompt_pass_cache(name, dtype, kvbits, n):
    spec = replace(mg.SPECS[name], dtype=dtype)
    host = mg.HostModel(spec, seed=3, kvbits=kvbits)
    _score_vs_serial(spec, host.tensors, mg.teacher_tokens(spec.vocab_size, n + 1), 0, kvbits, (), f"{name}/{dtype}/kv{kvbits}/n{n}")


def test_score_on_a_warm_cache():
    """pos0 = 37: the block attends to what is already cached; a caller continuing a context."""
    spec = mg.SPECS["pf-tiny"]
    host = mg.HostModel(spec, seed=4)
    warm = mg.teacher_tokens(spec.vocab_size, 37, start=500)
    _score_vs_serial(spec, host.tensors, mg.teacher_tokens(spec.vocab_size, 151), len(warm), 16, warm, "pf-tiny pos0 37")


def test_score_matches_oracle(oracle_pkg):
    spec = mg.SPECS["pf-tiny"]
    host = mg.HostModel(spec, seed=5)
    toks = mg.teacher_tokens(spec.vocab_size, 65)
    with lib.DeviceModel(spec, host.tensors) as dm:
        lp, served = dm.score(toks, 0)
    assert served == 1
    ck = oracle_pkg.Checker("port")
    ck.prepare(host)
    logits = np.stack([ck.forward(host, int(t), i) for i, t in enumerate(toks[:-1])])
    ck.release(host)
    want, _ = log_softmax_at(logits, toks[1:])
    err = np.abs(lp - want)
    print(f"  pf-tiny vs oracle: max |score - oracle| {err.max():.2e}")
    assert (err <= 2 * TOL_SIGMA * logits.std(1)).all()


# ---- 3. across the 2048-row block boundary
def test_score_across_the_block_boundary():
    """2100 tokens: rows 0..2047 are one block, 2048..2098 the next.  Position 2047's target is the next block's first token."""
    spec = mg.SPECS["pf-tiny"]
    host = mg.HostModel(spec, seed=6)
    toks = mg.teacher_tokens(spec.vocab_size, 2100)
    with lib.DeviceModel(spec, host.tensors, seq_len=4096) as dm:
        lp, served = dm.score(toks, 0)
    assert served == 1 and lp.shape == (2099,)
    with lib.DeviceModel(spec, host.tensors, seq_len=4096) as dm:
        for i, t in enumerate(toks[:2045]):
            dm.forward(int(t), i, FF_UPDATE_KV_ONLY)
        logits = np.stack([dm.forward(int(toks[p]), p) for p in range(2045, 2050)])
    want, _ = log_softmax_at(logits, toks[2046:2051])
    err = np.abs(lp[2045:2050] - want)
    print(f"  positions 2045..2049: |score - serial| {err}")
    assert (err <= 2 * TOL_SIGMA * logits.std(1)).all()


# ---- 4. the decode-path fallback
@pytest.mark.parametrize("name,seq_len,n", [("tiny-moe", None, 20), ("tiny-fp8", None, 20), ("pf-tiny", 64, 80)])
def test_score_falls_back_to_the_decode_path(name, seq_len, n):
    """MoE, head_dim 32, and a block past seq_len (pos0 + n - 1 > seq_len) return 0 and the log-softmax, in double, of the
    logits forward_cuda gives."""
    spec = mg.SPECS[name]
    host = mg.HostModel(spec, seed=0)
    toks = mg.teacher_tokens(spec.vocab_size, n)
    with lib.DeviceModel(spec, host.tensors, seq_len=seq_len) as dm:
        lp, served = dm.score(toks, 0)
    assert served == 0
    with lib.DeviceModel(spec, host.tensors, seq_len=seq_len) as dm:
        want, _ = serial_logprobs(dm, toks, 0)
    np.testing.assert_allclose(lp, want, rtol=1e-6, atol=1e-6)


# ---- 5. determinism and the edges
def test_score_is_deterministic_and_n_below_2_does_nothing():
    spec = mg.SPECS["pf-tiny"]
    host = mg.HostModel(spec, seed=8)
    toks = mg.teacher_tokens(spec.vocab_size, 300)
    with lib.DeviceModel(spec, host.tensors) as dm:
        a, _ = dm.score(toks, 0)
        b, _ = dm.score(toks, 0)
        assert np.array_equal(a, b)
        dm.prefill(toks[:20], 0)
        before = dm.forward(int(toks[20]), 20)
        for k in (0, 1):
            arr = np.array([int(toks[99])] * max(k, 1), np.int32)
            out = np.full(4, 7.0, np.float32)
            served = dm.lib.calm_b200_score(C.byref(dm.transformer), arr.ctypes.data_as(C.POINTER(C.c_int)), k, 5,
                                            out.ctypes.data_as(C.POINTER(C.c_float)))
            assert served == 1 and (out == 7.0).all()
        after = dm.forward(int(toks[20]), 20)
    assert np.array_equal(before, after)


def test_zz_summary_of_stage_errors():
    """Runs last in this file: the largest share of its bound each stage case showed, and the merge's measured share."""
    if not worst:
        pytest.skip("the stage cases did not run in this session")
    print("\n  score stage: " + ", ".join(f"{k} {r:.2f} of bound (beyond GEMM term {max(e, 0):.1e})" for k, (r, e) in sorted(worst.items())))
