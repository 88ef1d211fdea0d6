"""The prompt pass stage by stage against float64 at the shapes test_prefill_every_stage does not reach: prompts of several
2048-row blocks, full blocks, deep warm caches, a prompt that ends at the cache's last slot, Llama-3-70B and Qwen2-0.5B
widths, the scoring classifier over a full block at a real vocabulary, and activations at the spread of scales real
checkpoints carry.

The method is test_stages_gpu.py's: a one-layer model, each stage read back with calm_b200_read_state and compared with
tests/stage_ref.py fed the DEVICE's own output of the stage before it, under the same bounds (STAGE_TOL, pf_tol).  Two
things differ because of the sizes:

- A call of more than 2048 rows runs in blocks (pf_pass, engine.cu): block b holds rows 2048 b .. at cache slots
  pos0 + 2048 b ..  and reuses the same buffers, so afterwards the pf_* buffers' first m = n - 2048 floor((n - 1) / 2048)
  rows are the LAST block's.  Every cache entry the call wrote, in every block, is checked against float64 q / k / v of
  the exact embedding rows at their positions (with one layer, QKV's input is the embedding for every block).  The last
  block's Q, attention output, hidden and residual rows are checked on a row subset: every row of its first and last
  128-row token tile, rows 0, 127, 128, 255 and m - 1, and 34 rows spread evenly over the block.  Its attention is
  referenced over the device's cache slots [0, its slot], so the earlier blocks' keys are read as the device wrote them.
- The float64 matrix products run on the GPU: stage_ref.matvec is swapped for a torch float64 product on the device (the
  70B-width DOWN alone is 10^11 multiply-adds for 200 rows); norms, RoPE, activations and the attention stay stage_ref's
  numpy code.

Every case prints its wall time; the last test prints each stage's largest error beside its bound."""
import os
import sys
import time
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
import test_stages_gpu as ts  # noqa: E402
from test_score_gpu import log_softmax_at, stage_bound  # noqa: E402
from test_stages_gpu import DECODE, L8B, V4K, check_decode_step, check_entries, layer_cache, make_model, pf_tol, report  # noqa: E402
from test_variants_gpu import GROUPINGS, plan_of  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

BLOCK = 2048  # rows per block of the pass (pf_pass, engine.cu)
worst = {}  # this file's largest error per stage key, (error, bound, share)
score_worst = {}


def matvec_on_device(W, x, block=8192):
    """stage_ref.matvec in float64 on the GPU: W[d, n] . x[n] (or x[n, m]), W promoted 8192 rows at a time."""
    xd = torch.as_tensor(np.ascontiguousarray(x, np.float64), device="cuda")
    out = torch.empty((W.shape[0],) + tuple(xd.shape[1:]), dtype=torch.float64, device="cuda")
    for r in range(0, W.shape[0], block):
        out[r:r + block] = torch.as_tensor(W[r:r + block], device="cuda").to(torch.float64) @ xd
    return out.cpu().numpy()


@pytest.fixture
def f64(monkeypatch):
    """stage_ref's products on the device; the stage errors go to this file's record."""
    monkeypatch.setattr(sr, "matvec", matvec_on_device)
    monkeypatch.setattr(ts, "worst_seen", worst)


def rows_checked(m):
    """The last block's rows under test: its first and last token tile, the tile edges, 34 rows spread evenly."""
    last = (m - 1) // 128 * 128
    r = set(range(min(128, m))) | set(range(last, m)) | {t for t in (0, 127, 128, 255, m - 1) if t < m}
    r |= set(np.linspace(0, m - 1, 34).round().astype(int).tolist())
    return np.array(sorted(r))


def check_pass(dm, w, toks, pos0, kvbits, label, layer=0):
    """forward_prefill_cuda(toks, pos0) on a one-layer model, then every cache entry it wrote and the last block's Q,
    attention output, hidden and residual rows against float64.  Returns the float64 normed inputs and the device's hidden
    rows, for the cases that check their own premise.  The stages are those of `layer`, whose input must be the embedding
    rows: layer 0, or the last layer behind layers that pass them through."""
    s = w.spec
    n, hd, kv_mul = len(toks), s.head_dim, s.n_heads // s.n_kv_heads
    m = n - BLOCK * ((n - 1) // BLOCK)
    b0 = pos0 + n - m  # the last block's first slot
    assert dm.prefill(toks, pos0) == 1, f"{label}: the tensor-core pass did not serve this shape"
    R = rows_checked(m)
    Q = dm.read_state("pf_q").reshape(-1, s.q_dim)[:m]
    A = dm.read_state("pf_att").reshape(-1, s.q_dim)[:m]
    H = dm.read_state("pf_hb").reshape(-1, s.hidden_dim)[:m]
    X = dm.read_state("pf_x").reshape(-1, s.dim)[:m]
    keys, values = layer_cache(dm, s, layer)
    blocks = " + ".join(str(min(BLOCK, n - o)) for o in range(0, n, BLOCK))
    label = f"{label} kv{kvbits} pos0 {pos0} n {n} ({blocks})"

    X0 = w.mat("model.embed.weight")[toks].astype(np.float64)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, layer, X0, pos0 + np.arange(n))
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        got = dev[:, pos0:pos0 + n].transpose(1, 0, 2).reshape(n, -1)
        check_entries(label, name, "k_pf_gemm QKV", got, ref, kvbits, lambda i: f"slot {pos0 + i[0]} kv head {i[1] // hd} dim {i[1] % hd}", "pf_kv", pf_tol(s.dim))

    row = lambda i: f"last-block row {R[i[0]]} (slot {b0 + R[i[0]]})"  # noqa: E731
    last = n - m + R  # the checked rows among all n
    q_ref, X0, xn = q_ref[last], X0[last], xn[last]
    report(label, "Q", "k_pf_gemm QKV", Q[R], q_ref, np.abs(q_ref).max(), lambda i: f"{row(i)} head {i[1] // hd} dim {i[1] % hd}", "pf_q", pf_tol(s.dim))
    k64, v64 = keys.astype(np.float64), values.astype(np.float64)
    a_ref = np.stack([sr.attention(s, Q[t], k64, v64, b0 + t + 1) for t in R])
    vmax = np.maximum.accumulate(np.abs(values[:, :b0 + m]).max(2), 1)[:, b0 + R].T  # [rows, kv heads]: max |V| of the head so far
    report(label, "A", "k_pf_attn", A[R], a_ref, np.repeat(vmax, kv_mul * hd, 1), lambda i: f"{row(i)} head {i[1] // hd} dim {i[1] % hd}, keys 0..{b0 + R[i[0]]}", "pf_att")
    x1 = sr.wo(w, layer, X0, A[R])
    xn2 = sr.ffn_input(w, layer, x1, xn)
    h_ref = sr.ffn_up(w, layer, xn2)
    report(label, "H", "k_pf_gemm WO+UP", H[R], h_ref, np.abs(h_ref).max(), lambda i: f"{row(i)} hidden row {i[1]}", "pf_hb", pf_tol(max(s.dim, s.q_dim)))
    x_ref = sr.ffn_down(w, layer, x1, H[R])
    report(label, "X", "k_pf_gemm DOWN", X[R], x_ref, np.abs(x_ref).max(), lambda i: f"{row(i)} row {i[1]}", "pf_x", pf_tol(s.hidden_dim))
    return np.concatenate([xn.reshape(-1), xn2.reshape(-1)]), H


# ---- 1. blocks and caches: (spec, kvbits, seq_len, pos0 (a fill_kv'd warm cache below it), n)
L8B16 = replace(L8B, dtype="fp16")
BLOCKS = {
    "llama3-8b fp8 one full block": (L8B, 16, 4096, 0, 2048),  # 16 token tiles, the TMA box at the buffer's last rows
    "llama3-8b fp8 2048 + 1": (L8B, 8, 4096, 0, 2049),  # a 1-row partial tile at slot 2048 over 2049 keys
    "llama3-8b fp8 three blocks": (L8B, 16, 8192, 0, 4500),  # the last a partial tile at slot 4096
    "mistral gf4 deep cache": (DECODE["mistral-gf4"][0], 8, 8192, 3000, 1200),  # 94 key tiles before the block
    "llama3-8b fp16 to the last slot": (L8B16, 16, 4096, 1000, 3096),  # 2048 + 1048 rows, the last at slot 4095
    # dim 8192, hidden 28672 (DOWN: 448 k-stages), 64 / 8 heads: k_pf_attn<.., 4> passes over the keys twice per kv head
    "llama3-70b fp8": (DECODE["llama3-70b"][0], 16, 4096, 0, 2100),
    # dim 896 = 7 tiles, hidden 4864 = 38, kv_dim 128 = one tile, QKV bias, 14 / 2 heads of 64: k_pf_attn<.., 1>, kv_mul 7
    "qwen2-0.5b fp16": (replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=1, vocab_size=V4K), 16, 4096, 0, 2100),
    "kv1-hd64 warm cache": (replace(GROUPINGS["kv1-hd64"], n_layers=1, vocab_size=V4K), 8, 4096, 500, 2600),  # one query head per kv head
}


@pytest.mark.parametrize("case", list(BLOCKS))
def test_prefill_blocks_every_stage(case, f64):
    spec, kvbits, seq_len, pos0, n = BLOCKS[case]
    t0 = time.perf_counter()
    tensors, w = make_model(spec, 4)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        dm.fill_kv(pos0, seed=6)
        check_pass(dm, w, mg.teacher_tokens(spec.vocab_size, n), pos0, kvbits, case)
    print(f"  {case}: {time.perf_counter() - t0:.1f} s")


# ---- 2. the scoring classifier over a full block at Llama-3's vocabulary
def test_score_full_block_at_the_real_vocabulary(f64):
    """2049 tokens: one block of 2048 scored rows, 1002 vocabulary tiles x 16 token tiles of k_pf_gemm PF_CLS, and
    k_pf_logprob.  Every row against a float64 final norm, classifier and log-softmax of the device's own residual rows,
    under test_score_gpu.py's bound."""
    t0 = time.perf_counter()
    spec = replace(mg.SPECS["llama3-8b-fp8"], n_layers=1)
    n = 2049
    tensors, w = make_model(spec, 7)
    toks = mg.teacher_tokens(spec.vocab_size, n)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        lp, served = dm.score(toks, 0)
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n - 1]
    assert served == 1, "the tensor-core pass did not serve this shape"
    xn = torch.as_tensor(sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, False), device="cuda")
    W = w.classifier()
    logits = torch.empty((n - 1, spec.vocab_size), dtype=torch.float64, device="cuda")
    for r in range(0, W.shape[0], 16384):
        logits[:, r:r + 16384] = xn @ torch.as_tensor(W[r:r + 16384], device="cuda").to(torch.float64).T
    ref, lse = log_softmax_at(logits, toks[1:])
    amax = logits.abs().amax(1).cpu().numpy()
    err = np.abs(lp.astype(np.float64) - ref)
    bound = stage_bound(spec.dim, amax, lse)
    i = int(np.argmax(err / bound))
    score_worst["lp"] = (float(err[i]), float(err[i] / bound[i]))
    print(f"\n  llama3-8b vocab 128256, 2048 scored rows: max |logprob - float64| {err.max():.2e}; worst {err[i]:.2e} = {err[i] / bound[i]:.2f} of its bound"
          f" at position {i} (max |logit| {amax[i]:.2f}, lse {lse[i]:.2f}); {time.perf_counter() - t0:.1f} s")
    assert np.isfinite(lp).all() and (err <= bound).all(), f"position {i}: device {lp[i]!r} vs float64 {ref[i]!r}"


# ---- 3. checkpoint-like activation scales, on Llama-3-8B widths in fp16 (whose weights scale exactly)
def scaled_model(kind, seed=8):
    """'wide': attention and FFN norm weights drawn per feature log-uniformly from [2^-5, 2^3], and 8 embedding columns
    x64, the massive residual features of real checkpoints, with FFN norm weight 2^3 and attention norm weight 2^-5, and
    wo x2^-6 so that the attention output does not swamp them: the other features' normed inputs become small and the
    hidden rows reach 10^3.  'small': norm weights 2^-7 (1 + N(0, 0.05)), so every normed input lies below
    2^-3, where the lo half of its f16 pair is subnormal."""
    tensors = mg.generate(L8B16, seed, device="cuda")
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    norms = ("model.layers.0.attn.norm.weight", "model.layers.0.mlp.norm.weight")
    d = L8B16.dim
    if kind == "wide":
        cols = torch.randperm(d, generator=g, device="cuda")[:8]
        for name, big in zip(norms, (2.0 ** -5, 2.0 ** 3)):
            wt = 2.0 ** (-5.0 + 8.0 * torch.rand(d, generator=g, device="cuda"))
            wt[cols] = big  # see k_pf_attn's limit in DESIGN.md s.6: the attention norm damps the massive features
            tensors[name] = wt
        tensors["model.embed.weight"][:, cols] *= 64  # fp16: exact
        tensors["model.layers.0.attn.wo.weight"] *= 2.0 ** -6  # the attention's share of the residual stays small beside them
    else:
        for name in norms:
            tensors[name] = 2.0 ** -7 * (1.0 + 0.05 * torch.randn(d, generator=g, device="cuda"))
    torch.cuda.synchronize()
    return tensors, sr.Weights(L8B16, {k: v.cpu() for k, v in tensors.items()})


@pytest.mark.parametrize("kind", ["wide", "small"])
def test_prefill_at_checkpoint_scales(kind, f64, capfd, monkeypatch):
    """Every stage of a 300-row prompt, then one decode step (the fp32 path) on the same model: a prompt-pass failure with
    a passing decode step belongs to the hi + lo pairs, not to the model."""
    monkeypatch.delenv("CALM_B200_QUIET", raising=False)
    t0 = time.perf_counter()
    tensors, w = scaled_model(kind)
    with lib.DeviceModel(L8B16, tensors, seq_len=4096, kvbits=16) as dm:
        plan = plan_of(capfd)
        with capfd.disabled():
            normed, H = check_pass(dm, w, mg.teacher_tokens(V4K, 300), 0, 16, f"llama3-8b fp16 {kind}")
            hmax, below = float(np.abs(H).max()), float((np.abs(normed) < 2.0 ** -4).mean())
            print(f"  {kind}: max |H| {hmax:.3g}, normed inputs below 2^-4 {below:.0%}, max |normed input| {np.abs(normed).max():.3g}")
            if kind == "wide":
                assert 1e3 <= hmax < 3e4 and below >= 0.1, "the model no longer has the scales this case is about"
            else:
                assert np.abs(normed).max() < 2.0 ** -3, "the model no longer has the scales this case is about"
            check_decode_step(dm, w, 17, 300, 16, plan, f"llama3-8b fp16 {kind} decode")
    print(f"  {kind}: {time.perf_counter() - t0:.1f} s")


def test_zz_summary_of_largest_errors():
    """Runs last in this file: each stage's largest error in this file's cases, beside its bound."""
    if not worst and not score_worst:
        pytest.skip("the stage tests did not run in this session")
    line = ", ".join(f"{k} {e:.2e} of {tol:.1e}" for k, (e, tol, _) in sorted(worst.items()))
    if score_worst:
        line += ", score lp {:.2e} ({:.2f} of its bound)".format(*score_worst["lp"])
    print("\n  prompt pass, largest error per stage: " + line)
    assert all(e <= tol for e, tol, _ in worst.values())
