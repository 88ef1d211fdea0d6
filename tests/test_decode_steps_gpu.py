"""calm_b200_decode_sample_n and calm_b200_decode_sample_batch against float64 at every step and every layer.

test_decode_sample_n_gpu.py and test_decode_sample_batch_gpu.py check the last step of a one-layer model against float64
fed the device's own cache.  Here a whole call is rebuilt in float64, teacher-forced by the device's own tokens: row b at
step j feeds its input token (the call's first token at j = 0, the device's token of step j - 1 after) at RoPE position
p_b + j through every layer, and each layer's attention reads the DEVICE's keys and values of that layer in the row's
virtual order: its prompt's slots, then its own slots of steps 0 .. j.  A cache entry on the other side of a rounding
boundary therefore costs nothing, as in test_stages_gpu.py.  The float64 residual stream of layers >= 1 does drift from
the device's by what the layers before added, so those layers' bounds are measured (KV_TOL, LOGIT_DRIFT).

Per case:
1. every cache entry the call wrote, of every row, step and layer, is a rounding of the float64 k / v;
2. temperature 0: every step's token is the float64 argmax wherever the top-2 margin is more than twice the logit bound;
3. sampled: every step's token is the float64 draw with the coin of xs_advance(seed_b, j) wherever that coin is clear of
   its bin edges by the logit bound (coin_clear).  A row with more than SAMPLE_EXACT survivors has no draw defined to
   the bit; there the token must be a survivor within test_device_sampler_at_real_vocabulary's rank distance of the
   float64 draw;
4. the last step: every row's logits lie within the classifier bound of float64 from the device's own final residual row,
   every row's last token is lib.sample_logits of its logit row, and the float64 chain's logits lie within the logit
   bound of the device's.
Both 2 and 3 assert a minimum share of clear (row, step) pairs, so that neither passes by checking nothing.  A last test
runs calls whose attention needs more and then fewer chunks on one engine, each bit for bit what a fresh engine gives.

The float64 matrix products run on the GPU (test_prefill_stages_gpu.matvec_on_device), the attention as a float64 torch
product beside them.  Every case prints its wall time; the last test prints each check's largest error beside its bound."""
import math
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
from test_decode_sample_batch_gpu import cache_rows, layout, prompts_of  # noqa: E402
from test_decode_sample_n_gpu import SEEDS  # noqa: E402
from test_prefill_stages_gpu import matvec_on_device  # noqa: E402
from test_score_greedy_gpu import top2  # noqa: E402
from test_stages_gpu import _RING, DECODE, L8B, check_entries, make_model, pf_tol, report  # noqa: E402
from test_verify_sample_gpu import DEFAULT, coin, coin_clear, xs_advance  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

SAMPLE_EXACT = 2048  # stages.cuh: more survivors than this and the device sampler adds per-chunk sums

# Bounds beyond layer 0, on an H100 80GB HBM3 (700 W limit); the largest value over this file's cases beside each.
# Layer 0 reads the exact embedding row, so its cache entries keep the prompt pass's bound pf_tol(dim) unchanged.  Layer
# l >= 1 reads a float64 residual that has drifted from the device's by the layers before: its entries are bounded (beyond
# half a spacing, of max |row|) by KV_TOL[l].
KV_TOL = {1: 8e-6, 2: 8e-6}  # measured 1.6e-6 (Llama-3-8B widths, layer 1) and 1.1e-6 (pf-tiny, layer 2)
# The float64 chain's logits differ from the device's by the classifier's own error, 2 pf_tol(dim) of max |row|, and by the
# drift of the final residual row after n layers, LOGIT_DRIFT[n] of max |row| (measured at each call's last step as
# |classifier(device x) - chain|).  Their sum is the logit bound of checks 2 and 3.
LOGIT_DRIFT = {1: 1.5e-5, 2: 1.5e-5, 3: 1e-5}  # measured 3.3e-6, 3.3e-6 and 1.4e-6
# Checks 2 and 3 must find at least this share of their (row, step) pairs clear of the bound.  (With T 1.0 and min-p 0.1
# the random models leave hundreds to thousands of survivors, whose bins are narrower than the bound moves them and some of
# which lie within the bound of the cutoff: at vocabulary 128256 one draw in 48 was clear.  The vocabulary-128256 and
# kv_mul-6 cases therefore sample at T 0.5, where a handful of tokens survive.  Measured: 56% at the least, Mistral's.)
MIN_CLEAR = 0.25

worst = {}  # this file's largest error per check, (error, bound, share)


@pytest.fixture
def f64(monkeypatch):
    """stage_ref's products on the device; check_entries' and report's errors go to this file's record."""
    monkeypatch.setattr(sr, "matvec", matvec_on_device)
    monkeypatch.setattr(ts, "worst_seen", worst)


def note(key, e, tol):
    if e / tol >= worst.get(key, (0.0, 1.0, -1.0))[2]:
        worst[key] = (e, tol, e / tol)


class Rows:
    """Where one call's rows live: row b's input at step 0 and RoPE position p[b] there, its prompt's cache slots, and
    its own slot base + j nseq + b at step j."""

    def __init__(self, first, p, prompt_slots, base):
        self.first, self.p, self.prompt, self.base = np.asarray(first), np.asarray(p), prompt_slots, base
        self.nseq = len(self.first)

    def own(self, j):
        return self.base + j * self.nseq + np.arange(self.nseq)

    def keys_of(self, b, j):
        """Row b's key slots at step j in virtual order."""
        return np.concatenate([self.prompt[b], self.base + np.arange(j + 1) * self.nseq + b])


def sample_n_rows(token0, pos0, nseq):
    return Rows(np.full(nseq, token0), np.full(nseq, pos0), [np.arange(pos0)] * nseq, pos0)


def batch_rows(prompts):
    starts, G = layout([len(p) for p in prompts])
    L = np.asarray([len(p) - 1 for p in prompts])
    return Rows([p[-1] for p in prompts], L, [s + np.arange(n) for s, n in zip(starts, L)], G)


def attend(spec, q, K, V):
    """stage_ref.attention of one row in float64 on the device: q[q_dim] over K / V[n_kv_heads, keys, head_dim]."""
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    sc = q.reshape(spec.n_kv_heads, kv_mul, hd) @ K.transpose(1, 2) / math.sqrt(hd)
    return (torch.softmax(sc, -1) @ V).reshape(-1)


def classify(w, X):
    """stage_ref.classifier of the rows X[n, dim]: [n, vocab]."""
    s = w.spec
    return sr.matvec(w.classifier(), sr.norm(X, w.vec("model.norm.weight"), s.norm_eps, s.norm_type != "rmsnorm").T).T


def rebuild(dm, w, rows, toks, kvbits, label):
    """Check 1 on every entry the call wrote, and the float64 chain's logits of every step, [n_tokens][nseq, vocab]."""
    s = w.spec
    hd, n = s.head_dim, toks.shape[1]
    shape = (s.n_kv_heads, dm.seq_len, hd)
    cache = [[dm.read_state(which, l).reshape(shape) for which in ("keys", "values")] for l in range(s.n_layers)]
    dev = [[torch.as_tensor(a, device="cuda").to(torch.float64) for a in kv] for kv in cache]
    idx = [[torch.as_tensor(rows.keys_of(b, j), device="cuda") for b in range(rows.nseq)] for j in range(n)]
    got = [([], []) for _ in range(s.n_layers)]
    want = [([], []) for _ in range(s.n_layers)]
    E = w.mat("model.embed.weight")
    logits = []
    for j in range(n):
        x = E[rows.first if j == 0 else toks[:, j - 1]].astype(np.float64)
        for l in range(s.n_layers):
            q, k, v, xn = sr.qkv(w, l, x, rows.p + j)
            for i, ref in enumerate((k, v)):
                got[l][i].append(cache[l][i][:, rows.own(j)].transpose(1, 0, 2).reshape(rows.nseq, -1))
                want[l][i].append(ref)
            qd = torch.as_tensor(q, device="cuda")
            K, V = dev[l]
            att = torch.stack([attend(s, qd[b], K[:, idx[j][b]], V[:, idx[j][b]]) for b in range(rows.nseq)]).cpu().numpy()
            x1 = sr.wo(w, l, x, att)
            x = sr.ffn_down(w, l, x1, sr.ffn_up(w, l, sr.ffn_input(w, l, x1, xn)))
        logits.append(classify(w, x))
    nseq = rows.nseq
    for l in range(s.n_layers):
        tol = pf_tol(s.dim) if l == 0 else KV_TOL[l]
        for i, name in enumerate("KV"):
            check_entries(label, f"{name} L{l}", "k_vf_gemm QKV", np.concatenate(got[l][i]), np.concatenate(want[l][i]), kvbits,
                          lambda e: f"step {e[0] // nseq} row {e[0] % nseq} kv head {e[1] // hd} dim {e[1] % hd}", f"kv L{l}", tol)
    return logits


def draw(L, c, temperature, minp):
    """The float64 sampler: (token, survivors) of logits L with coin c (the first index whose cumulative share passes c)."""
    mx = L.max()
    cut = mx + math.log(minp) * temperature if minp > 0 else -np.inf
    p = np.where(L >= cut, np.exp((L - mx) / temperature), 0.0)
    F = np.cumsum(p) / p.sum()
    return int(np.searchsorted(F, c, side="right")), np.nonzero(L >= cut)[0]


def check_steps(label, logits, toks, seeds, temperature, minp, drift, dim):
    """Checks 2 and 3 on every (row, step) of the call."""
    greedy = temperature == 0.0 or minp >= 1.0
    nseq, n = toks.shape
    clear = flat = rank = 0
    for j in range(n):
        L = logits[j]
        B = (2 * pf_tol(dim) + drift) * np.abs(L).max(1)
        if greedy:
            best, margin = top2(L)
            ok = margin > 2 * B
            bad = np.nonzero(ok & (toks[:, j] != best))[0]
            assert len(bad) == 0, f"{label}: step {j} row {bad[0]}: token {toks[bad[0], j]} vs the float64 argmax {best[bad[0]]} (margin {margin[bad[0]]:.3g}, bound {B[bad[0]]:.3g})"
            clear += int(ok.sum())
            continue
        for b in range(nseq):
            c = coin(xs_advance(seeds[b], j))
            want, keep = draw(L[b], c, temperature, minp)
            tok = int(toks[b, j])
            if len(keep) > SAMPLE_EXACT:
                flat += 1
                assert tok in keep, f"{label}: step {j} row {b}: token {tok} is not a survivor"
                dist = abs(int(np.searchsorted(keep, tok)) - int(np.searchsorted(keep, want)))
                rank = max(rank, dist)
                assert dist <= max(4, len(keep) // 4000), f"{label}: step {j} row {b}: token {tok} is {dist} survivors from the float64 draw {want} ({len(keep)} survivors)"
            elif coin_clear(L[b], c, temperature, minp, B[b]):
                clear += 1
                assert tok == want, f"{label}: step {j} row {b}: token {tok} vs the float64 draw {want} (coin {c:.6f} clear of its bin edges)"
    exact = nseq * n - flat
    share = clear / exact if exact else 1.0
    kind = "argmax" if greedy else "draws"
    print(f"  {label}: {kind} clear of the bound in {clear} of {exact} (row, step) pairs ({share:.0%})" + (f"; {flat} flat rows, worst rank distance {rank}" if flat else ""))
    assert share >= MIN_CLEAR, f"{label}: only {share:.0%} of the (row, step) pairs are clear of the logit bound"


def check_last(label, dm, w, logits, toks, seeds, temperature, minp, drift):
    """Check 4, and the drift of the chain's final residual row against the device's."""
    s = w.spec
    nseq = toks.shape[0]
    X = dm.read_state("pf_x").reshape(-1, s.dim)[:nseq]
    ref = classify(w, X)
    amax = np.abs(ref).max(1, keepdims=True)
    d = float((np.abs(ref - logits[-1]) / amax).max())
    note(f"logit drift L{s.n_layers}", d, drift)
    print(f"  {label}: chain logits drift {d:.2e} of max |row| from the device's final residual (tol {drift:.0e})")
    assert d <= drift, f"{label}: the float64 chain's last logits drift {d:.2e} of max |row| > {drift:.0e}"
    if temperature == 0.0 or minp >= 1.0:
        best, margin = top2(ref)
        ok = margin > 4 * pf_tol(s.dim) * amax[:, 0]
        assert (toks[ok, -1] == best[ok]).all(), f"{label}: a last token is not the float64 argmax of its row's logits"
        return
    Ld = dm.read_state("pf_logits").reshape(-1, s.vocab_size)[:nseq]
    report(label, "logits", "k_vf_gemm CLS", Ld, ref, amax, lambda i: f"row {i[0]} token {i[1]}", "logits", 2 * pf_tol(s.dim))
    for r in range(nseq):
        tok, _ = lib.sample_logits(Ld[r], temperature, minp, xs_advance(seeds[r], toks.shape[1] - 1))
        assert tok == toks[r, -1], f"{label}: row {r}: last token {toks[r, -1]} vs lib.sample_logits of its logit row {tok}"


# ---- cases: (spec, kvbits, seq_len, ("n", nseq, n_tokens, pos0) or ("batch", prompt lengths, n_tokens), [(T, min-p)])
L8B2 = replace(L8B, n_layers=2)
QWEN = replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=2)
KV6 = replace(_RING, n_heads=12, n_kv_heads=2, n_layers=2)  # kv_mul 6 at head_dim 128: KM = 2, three groups per row
GREEDY = (0.0, 0.1)
SHARP = (0.5, 0.1)
CASES = {
    # 46 prompt chunks shared by all rows, one suffix chunk per row; k_sn_fold over 47 chunks; layer 1's cache
    "llama3-8b fp8 2l n16 t4 pos0 6000": (L8B2, 16, 8192, ("n", 16, 4, 6000), [DEFAULT]),
    "llama3-8b fp8 2l e5m2 n16 t4 pos0 6000": (L8B2, 8, 8192, ("n", 16, 4, 6000), [GREEDY]),
    # the row sampler over 126 chunks: the exact walk at min-p 0.1, the chunk-sum walk at min-p 0 (every token survives)
    "llama3-8b fp8 vocab 128256 n16 t3": (replace(L8B, vocab_size=128256), 16, 1024, ("n", 16, 3, 300), [SHARP, (1.0, 0.0)]),
    # kv_mul 7 (KM = 1), head_dim 64, QKV bias, tied classifier, 149 sampler chunks
    "qwen2-0.5b 2l vocab 151936 n16 t3": (QWEN, 16, 1024, ("n", 16, 3, 200), [DEFAULT]),
    "qwen2-0.5b 2l vocab 151936 batch9 t3": (QWEN, 16, 4096, ("batch", [300, 1, 129, 57, 1000, 2, 260, 40, 700], 3), [GREEDY]),
    "kv_mul6 hd128 2l n16 t4": (KV6, 16, 1024, ("n", 16, 4, 300), [SHARP]),
    "kv_mul6 hd128 2l e5m2 batch6 t4": (KV6, 8, 4096, ("batch", [200, 1, 129, 300, 64, 1000], 4), [GREEDY]),
    # a BATCH row of 40 chunks beside an empty prompt; prompts across the 2048-row block edges
    "mistral gf4 2l e5m2 batch6 t3": (replace(DECODE["mistral-gf4"][0], n_layers=2), 8, 8192, ("batch", [5000, 1, 300, 129, 2049, 40], 3), [DEFAULT]),
    # 200 keys per row: two suffix chunks, no shared chunk; 140 steps over 480 of the 512 slots
    "pf-tiny 3l n3 t140 pos0 60": (replace(mg.SPECS["pf-tiny"], n_layers=3), 16, 512, ("n", 3, 140, 60), [GREEDY, DEFAULT]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_every_step_and_layer(case, f64, capfd):
    spec, kvbits, seq_len, call, settings = CASES[case]
    t0 = time.perf_counter()
    tensors, w = make_model(spec, 4)
    drift = LOGIT_DRIFT[spec.n_layers]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm, capfd.disabled():
        if call[0] == "n":
            _, nseq, n, pos0 = call
            dm.fill_kv(pos0, seed=6)
            rows = sample_n_rows(3, pos0, nseq)
        else:
            _, lens, n = call
            prompts = prompts_of(spec.vocab_size, lens, start=3)
            nseq, rows = len(lens), batch_rows(prompts)
        seeds = SEEDS[:nseq]
        for temperature, minp in settings:
            if call[0] == "n":
                toks, states, served = dm.decode_sample_n(3, pos0, n, temperature, minp, seeds)
            else:
                toks, states, served = dm.decode_sample_batch(prompts, n, temperature, minp, seeds)
            assert served == 1, f"{case}: the call was not served by the step loop"
            label = f"{case} kv{kvbits} T {temperature} min-p {minp}"
            logits = rebuild(dm, w, rows, toks, kvbits, label)
            check_last(label, dm, w, logits, toks, seeds, temperature, minp, drift)
            check_steps(label, logits, toks, seeds, temperature, minp, drift, spec.dim)
    print(f"  {case}: {time.perf_counter() - t0:.1f} s")


# ---- 5. the chunk partials grow and are reused: one engine against a fresh engine per call
def growth_call(dm, spec, call):
    kind, arg = call
    if kind == "n":
        dm.fill_kv(arg, seed=6)
        toks, states, served = dm.decode_sample_n(3, arg, 5, *DEFAULT, SEEDS)
        own = arg + np.arange(5 * 16)
    else:
        prompts = prompts_of(spec.vocab_size, arg, start=9)
        toks, states, served = dm.decode_sample_batch(prompts, 5, *DEFAULT, SEEDS[:len(arg)])
        own = layout(arg)[1] + np.arange(5 * len(arg))
    assert served == 1
    nseq = toks.shape[0]
    return [toks, np.asarray(states, np.uint64), dm.read_state("pf_x").reshape(-1, spec.dim)[:nseq],
            dm.read_state("pf_att").reshape(-1, spec.q_dim)[:nseq]] + cache_rows(dm, spec, own)


def test_growing_and_shrinking_calls_on_one_engine():
    """decode_sample_n at pos0 100 (1 chunk per row), at pos0 6000 (47: the partials regrow), decode_sample_batch with a
    5000-row prompt (40 chunks, the pass's rows regrow), then pos0 100 again on the larger buffers."""
    spec = L8B2
    tensors = mg.generate(spec, 9, device="cuda")
    calls = [("n", 100), ("n", 6000), ("batch", [5001, 40, 1]), ("n", 100)]
    with lib.DeviceModel(spec, tensors, seq_len=8192) as dm:
        dirty = [growth_call(dm, spec, c) for c in calls]
    for c, d in zip(calls, dirty):
        with lib.DeviceModel(spec, tensors, seq_len=8192) as dm:
            fresh = growth_call(dm, spec, c)
        for i, (f, x) in enumerate(zip(fresh, d)):
            if f.dtype.kind == "f":
                assert np.isfinite(f).all(), f"{c}: item {i} not finite"
            assert np.array_equal(x, f), f"{c}: item {i} differs between the engine that ran the other calls and a fresh one"


def test_zz_summary_of_largest_errors():
    """Runs last in this file: each check's largest error in this file's cases, beside its bound."""
    if not worst:
        pytest.skip("the step tests did not run in this session")
    print("\n  decode steps, largest error per check: " + ", ".join(f"{k} {e:.2e} of {tol:.1e}" for k, (e, tol, _) in sorted(worst.items())))
    assert all(e <= tol for e, tol, _ in worst.values())
