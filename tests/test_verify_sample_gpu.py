"""calm_b200_verify_sample (a short block whose rows are drawn by the reference sampler) and calm_b200_decode_lookup_sample
(prompt-lookup decoding at temperature > 0, each draft accepted exactly when the target's own sample equals it).

1. The logit rows (CALM_B200_STATE_PF_LOGITS) against float64 from the device's own final residual rows, within the
   classifier bound of test_score_gpu.
2. They are the values of the greedy path: each row's argmax is verify_greedy's token, exact ties included.
3. Each row's token is lib.sample_logits of that row with the generator state of its draw, bit for bit, and the returned
   state is the state after the emitted draws (a Python xorshift*, integer and exact).
4. Temperature 0 and minp >= 1 are the greedy calls and leave the generator alone.
5. A lookup run that never finds a draft is calm_b200_decode_sample, bit for bit.
6. The lookup loop on a seed whose every coin sits clear of its bin edges reproduces decode_sample's stream and state.
7. Fallback shapes give exactly n forward_sample calls.  8. No result depends on history.  9. Bad arguments raise."""
import math
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_score_greedy_gpu import K_COL, TIES, tie_model, top2  # noqa: E402
from test_stages_gpu import V4K, make_model, pf_tol  # noqa: E402
from test_verify_gpu import TINY1, simulate  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
DEFAULT = (1.0, 0.1)  # calm's run.c defaults: -t 1.0, -p 0.1


def xs_step(s):
    """The reference's xorshift* state step (sampler.c:7-13)."""
    s ^= s >> 12
    s ^= (s << 25) & M64
    s ^= s >> 27
    return s


def xs_advance(s, k):
    for _ in range(k):
        s = xs_step(s)
    return s


def coin(s):
    """The coin of the next draw from state s (sampler.c:15-17), exact as a float64."""
    s = xs_step(s)
    return ((((s * 0x2545F4914F6CDD1D) & M64) >> 32) >> 8) / 16777216.0


def accepted(tokens, sampled):
    a = 0
    while a < len(tokens) - 1 and sampled[a] == tokens[a + 1]:
        a += 1
    return a


def logit_rows(dm, n):
    return dm.read_state("pf_logits").reshape(n, dm.vocab)


def float64_logits(spec, w, X):
    xn = torch.as_tensor(sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, spec.norm_type != "rmsnorm"), device="cuda")
    W = w.classifier()
    logits = torch.empty((len(X), spec.vocab_size), dtype=torch.float64, device="cuda")
    for r in range(0, W.shape[0], 16384):
        logits[:, r:r + 16384] = xn @ torch.as_tensor(W[r:r + 16384], device="cuda").to(torch.float64).T
    return logits.cpu().numpy()


# ---- 1 + 2. the logit rows against float64, and the greedy path's argmax on the same engine state
LOGITS = {
    "llama3-8b fp8 vocab 128256 n16": (replace(mg.SPECS["llama3-8b-fp8"], n_layers=1), 16, 16),
    "mistral gf4 vocab 32000 kv8 n9": (replace(mg.SPECS["mistral-7b-gf4"], n_layers=1), 8, 9),
    "pf-tiny fp16 vocab 512 n1": (replace(TINY1, dtype="fp16"), 16, 1),
    "pf-tiny fp8 vocab 4100 n16": (replace(TINY1, vocab_size=4100), 16, 16),  # a last tile of 4 rows
    "pf-tiny gf4 vocab 4100 n9": (replace(TINY1, dtype="gf4", vocab_size=4100), 16, 9),
}


@pytest.mark.parametrize("case", sorted(LOGITS))
def test_logit_rows_against_float64(case):
    spec, kvbits, n = LOGITS[case]
    tensors, w = make_model(spec, 7)
    toks = mg.teacher_tokens(spec.vocab_size, n, start=5)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        dm.fill_kv(40, seed=2)
        greedy, served_g = dm.verify_greedy(toks, 40)
        Xg = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
        sampled, state, served = dm.verify_sample(toks, 40, *DEFAULT, 99)
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
        L = logit_rows(dm, n)
    assert served == 1 and served_g == 1
    assert np.array_equal(X, Xg), f"{case}: the two calls' residual rows differ"
    assert np.array_equal(L.argmax(1), greedy), f"{case}: a logit row's argmax is not verify_greedy's token"
    assert ((sampled >= 0) & (sampled < spec.vocab_size)).all()
    ref = float64_logits(spec, w, X)
    err = np.abs(L.astype(np.float64) - ref)
    bound = np.broadcast_to(2 * pf_tol(spec.dim) * np.abs(ref).max(1, keepdims=True), ref.shape)
    i = np.unravel_index(int(np.argmax(err / bound)), err.shape)
    print(f"\n  {case}: max |logit - float64| {err.max():.2e} = {float(err[i] / bound[i]):.2f} of its bound at row {i[0]} token {i[1]}")
    assert np.isfinite(L).all() and (err <= bound).all(), f"{case}: row {i[0]} token {i[1]}: {L[i]!r} vs float64 {ref[i]!r}"
    best, margin = top2(ref)
    clear = margin > 2 * bound[:, 0]
    assert (greedy[clear] == best[clear]).all(), f"{case}: a greedy token is not the float64 argmax where the top-2 margin is clear"


@pytest.mark.parametrize("dtype", ["fp8", "fp16", "gf4"])
@pytest.mark.parametrize("vocab", sorted(TIES))
def test_exact_ties_are_the_greedy_tokens(vocab, dtype):
    """The exact-tie models of test_score_greedy_gpu: the first maximum of every logit row is verify_greedy's token."""
    spec = replace(mg.SPECS["pf-tiny"], dtype=dtype, vocab_size=vocab, n_layers=1)
    toks = mg.teacher_tokens(vocab, 112)
    for name, fam_p, fam_n in TIES[vocab]:
        tensors = tie_model(spec, fam_p, fam_n, 31)
        w = sr.Weights(spec, tensors)
        signs = []
        with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
            for p in range(0, len(toks), 16):
                g, served_g = dm.verify_greedy(toks[p:p + 16], p)
                _, _, served = dm.verify_sample(toks[p:p + 16], p, *DEFAULT, 5)
                assert served == 1 and served_g == 1
                L = logit_rows(dm, 16)
                assert np.array_equal(L.argmax(1), g), f"vocab {vocab} {dtype} {name}: block at {p}: argmax {L.argmax(1)} vs greedy {g}"
                X = dm.read_state("pf_x").reshape(-1, spec.dim)[:16]
                signs.append(sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, False)[:, K_COL])
        xk = np.concatenate(signs)
        assert (xk > 0).any() and (xk < 0).any(), f"vocab {vocab} {dtype} {name}: x_k took one sign only"


# ---- 3. every row's draw, bit for bit
@pytest.mark.parametrize("temperature,minp", [(1.0, 0.1), (0.7, 0.05), (1.3, 0.0)])
def test_each_row_is_the_reference_draw(temperature, minp):
    """vocab 4100: at minp 0 every token survives, more than SAMPLE_EXACT, so the chunk-sum walk runs.  The drafts are set
    so that a = n - 1, a mid-block value and 0 all occur."""
    spec = replace(TINY1, vocab_size=4100)
    tensors = mg.generate(spec, 12)
    n, pos0, seed = 16, 30, 0x1234_5678_9ABC_DEF1
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, pos0 + 1, start=3), np.int32)
    seen = set()
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1

        def run(block):
            sampled, state, served = dm.verify_sample(block, pos0, temperature, minp, seed)
            assert served == 1
            L = logit_rows(dm, n)
            for i in range(n):
                tok, after = lib.sample_logits(L[i], temperature, minp, xs_advance(seed, i))
                assert tok == sampled[i], f"row {i}: {sampled[i]} vs the reference draw {tok}"
                assert after == xs_advance(seed, i + 1)
            a = accepted(block, sampled)
            assert state == xs_advance(seed, a + 1), f"state after {a} accepted drafts"
            return sampled, a

        block = np.concatenate([[prompt[-1]], np.zeros(n - 1, np.int32)]).astype(np.int32)
        for target in (n - 1, n // 2, 0):
            for _ in range(n):
                sampled, a = run(block)
                if a == target:
                    break
                if a < target:
                    block[a + 1] = sampled[a]  # accept one more
                else:
                    block[target + 1] = (sampled[target] + 1) % spec.vocab_size  # reject at the target
            assert a == target, f"drafts for {target} accepted ones gave {a}"
            seen.add(a)
    assert seen == {0, n // 2, n - 1}


# ---- 4. greedy settings
@pytest.mark.parametrize("temperature,minp", [(0.0, 0.1), (1.0, 1.0)])
def test_greedy_settings_are_the_greedy_calls(temperature, minp):
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 46)
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    block = np.asarray(mg.teacher_tokens(spec.vocab_size, 9, start=4), np.int32)
    seed = 77
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        g, served_g = dm.verify_greedy(block, 59)
        s, state, served = dm.verify_sample(block, 59, temperature, minp, seed)
    assert np.array_equal(s, g) and served == served_g == 1 and state == seed
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        out_g, steps_g = dm.decode_lookup(prompt, 30, source=None, max_draft=7)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        out, steps, state = dm.decode_lookup_sample(prompt, 30, temperature, minp, seed, source=None, max_draft=7)
    assert np.array_equal(out, out_g) and steps == steps_g and state == seed


# ---- 5. no match is decode_sample
@pytest.mark.parametrize("seed", [1, 0xDEADBEEF, (1 << 63) + 7])
def test_lookup_without_a_match_is_decode_sample(seed):
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 5)
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 40, start=2), np.int32)
    n = 40
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        G, state = dm.decode_sample(int(prompt[-1]), len(prompt) - 1, n, *DEFAULT, seed)
    absent = np.setdiff1d(np.arange(spec.vocab_size), np.concatenate([prompt, G]))[:3].astype(np.int32)
    for src in (absent, absent[:0]):
        with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
            assert dm.prefill(prompt[:-1], 0) == 1
            out, steps, st = dm.decode_lookup_sample(prompt, n, *DEFAULT, seed, source=src, max_draft=7)
        assert np.array_equal(out, G) and st == state and steps == n


# ---- 6. the lookup loop on a qualified seed
PEAKED_ROWS, PEAKED_GAIN = np.arange(8) * 37 + 3, 40.0


def peaked_model():
    """pf-tiny with eight classifier rows scaled by 40: a few tokens stand far above a flat bulk, as in a trained model, so at
    minp 0.1 one to four tokens survive and the cutoff falls in the gap between them and the bulk."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 46)
    W = torch.as_tensor(sr.Weights(spec, tensors).classifier())
    W[PEAKED_ROWS] *= PEAKED_GAIN
    tensors["model.output.weight"] = mg.quantize(W.float(), spec.dtype)
    return spec, tensors


def coin_clear(logits, c, temperature, minp, d=None):
    """No change of any logit by up to d (default 2 TOL_SIGMA sigma of the row) moves the coin c across a bin edge
    (float64): no logit lies within 2 d of the min-p cutoff, and the coin stays inside its bin when every survivor's weight
    exp(l / T) moves by exp(+-d / T), which bounds the odds of every cumulative share by exp(+-2 d / T)."""
    L = np.asarray(logits, np.float64)
    if d is None:
        d = 2 * TOL_SIGMA * L.std()
    mx = L.max()
    cut = mx + math.log(minp) * temperature if minp > 0 else -np.inf
    if np.isfinite(cut) and np.abs(L - cut).min() <= 2 * d:
        return False
    p = np.where(L >= cut, np.exp((L - mx) / temperature), 0.0)
    F = np.cumsum(p) / p.sum()
    j = int(np.searchsorted(F, c, side="right"))
    r = math.exp(2 * d / temperature)
    lo = F[j - 1] * r / (F[j - 1] * r + 1 - F[j - 1]) if j > 0 else 0.0
    hi = F[j] / r / (F[j] / r + 1 - F[j]) if F[j] < 1 else 1.0
    return lo < c < hi


@pytest.fixture(scope="module")
def sampled_stream():
    """The first seed in 1 .. 32 whose decode_sample stream of 32 tokens after a 60-token prompt has every coin clear of
    its bin edges (coin_clear on the decode logits of each step).  Returns spec, tensors, prompt, seed, stream, final state."""
    spec, tensors = peaked_model()
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    P, N = len(prompt), 32
    for seed in range(1, 33):
        with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
            assert dm.prefill(prompt[:-1], 0) == 1
            tok, s, stream, ok = int(prompt[-1]), seed, [], True
            for e in range(N):
                c = coin(s)
                tok, s = dm.forward_sample(tok, P - 1 + e, *DEFAULT, s)
                stream.append(tok)
                if not coin_clear(dm.device_logits(), c, *DEFAULT):
                    ok = False
                    break
        if ok:
            break
    else:
        pytest.fail("no seed in 1 .. 32 has every coin of its stream clear of the bin edges")
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        G, state = dm.decode_sample(int(prompt[-1]), P - 1, N, *DEFAULT, seed)
    assert np.array_equal(G, stream) and state == s, "forward_sample steps differ from decode_sample"
    print(f"\n  seed {seed}: stream {G.tolist()}")
    return spec, tensors, prompt, seed, G, state


def run_lookup_sample(spec, tensors, prompt, n, source, max_draft, seed):
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        return dm.decode_lookup_sample(prompt, n, *DEFAULT, seed, source=source, max_draft=max_draft)


@pytest.mark.parametrize("max_draft", [3, 7, 15])
def test_lookup_sample_with_the_stream_as_source(sampled_stream, max_draft):
    spec, tensors, prompt, seed, G, state = sampled_stream
    n = len(G)
    source = np.concatenate([prompt, G]).astype(np.int32)
    out, steps, st = run_lookup_sample(spec, tensors, prompt, n, source, max_draft, seed)
    want, kinds = simulate(prompt, G, n, source, max_draft, 512)
    print(f"  max_draft {max_draft}: {n} tokens in {steps} steps, kinds {kinds}")
    assert np.array_equal(out, G) and st == state and steps == want and steps < n


def test_lookup_sample_with_a_corrupted_source(sampled_stream):
    """test_lookup_with_a_corrupted_source's construction: full acceptance, a rejection mid-way and a step without a match."""
    spec, tensors, prompt, seed, G, state = sampled_stream
    n = len(G)
    fresh = int(np.setdiff1d(np.arange(spec.vocab_size), np.concatenate([prompt, G]))[0])
    for j in range(2, n - 2):
        source = np.where(np.concatenate([prompt, G]) == G[j], fresh, np.concatenate([prompt, G])).astype(np.int32)
        want, kinds = simulate(prompt, G, n, source, 7, 512)
        if {"all", "mid", "none"} <= set(kinds):
            break
    else:
        pytest.fail("no corruption gives every kind of step")
    out, steps, st = run_lookup_sample(spec, tensors, prompt, n, source, 7, seed)
    print(f"  stream token {j} corrupted: {steps} steps, kinds {kinds}")
    assert np.array_equal(out, G) and st == state and steps == want


# ---- 7. fallback
@pytest.mark.parametrize("name,seq_len,n,pos0", [("tiny-moe", None, 9, 5), ("pf-tiny", 64, 8, 60)])
def test_fallback_is_forward_sample(name, seq_len, n, pos0):
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    toks = np.asarray(mg.teacher_tokens(spec.vocab_size, pos0 + n), np.int32)
    seed = 4242
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        dm.prefill(toks[:pos0], 0)
        sampled, state, served = dm.verify_sample(toks[pos0:], pos0, *DEFAULT, seed)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        dm.prefill(toks[:pos0], 0)
        want, s = [], seed
        for i, t in enumerate(toks[pos0:]):
            tok, s = dm.forward_sample(int(t), pos0 + i, *DEFAULT, s)
            want.append(tok)
    assert served == 0 and np.array_equal(sampled, want)
    assert state == xs_advance(seed, accepted(toks[pos0:], sampled) + 1)


# ---- 8. history
HIST = {"pf-tiny-v1000": replace(mg.SPECS["pf-tiny"], vocab_size=1000), "llama-2l": replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K)}
BLOCKS = [(16, 60), (1, 76), (7, 77), (9, 84)]


def sample_run(dm, toks, seed):
    assert dm.prefill(toks[:60], 0) == 1
    out = []
    for n, p in BLOCKS:
        sampled, state, served = dm.verify_sample(toks[p:p + n], p, *DEFAULT, seed + p)
        assert served == 1
        out += [sampled, np.asarray([state], np.uint64), logit_rows(dm, n), dm.read_state("pf_x").reshape(-1, dm.spec.dim)[:n]]
    return out


@pytest.mark.parametrize("name", sorted(HIST))
def test_verify_sample_does_not_depend_on_history(name):
    spec = HIST[name]
    tensors = mg.generate(spec, 31, device="cuda")
    torch.cuda.synchronize()
    toks = np.asarray(mg.teacher_tokens(spec.vocab_size, 100, start=4), np.int32)
    other = np.asarray(mg.teacher_tokens(spec.vocab_size, 300, start=9), np.int32)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        fresh = sample_run(dm, toks, 3)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        dm.prefill(other[:250], 0)
        dm.decode_lookup_sample(other[:251], 30, 0.8, 0.02, 11, max_draft=15)
        dm.verify_sample(other[:16], 200, 1.3, 0.0, 12)
        dm.poison(0)
        dirty = sample_run(dm, toks, 3)
    for i, (f, d) in enumerate(zip(fresh, dirty)):
        if f.dtype.kind == "f":
            assert np.isfinite(f).all(), f"{name}: item {i} not finite"
        assert np.array_equal(d, f), f"{name}: item {i}: after another history and poisoning the results changed"


# ---- 9. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        for toks in ([], list(range(17)), None):
            with pytest.raises(ValueError):
                dm.verify_sample(toks if toks is None else np.asarray(toks, np.int32), 0, *DEFAULT, 1)
        with pytest.raises(ValueError):
            dm.verify_sample([1, 2], 0, *DEFAULT, None)
        for md in (0, 16, -1):
            with pytest.raises(ValueError):
                dm.decode_lookup_sample([1, 2, 3], 4, *DEFAULT, 1, max_draft=md)
        for toks in ([], None):
            with pytest.raises(ValueError):
                dm.decode_lookup_sample(toks, 4, *DEFAULT, 1)
        with pytest.raises(ValueError):
            dm.decode_lookup_sample([1, 2, 3], 4, *DEFAULT, None)
        out, steps, state = dm.decode_lookup_sample([1, 2, 3], 0, *DEFAULT, 9)  # nothing wanted: no step, no draw
        assert len(out) == 0 and steps == 0 and state == 9
