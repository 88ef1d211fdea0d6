"""calm_b200_verify_greedy (a block of up to 16 tokens on a live cache, with the short-block GEMM k_vf_gemm) and
calm_b200_decode_lookup (greedy decoding with prompt-lookup drafts).

1. Stage by stage: the block's Q rows, cache entries, attention output, hidden rows and residual rows, each against float64
   fed the device's own previous stage, as test_prefill_every_stage checks the prompt pass.
2. Greedy tokens: the argmax of float64 logits from the device's own final residual rows wherever the top-2 margin
   exceeds the classifier's bound, and exact ties across lanes, tiles and a partial last tile.
3. Against the decode: the draft-verification loop on verify_greedy reproduces calm_b200_decode_greedy's stream.
4. The lookup loop: full acceptance, corrupted sources, a source that never matches, prompt lookup on the sequence itself,
   and the end of the cache.  A Python model of the loop predicts every step count.
5. Fallback: shapes the short-block path does not serve give exactly n forward_argmax results.
6. Repeated calls, fresh engines and poisoned engines with another history give the same bits."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_score_greedy_gpu import K_COL, TIES, VERIFY_STEPS, greedy_stream, tie_check, tie_model, top2  # noqa: E402
from test_stages_gpu import DECODE, L8B, V4K, check_entries, layer_cache, make_model, note, pf_tol, report, worst_seen  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

# ---- 1. every stage of the block: (spec, kvbits, n, pos0)
TINY1 = replace(mg.SPECS["pf-tiny"], n_layers=1)
VERIFY = {
    "llama3-8b fp8 n16 pos 300": (L8B, 16, 16, 300),  # dim 4096, hidden 14336: the 28-slice fold of w2
    "llama3-8b fp8 kv8 n9 pos 1000": (L8B, 8, 9, 1000),
    "llama3-8b fp16 n2 pos 50": (replace(mg.SPECS["llama3-8b-fp16"], n_layers=1, vocab_size=V4K), 16, 2, 50),
    "llama3-70b n8 pos 200": (replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K), 16, 8, 200),
    "mistral-gf4 kv8 n7 pos 100": (DECODE["mistral-gf4"][0], 8, 7, 100),
    "pf-tiny fp8 n1 pos 37": (TINY1, 16, 1, 37),  # K = 256: one partial slice
    "pf-tiny gf4 kv8 n16 pos 5": (replace(TINY1, dtype="gf4"), 8, 16, 5),
    "pf-tiny fp16 n8 pos 120": (replace(TINY1, dtype="fp16"), 16, 8, 120),
    "pf-tiny-hd128 bias n9 pos 37": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 16, 9, 37),
    "switch-gelu-clip-rot64 n7 pos 64": (DECODE["switch-gelu-clip-rot64"][0], 16, 7, 64),
    "switch-layernorm-par kv8 n16 pos 64": (DECODE["switch-layernorm-par"][0], 8, 16, 64),
}


@pytest.mark.parametrize("case", sorted(VERIFY))
def test_verify_every_stage(case, capfd):
    spec, kvbits, n, pos0 = VERIFY[case]
    tensors, w = make_model(spec, 4)
    with lib.DeviceModel(spec, tensors, seq_len=2048, kvbits=kvbits) as dm, capfd.disabled():
        dm.fill_kv(pos0, seed=6)
        check_block(dm, w, kvbits, n, pos0, case)


def check_block(dm, w, kvbits, n, pos0, case):
    """verify_greedy of n tokens at pos0 over the cache below it, then every stage of the block against float64."""
    spec = w.spec
    toks = mg.teacher_tokens(spec.vocab_size, n, start=3)
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    greedy, served = dm.verify_greedy(toks, pos0)
    X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
    Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:n]
    A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:n]
    H = dm.read_state("pf_hb").reshape(-1, spec.hidden_dim)[:n]
    keys, values = layer_cache(dm, spec)
    assert served == 1, f"{case}: the short-block path did not serve this shape"
    label = f"verify {case} kv{kvbits}"
    X0 = w.mat("model.embed.weight")[toks].astype(np.float64)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, 0, X0, pos0 + np.arange(n))
    report(label, "Q", "k_vf_gemm QKV", Q, q_ref, np.abs(q_ref).max(), lambda i: f"token row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "vf_q", pf_tol(spec.dim))
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        got = dev[:, pos0:pos0 + n].transpose(1, 0, 2).reshape(n, -1)
        check_entries(label, name, "k_vf_gemm QKV", got, ref, kvbits, lambda i: f"token row {i[0]} kv head {i[1] // hd} dim {i[1] % hd}", "vf_kv", pf_tol(spec.dim))
    a_ref = np.stack([sr.attention(spec, Q[t], keys, values, pos0 + t + 1) for t in range(n)])
    vmax = np.repeat(np.maximum.accumulate(np.abs(values[:, :pos0 + n]).max(2), 1)[:, pos0:].T, kv_mul * hd, 1)
    report(label, "A", "k_pf_attn", A, a_ref, vmax, lambda i: f"token row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")
    x1 = sr.wo(w, 0, X0, A)
    h_ref = sr.ffn_up(w, 0, sr.ffn_input(w, 0, x1, xn))
    report(label, "H", "k_vf_gemm WO+UP", H, h_ref, np.abs(h_ref).max(), lambda i: f"token row {i[0]} hidden row {i[1]}", "vf_hb", pf_tol(max(spec.dim, spec.q_dim)))
    x_ref = sr.ffn_down(w, 0, x1, H)
    report(label, "X", "k_vf_gemm DOWN", X, x_ref, np.abs(x_ref).max(), lambda i: f"token row {i[0]} row {i[1]}", "vf_x", pf_tol(spec.hidden_dim))
    check_greedy(label, spec, w, X, greedy)


# ---- 2. the greedy tokens, from the device's own final residual rows
def check_greedy(label, spec, w, X, greedy):
    xn = torch.as_tensor(sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, spec.norm_type != "rmsnorm"), device="cuda")
    W = w.classifier()
    logits = torch.empty((len(X), spec.vocab_size), dtype=torch.float64, device="cuda")
    for r in range(0, W.shape[0], 16384):
        logits[:, r:r + 16384] = xn @ torch.as_tensor(W[r:r + 16384], device="cuda").to(torch.float64).T
    ref = logits.cpu().numpy()
    assert ((greedy >= 0) & (greedy < spec.vocab_size)).all(), f"{label}: a greedy token outside the vocabulary"
    bound = 2 * pf_tol(spec.dim) * np.abs(ref).max(1)
    best, margin = top2(ref)
    short = ref.max(1) - ref[np.arange(len(X)), greedy]
    i = int(np.argmax(short / bound))
    note("vf_greedy", float(short[i] / bound[i]), 1.0)
    print(f"  {label}: greedy logit below the float64 maximum by at most {short.max():.2e} = {short[i] / bound[i]:.2f} of its bound")
    assert (short <= bound).all(), f"{label}: row {i}: greedy {greedy[i]} is {short[i]:.3e} below the maximum (bound {bound[i]:.3e})"
    bad = np.nonzero((margin > bound) & (greedy != best))[0]
    assert len(bad) == 0, f"{label}: row {bad[0]}: greedy {greedy[bad[0]]} vs float64 argmax {best[bad[0]]} (margin {margin[bad[0]]:.3e})"


GREEDY = {
    "llama3-8b fp8 vocab 128256": (replace(mg.SPECS["llama3-8b-fp8"], n_layers=1), 16, 16),  # 1002 tiles: four classifier launches
    "mistral gf4 vocab 32000 kv8": (replace(mg.SPECS["mistral-7b-gf4"], n_layers=1), 8, 9),
    "pf-tiny vocab 1000": (replace(TINY1, vocab_size=1000), 16, 16),  # a partial vocabulary tile
    "switch-layernorm-par": (DECODE["switch-layernorm-par"][0], 16, 7),  # a LayerNorm final norm
}


@pytest.mark.parametrize("case", sorted(GREEDY))
def test_verify_greedy_against_float64(case):
    spec, kvbits, n = GREEDY[case]
    tensors, w = make_model(spec, 7)
    toks = mg.teacher_tokens(spec.vocab_size, n, start=5)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        dm.fill_kv(40, seed=2)
        greedy, served = dm.verify_greedy(toks, 40)
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
    assert served == 1
    check_greedy(case, spec, w, X, greedy)


@pytest.mark.parametrize("dtype", ["fp8", "fp16", "gf4"])
@pytest.mark.parametrize("vocab", sorted(TIES))
def test_exact_ties_go_to_the_lowest_index(vocab, dtype):
    """Classifier rows with one nonzero weight give bit-identical logits whatever the order of accumulation: the lowest
    index must win inside a lane, across lanes, across tiles and in a partial last tile.  Blocks of 16 cover 112 rows."""
    spec = replace(mg.SPECS["pf-tiny"], dtype=dtype, vocab_size=vocab, n_layers=1)
    toks = mg.teacher_tokens(vocab, 112)
    for name, fam_p, fam_n in TIES[vocab]:
        tensors = tie_model(spec, fam_p, fam_n, 31)
        w = sr.Weights(spec, tensors)
        greedy, X = [], []
        with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
            for p in range(0, len(toks), 16):
                g, served = dm.verify_greedy(toks[p:p + 16], p)
                assert served == 1
                greedy.append(g)
                X.append(dm.read_state("pf_x").reshape(-1, spec.dim)[:16])
        greedy, X = np.concatenate(greedy), np.concatenate(X)
        xk = sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, False)[:, K_COL]
        tie_check(greedy, np.where(np.abs(xk) > 1e-6 * np.abs(xk).max(), xk, 0), fam_p, fam_n, f"vocab {vocab} {dtype} {name}")


# ---- 3. against the decode
def test_verify_loop_reproduces_the_greedy_stream():
    """test_draft_verification_reproduces_the_greedy_stream's loop and seed (no top-2 margin of the stream inside twice the
    tolerance) on verify_greedy; then the next logits of the decode path stay within the tolerance."""
    spec = mg.SPECS["pf-tiny"]
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    P, N = len(prompt), 48
    tensors = mg.generate(spec, 46)
    stream, logits = greedy_stream(spec, tensors, prompt, N)
    _, margin = top2(logits)
    assert (margin > 2 * TOL_SIGMA * logits.std(1)).all(), "a top-2 margin inside the tolerance; the seed no longer qualifies"
    out, e, seen = [], 0, set()
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        for step in range(len(VERIFY_STEPS) * 3):
            k, bad = VERIFY_STEPS[step % len(VERIFY_STEPS)]
            if e + k + 1 >= N:
                break
            drafts = stream[e + 1:e + 1 + k].copy()
            if bad is not None:
                drafts[bad] = (drafts[bad] + 1) % spec.vocab_size
            greedy, served = dm.verify_greedy(np.concatenate([[stream[e]], drafts]), P - 1 + e)
            assert served == 1 and len(greedy) == k + 1
            acc = 0
            while acc < k and greedy[acc] == drafts[acc]:
                acc += 1
            assert acc == (k if bad is None else bad), f"step {step}: accepted {acc} of {k} drafts (corrupted: {bad})"
            seen.add("all" if acc == k else ("first" if acc == 0 else "mid"))
            out += drafts[:acc].tolist() + [int(greedy[acc])]
            e += acc + 1
        assert seen == {"all", "first", "mid"}
        assert np.array_equal(out, stream[1:e + 1]), "the verify loop does not reproduce the stream"
        nxt = dm.forward(int(stream[e]), P - 1 + e)
    err, sigma = float(np.abs(nxt - logits[e]).max()), float(logits[e].std())
    print(f"  {e} tokens verified; next logits |verify - serial| {err:.2e} = {err / sigma:.1e} sigma")
    assert err <= TOL_SIGMA * sigma


# ---- 4. the lookup loop
def lookup_draft(seq, source, cap):
    """calm_b200_decode_lookup's draft rule: keys of 3, 2, 1 tokens; the rightmost occurrence some token follows."""
    corpus = list(source) if source is not None else list(seq)
    for gl in (3, 2, 1):
        if len(seq) < gl:
            continue
        key = list(seq[-gl:])
        for i in range(len(corpus) - gl - 1, -1, -1):
            if corpus[i:i + gl] == key:
                return corpus[i + gl:i + gl + cap]
    return []


def simulate(tokens, G, n_tokens, source, max_draft, seq_len):
    """The loop's steps when every verification agrees with the stream G: (step count, kind of each step)."""
    seq, pos, e, kinds = [int(t) for t in tokens], len(tokens) - 1, 0, []
    while e < n_tokens:
        cap = min(max_draft, n_tokens - e - 1, seq_len - 1 - pos)
        d = lookup_draft(seq, source, cap) if cap > 0 else []
        if not d:
            kinds.append("none")
            acc = 0
        else:
            acc = 0
            while acc < len(d) and d[acc] == G[e + acc]:
                acc += 1
            kinds.append("all" if acc == len(d) else ("first" if acc == 0 else "mid"))
        seq += [int(t) for t in G[e:e + acc + 1]]
        e, pos = e + acc + 1, pos + acc + 1
    return len(kinds), kinds


@pytest.fixture(scope="module")
def qualified():
    """The seed of test 3: the pf-tiny stream after its 60-token prompt, 48 steps with every top-2 margin clear."""
    spec = mg.SPECS["pf-tiny"]
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    tensors = mg.generate(spec, 46)
    stream, _ = greedy_stream(spec, tensors, prompt, 48)
    return spec, tensors, prompt, stream[1:]


def run_lookup(spec, tensors, prompt, n_tokens, source, max_draft, seq_len=512):
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        return dm.decode_lookup(prompt, n_tokens, source=source, max_draft=max_draft)


@pytest.mark.parametrize("max_draft", [3, 7, 15])
def test_lookup_with_the_stream_as_source(qualified, max_draft):
    spec, tensors, prompt, G = qualified
    n = 47
    source = np.concatenate([prompt, G])
    out, steps = run_lookup(spec, tensors, prompt, n, source, max_draft)
    want, kinds = simulate(prompt, G, n, source, max_draft, 512)
    print(f"  max_draft {max_draft}: {n} tokens in {steps} steps ({kinds.count('all')} fully accepted)")
    assert np.array_equal(out, G[:n]) and steps == want and steps < n


def test_lookup_with_a_corrupted_source(qualified):
    """Every source copy of one stream token replaced by a token the stream never holds: the draft that reaches it is
    rejected there, and after the correction no key matches, since the key's last token no longer occurs in the source.
    The output is still the stream, and the steps include full acceptance, a rejection mid-way and a step without a
    match.  The first stream position whose corruption gives all three (by the Python model) is used."""
    spec, tensors, prompt, G = qualified
    n = 47
    fresh = int(np.setdiff1d(np.arange(spec.vocab_size), np.concatenate([prompt, G]))[0])
    for j in range(4, 40):
        source = np.concatenate([prompt, G])
        source = np.where(source == G[j], fresh, source).astype(np.int32)
        want, kinds = simulate(prompt, G, n, source, 7, 512)
        if {"all", "mid", "none"} <= set(kinds):
            break
    else:
        pytest.fail("no corruption gives every kind of step")
    out, steps = run_lookup(spec, tensors, prompt, n, source, 7)
    print(f"  stream token {j} corrupted: {steps} steps, kinds {kinds}")
    assert np.array_equal(out, G[:n]) and steps == want


def test_lookup_without_a_match_is_decode_greedy():
    """A source that never matches: every step is a decode step, and the tokens are calm_b200_decode_greedy's, bit for
    bit, with no tolerance needed (any seed)."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 5)
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 40, start=2), np.int32)
    n = 60
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        G = dm.decode_greedy(int(prompt[-1]), len(prompt) - 1, n)
    absent = np.setdiff1d(np.arange(spec.vocab_size), np.concatenate([prompt, G]))[:3].astype(np.int32)
    out, steps = run_lookup(spec, tensors, prompt, n, absent, 7)
    assert np.array_equal(out, G) and steps == n
    out, steps = run_lookup(spec, tensors, prompt, n, absent[:0], 7)  # an empty source
    assert np.array_equal(out, G) and steps == n


def test_prompt_lookup_on_a_repeating_prompt():
    """source == NULL: drafts come from the prompt and the tokens emitted so far.  The prompt repeats itself; the run is
    as long as the stream's top-2 margins stay clear of twice the tolerance."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 46)
    half = np.asarray(mg.teacher_tokens(spec.vocab_size, 30, start=11), np.int32)
    prompt = np.concatenate([half, half, half[:10]])
    stream, logits = greedy_stream(spec, tensors, prompt, 40)
    _, margin = top2(logits)
    clear = margin > 2 * TOL_SIGMA * logits.std(1)
    n = int(np.argmin(clear)) if not clear.all() else len(clear)
    assert n >= 16, f"only {n} clear steps: the seed no longer qualifies"
    G = stream[1:]
    out, steps = run_lookup(spec, tensors, prompt, n, None, 7)
    want, kinds = simulate(prompt, G, n, None, 7, 512)
    print(f"  {n} tokens in {steps} steps, kinds {kinds}")
    assert np.array_equal(out, G[:n]) and steps == want
    assert any(k != "none" for k in kinds), "no step drew a draft from the prompt"


def test_lookup_drafts_stop_at_the_end_of_the_cache(qualified):
    """seq_len = prompt + 24: the last cache slot is the last fed token's, and the long drafts shrink to fit."""
    spec, tensors, prompt, G = qualified
    seq_len = len(prompt) + 24
    n = seq_len - len(prompt) + 1
    source = np.concatenate([prompt, G])
    out, steps = run_lookup(spec, tensors, prompt, n, source, 15, seq_len=seq_len)
    want, _ = simulate(prompt, G, n, source, 15, seq_len)
    assert np.array_equal(out, G[:n]) and steps == want


def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        for toks in ([], list(range(17))):
            with pytest.raises(ValueError):
                dm.verify_greedy(np.asarray(toks, np.int32), 0)
        for md in (0, 16, -1):
            with pytest.raises(ValueError):
                dm.decode_lookup([1, 2, 3], 4, max_draft=md)
        with pytest.raises(ValueError):
            dm.decode_lookup([], 4)


# ---- 5. fallback
@pytest.mark.parametrize("name,seq_len,n,pos0", [("tiny-moe", None, 9, 5), ("tiny-fp8", None, 16, 7), ("pf-tiny", 64, 8, 60)])
def test_fallback_is_forward_argmax(name, seq_len, n, pos0):
    """MoE, head_dim 32 and a block past seq_len: served 0 and exactly the results of n forward_argmax calls."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    toks = np.asarray(mg.teacher_tokens(spec.vocab_size, pos0 + n), np.int32)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        dm.prefill(toks[:pos0], 0)
        greedy, served = dm.verify_greedy(toks[pos0:], pos0)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        dm.prefill(toks[:pos0], 0)
        am = np.asarray([dm.forward_argmax(int(t), pos0 + i) for i, t in enumerate(toks[pos0:])], np.int32)
    assert served == 0 and np.array_equal(greedy, am)
    if name != "pf-tiny":
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            dm.prefill(toks[:pos0], 0)
            G = dm.decode_greedy(int(toks[pos0]), pos0, 12)
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            dm.prefill(toks[:pos0], 0)
            out, steps = dm.decode_lookup(toks[:pos0 + 1], 12, source=np.concatenate([toks, G]), max_draft=7)
        assert np.array_equal(out, G) and steps == 12


# ---- 6. history
@pytest.fixture(scope="module")
def weights():
    """Each spec's tensors, generated on the device once and kept while DeviceModels come and go."""
    made = {}

    def get(name):
        if name not in made:
            made[name] = mg.generate(HIST[name], 31, device="cuda")
            torch.cuda.synchronize()
        return made[name]

    yield get
    made.clear()


HIST = {"pf-tiny-v1000": replace(mg.SPECS["pf-tiny"], vocab_size=1000), "llama-2l": replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K)}
BLOCKS = [(16, 60), (1, 76), (7, 77), (9, 84)]  # (n, pos0): consecutive blocks after a 60-token prompt


def verify_run(dm, toks):
    """The prompt, then BLOCKS; every block's greedy tokens and pass rows, and the cache slots they wrote."""
    assert dm.prefill(toks[:60], 0) == 1
    out = []
    for n, p in BLOCKS:
        g, served = dm.verify_greedy(toks[p:p + n], p)
        assert served == 1
        out.append(g)
        out += [dm.read_state(k).reshape(-1, d)[:n] for k, d in (("pf_x", dm.spec.dim), ("pf_q", dm.spec.q_dim))]
    shape = (dm.spec.n_kv_heads, dm.seq_len, dm.spec.head_dim)
    out += [dm.read_state(w, l).reshape(shape)[:, 60:93] for l in range(dm.spec.n_layers) for w in ("keys", "values")]
    return out


@pytest.mark.parametrize("name", sorted(HIST))
@pytest.mark.parametrize("before", ["poison", "score+verify+poison", "prefill+lookup+poison"])
def test_verify_does_not_depend_on_history(weights, name, before):
    spec = HIST[name]
    toks = np.asarray(mg.teacher_tokens(spec.vocab_size, 100, start=4), np.int32)
    other = np.asarray(mg.teacher_tokens(spec.vocab_size, 300, start=9), np.int32)
    with lib.DeviceModel(spec, weights(name), seq_len=512) as dm:
        fresh = verify_run(dm, toks)
        again = verify_run(dm, toks)
    with lib.DeviceModel(spec, weights(name), seq_len=512) as dm:
        if before.startswith("score"):
            dm.score_greedy(other, 0)
            dm.verify_greedy(other[:16], 200)
        elif before.startswith("prefill"):
            dm.prefill(other[:250], 0)
            dm.decode_lookup(other[:251], 30, max_draft=15)
        dm.poison(0)
        dirty = verify_run(dm, toks)
    for i, (f, a, d) in enumerate(zip(fresh, again, dirty)):
        assert np.isfinite(f.astype(np.float64)).all(), f"{name}: item {i} not finite"
        assert np.array_equal(a, f), f"{name}: item {i}: a repeated run differs"
        assert np.array_equal(d, f), f"{name}: item {i}: after {before} the results changed"


def test_zz_summary_of_largest_errors():
    """Runs last in this file: the largest share of its bound each verify stage showed in this session."""
    seen = {k: v for k, v in worst_seen.items() if k.startswith("vf_") or k == "pf_att"}
    if not seen:
        pytest.skip("the stage tests did not run in this session")
    print("\n  largest share of its bound per stage: " + ", ".join(f"{k} {e:.2e} of {tol:.1e}" for k, (e, tol, _) in sorted(seen.items())))
    assert all(e <= tol for e, tol, _ in seen.values())
