"""calm_b200_decode_sample_batch: nseq sequences with their own prompts.  The prompts go through the prompt pass packed from
cache slot 0 (k_pf_attn<.., SEG> at nonzero block bases, prompts straddling the 2048-row block edge), then every step is
one short block whose rows are the sequences, each attending over its own prompt and its own interleaved slots
(sample_n.cuh's BATCH kernels).

1. The last step's stages against float64 fed the device's own previous stage: Q, each row's new cache entries, the
   attention output over each row's gathered keys (its prompt's slots, then its own), the hidden and residual rows.
2. Prefill: prompt b's cache entries at [s_b, s_b + L_b) are bit for bit forward_prefill_cuda's of the prompt alone.
3. A sequence equals itself alone: its tokens, state, last logit row and own cache entries are bit-identical to
   forward_prefill_cuda + decode_sample_n(nseq = 1) of its prompt, as row 0 of 1, row 0 of 5 and row 15 of 16; each row's
   last token is lib.sample_logits of its logit row; states advance by n_tokens draws (untouched at temperature 0).
4. On a seed whose every coin clears its bin edges, the sequences are decode_sample's stream; at temperature 0 on a seed
   with clear top-2 margins, decode_greedy's.
5. Fallback shapes give exactly the per-sequence prefill + decode_sample pairs.  6. No result depends on history.
7. Bad arguments raise."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_decode_sample_n_gpu import SEEDS  # noqa: E402
from test_score_greedy_gpu import greedy_stream, top2  # noqa: E402
from test_stages_gpu import DECODE, L8B, V4K, check_entries, layer_cache, make_model, pf_tol, report  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402
from test_verify_sample_gpu import DEFAULT, sampled_stream, xs_advance  # noqa: E402,F401  (sampled_stream is a fixture)

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu


def layout(lens):
    """(first slot s_b of every prompt's L_b = len - 1 entries, G = the end of the packed prompt region)."""
    rows = [-(-(n - 1) // 8) * 8 for n in lens]
    starts = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(int)
    return starts, int(sum(rows))


def own_slots(G, nseq, b, steps):
    """Cache slots of sequence b's decoded entries after `steps` steps."""
    return G + np.arange(steps) * nseq + b


def prompts_of(vocab, lens, start=0):
    return [np.asarray(mg.teacher_tokens(vocab, n, start=start + 31 * b), np.int32) for b, n in enumerate(lens)]


# ---- 1. the last step's stages: (spec, kvbits, prompt lengths, n_tokens, seq_len)
# Prompt lengths len = L + 1: L = 0 (no prompt rows); prompts ending inside a 128-key chunk (300), on its edge (256) and
# past it (129); prompts longer than a 2048-row block, and prompts straddling the block edges at slots 2048 and 4096.
LONG16 = [301, 257, 130, 1, 1500, 2101, 40, 5, 129, 128, 1, 64, 700, 9, 17, 300]
STAGES = {
    "llama3-8b fp8 kv_mul4 n16 t9": (L8B, 16, LONG16, 9, 8192),
    "llama3-8b fp8 e5m2 n5 t1": (L8B, 8, [129, 2300, 1, 257, 40], 1, 4096),
    "llama3-8b fp16 n1 t10 no prompt": (replace(mg.SPECS["llama3-8b-fp16"], n_layers=1, vocab_size=V4K), 16, [1], 10, 1024),
    "llama3-70b kv_mul8 n5 t9": (replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K), 16, [38, 1, 2060, 129, 60], 9, 4096),
    "mistral gf4 e5m2 n16 t1": (DECODE["mistral-gf4"][0], 8, [1 + 37 * b for b in range(16)], 1, 8192),
    "pf-tiny hd64 kv_mul2 gf4 n5 t12": (replace(TINY1, dtype="gf4"), 16, [37, 1, 250, 129, 1], 12, 1024),
    "pf-tiny hd64 kv_mul1 fp16 e5m2 n16 t10": (replace(TINY1, dtype="fp16", n_kv_heads=4), 8, LONG16, 10, 8192),
    "pf-tiny-hd128 kv_mul4 bias n16 t1": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 16, [128 + b for b in range(16)], 1, 4096),
    "pf-tiny-hd128 kv_mul4 e5m2 n1 t9 long": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 8, [2100], 9, 4096),
}


@pytest.mark.parametrize("case", sorted(STAGES))
def test_last_step_every_stage(case, capfd):
    spec, kvbits, lens, n_tokens, seq_len = STAGES[case]
    tensors, w = make_model(spec, 4)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm, capfd.disabled():
        check_last_step(dm, w, kvbits, lens, n_tokens, case)


def check_last_step(dm, w, kvbits, lens, n_tokens, case):
    """decode_sample_batch of prompts of these lengths for n_tokens, then the last step's stages against float64."""
    spec = w.spec
    nseq, j = len(lens), n_tokens - 1
    prompts = prompts_of(spec.vocab_size, lens, start=3)
    starts, G = layout(lens)
    L = np.asarray(lens) - 1
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    toks, states, served = dm.decode_sample_batch(prompts, n_tokens, *DEFAULT, SEEDS[:nseq])
    X = dm.read_state("pf_x").reshape(-1, spec.dim)[:nseq]
    Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:nseq]
    A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:nseq]
    H = dm.read_state("pf_hb").reshape(-1, spec.hidden_dim)[:nseq]
    keys, values = layer_cache(dm, spec)
    assert served == 1, f"{case}: the packed path did not serve this shape"
    assert states == [xs_advance(s, n_tokens) for s in SEEDS[:nseq]]
    label = f"sample_batch {case} kv{kvbits}"
    inputs = toks[:, j - 1] if j > 0 else np.asarray([p[-1] for p in prompts])
    X0 = w.mat("model.embed.weight")[inputs].astype(np.float64)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, 0, X0, L + j)
    report(label, "Q", "k_vf_gemm QKV", Q, q_ref, np.abs(q_ref).max(), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "vf_q", pf_tol(spec.dim))
    slots = G + j * nseq + np.arange(nseq)
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        got = dev[:, slots].transpose(1, 0, 2).reshape(nseq, -1)
        check_entries(label, name, "k_vf_gemm QKV", got, ref, kvbits, lambda i: f"row {i[0]} kv head {i[1] // hd} dim {i[1] % hd}", "vf_kv", pf_tol(spec.dim))
    a_ref, vmax = [], []
    for b in range(nseq):
        idx = np.concatenate([starts[b] + np.arange(L[b]), own_slots(G, nseq, b, j + 1)])
        K, V = keys[:, idx], values[:, idx]
        a_ref.append(sr.attention(spec, Q[b], K, V, L[b] + j + 1))
        vmax.append(np.repeat(np.abs(V).max((1, 2)), kv_mul * hd))
    report(label, "A", "k_sn_attn BATCH", A, np.stack(a_ref), np.stack(vmax), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")
    x1 = sr.wo(w, 0, X0, A)
    h_ref = sr.ffn_up(w, 0, sr.ffn_input(w, 0, x1, xn))
    report(label, "H", "k_vf_gemm WO+UP", H, h_ref, np.abs(h_ref).max(), lambda i: f"row {i[0]} hidden row {i[1]}", "vf_hb", pf_tol(max(spec.dim, spec.q_dim)))
    x_ref = sr.ffn_down(w, 0, x1, H)
    report(label, "X", "k_vf_gemm DOWN", X, x_ref, np.abs(x_ref).max(), lambda i: f"row {i[0]} row {i[1]}", "vf_x", pf_tol(spec.hidden_dim))


# ---- 2. the packed prompt pass leaves each prompt's entries exactly as the prompt alone does
def cache_rows(dm, spec, slots):
    shape = (spec.n_kv_heads, dm.seq_len, spec.head_dim)
    return [dm.read_state(which, layer).reshape(shape)[:, slots].copy() for layer in range(spec.n_layers) for which in ("keys", "values")]


@pytest.mark.parametrize("kvbits", [16, 8])
def test_packed_prompts_are_each_prompt_alone(kvbits):
    spec = replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K)
    tensors = mg.generate(spec, 12, device="cuda")
    lens = [300, 1, 1900, 2101, 129, 40]  # the third straddles slot 2048, the fourth is longer than a block and straddles 4096
    prompts = prompts_of(spec.vocab_size, lens, start=7)
    starts, G = layout(lens)
    with lib.DeviceModel(spec, tensors, seq_len=8192, kvbits=kvbits) as dm:
        _, _, served = dm.decode_sample_batch(prompts, 2, *DEFAULT, SEEDS[:len(lens)])
        assert served == 1
        packed = [cache_rows(dm, spec, starts[b] + np.arange(n - 1)) for b, n in enumerate(lens)]
    with lib.DeviceModel(spec, tensors, seq_len=8192, kvbits=kvbits) as dm:
        for b, p in enumerate(prompts):
            assert dm.prefill(p[:-1], 0) == 1
            for i, (x, y) in enumerate(zip(packed[b], cache_rows(dm, spec, np.arange(len(p) - 1)))):
                assert np.array_equal(x, y), f"prompt {b} (len {len(p)}, slot {starts[b]}): cache item {i} differs from the prompt alone"


# ---- 3. a sequence equals itself alone, wherever it sits in the batch
def lone_run(spec, tensors, kvbits, prompt, n, temperature, minp, seed):
    """forward_prefill_cuda + decode_sample_n(nseq = 1): tokens, state, own cache entries and, sampled, the last logit row."""
    with lib.DeviceModel(spec, tensors, seq_len=4096, kvbits=kvbits) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        toks, after, served = dm.decode_sample_n(int(prompt[-1]), len(prompt) - 1, n, temperature, minp, [seed])
        assert served == 1
        out = [toks[0], np.asarray(after, np.uint64)] + cache_rows(dm, spec, len(prompt) - 1 + np.arange(n))
        if temperature > 0:
            out.append(dm.read_state("pf_logits").reshape(-1, dm.vocab)[0].copy())
        return out


INVARIANCE = {
    "llama-2l fp8": (replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K), 16, 200),
    "pf-tiny vocab 4100 e5m2": (replace(mg.SPECS["pf-tiny"], vocab_size=4100), 8, 90),
}


@pytest.mark.parametrize("temperature,minp", [(1.0, 0.1), (1.3, 0.0), (0.0, 0.1)])
@pytest.mark.parametrize("case", sorted(INVARIANCE))
def test_a_sequence_is_itself_alone(case, temperature, minp):
    spec, kvbits, plen = INVARIANCE[case]
    tensors = mg.generate(spec, 21, device="cuda")
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, plen + 1, start=5), np.int32)
    n, seed = 12, SEEDS[3]
    greedy = temperature == 0.0
    want = lone_run(spec, tensors, kvbits, prompt, n, temperature, minp, seed)
    with lib.DeviceModel(spec, tensors, seq_len=4096, kvbits=kvbits) as dm:
        for nseq, b in ((1, 0), (5, 0), (16, 15)):
            lens = [1 + (37 * i + 11) % 260 for i in range(nseq)]
            prompts = prompts_of(spec.vocab_size, lens, start=40)
            prompts[b] = prompt
            lens[b] = len(prompt)
            starts, G = layout(lens)
            states = [SEEDS[(i + 7) % 16] for i in range(nseq)]
            states[b] = seed
            toks, after, served = dm.decode_sample_batch(prompts, n, temperature, minp, states)
            assert served == 1
            got = [toks[b], np.asarray([after[b]], np.uint64)] + cache_rows(dm, spec, own_slots(G, nseq, b, n))
            if greedy:
                assert after == states, f"{case} nseq {nseq}: temperature 0 moved the states"
            else:
                Lg = dm.read_state("pf_logits").reshape(nseq, dm.vocab)
                for r in range(nseq):  # every row's last draw and every state
                    tok, st = lib.sample_logits(Lg[r], temperature, minp, xs_advance(states[r], n - 1))
                    assert tok == toks[r, -1], f"{case} nseq {nseq} row {r}: last token {toks[r, -1]} vs the reference draw {tok}"
                    assert st == after[r] == xs_advance(states[r], n)
                got.append(Lg[b].copy())
            assert len(got) == len(want)
            for i, (x, y) in enumerate(zip(want, got)):
                assert np.array_equal(x, y), f"{case} T {temperature}: item {i} of row {b} of {nseq} differs from the sequence alone"
    assert greedy or np.isfinite(want[-1]).all()


# ---- 4. against decode_sample on a seed whose coins clear their bin edges, and decode_greedy on clear margins
@pytest.mark.parametrize("nseq", [1, 16])
def test_sequences_are_the_decode_sample_stream(sampled_stream, nseq):  # noqa: F811
    spec, tensors, prompt, seed, Gs, state = sampled_stream
    clear = {b for b in (0, 3, nseq - 1) if b < nseq}
    prompts = prompts_of(spec.vocab_size, [5 + 9 * b for b in range(nseq)], start=70)
    states = [SEEDS[b] for b in range(nseq)]
    for b in clear:
        prompts[b], states[b] = prompt, seed
    with lib.DeviceModel(spec, tensors, seq_len=2048) as dm:
        toks, after, served = dm.decode_sample_batch(prompts, len(Gs), *DEFAULT, states)
    assert served == 1
    for b in clear:
        assert np.array_equal(toks[b], Gs), f"sequence {b}: {toks[b].tolist()} vs decode_sample {Gs.tolist()}"
        assert after[b] == state


@pytest.mark.parametrize("temperature,minp", [(0.0, 0.1), (1.0, 1.0)])
def test_greedy_settings_give_the_greedy_stream(temperature, minp):
    """test_draft_verification_reproduces_the_greedy_stream's model seed: no top-2 margin of the stream inside the tolerance."""
    spec = mg.SPECS["pf-tiny"]
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    N = 24
    tensors = mg.generate(spec, 46)
    stream, logits = greedy_stream(spec, tensors, prompt, N)
    _, margin = top2(logits)
    assert (margin > 2 * TOL_SIGMA * logits.std(1)).all()
    prompts = prompts_of(spec.vocab_size, [3, 60, 1, 90, 17, 60, 33], start=2)
    for b in (1, 5):
        prompts[b] = prompt
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        toks, states, served = dm.decode_sample_batch(prompts, N, temperature, minp, SEEDS[:7])
    assert served == 1 and states == SEEDS[:7]
    for b in (1, 5):
        assert np.array_equal(toks[b], stream[1:]), f"sequence {b}: {toks[b].tolist()} vs decode_greedy {stream[1:].tolist()}"


# ---- 5. fallback
@pytest.mark.parametrize("name,seq_len,lens,n", [("tiny-moe", None, [6, 1, 12], 9), ("pf-tiny", 64, [21, 30, 11], 8)])
def test_fallback_is_prefill_and_decode_sample_per_sequence(name, seq_len, lens, n):
    """A MoE model, and a served shape whose packed layout (here 24 + 32 + 16 prompt slots and 3 x 8 step slots) passes
    seq_len while each sequence alone fits."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    prompts = prompts_of(spec.vocab_size, lens, start=1)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        toks, states, served = dm.decode_sample_batch(prompts, n, *DEFAULT, SEEDS[:len(lens)])
    want = []
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        for p, s in zip(prompts, SEEDS):
            dm.prefill(p[:-1], 0)
            want.append(dm.decode_sample(int(p[-1]), len(p) - 1, n, *DEFAULT, s))
    assert served == 0
    assert np.array_equal(toks, np.stack([t for t, _ in want])) and states == [s for _, s in want]


# ---- 6. history
HIST = {"pf-tiny-v1000": replace(mg.SPECS["pf-tiny"], vocab_size=1000), "llama-2l": replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K)}


def batch_run(dm, spec):
    out = []
    for lens, n in (([141, 1, 300, 9, 2200] + [20 + 7 * i for i in range(11)], 6), ([50, 129, 1, 77, 256], 13), ([141], 3)):
        prompts = prompts_of(spec.vocab_size, lens, start=4)
        toks, states, served = dm.decode_sample_batch(prompts, n, *DEFAULT, SEEDS[:len(lens)])
        assert served == 1
        nseq = len(lens)
        out += [toks, np.asarray(states, np.uint64), dm.read_state("pf_logits"), dm.read_state("pf_x").reshape(-1, spec.dim)[:nseq],
                dm.read_state("pf_att").reshape(-1, spec.q_dim)[:nseq]]
    return out


@pytest.mark.parametrize("name", sorted(HIST))
def test_decode_sample_batch_does_not_depend_on_history(name):
    spec = HIST[name]
    tensors = mg.generate(spec, 31, device="cuda")
    other = np.asarray(mg.teacher_tokens(spec.vocab_size, 3000, start=9), np.int32)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        fresh = batch_run(dm, spec)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        dm.prefill(other[:250], 0)
        dm.decode_sample_n(int(other[250]), 250, 16, 0.8, 0.02, SEEDS)
        dm.decode_sample_batch([other[:2800], other[5:100]], 40, 1.1, 0.0, SEEDS[:2])  # more chunks than the runs need
        dm.verify_sample(other[:16], 200, 1.3, 0.0, 12)
        dm.poison(0)
        dirty = batch_run(dm, spec)
    for i, (f, d) in enumerate(zip(fresh, dirty)):
        if f.dtype.kind == "f":
            assert np.isfinite(f).all(), f"{name}: item {i} not finite"
        assert np.array_equal(d, f), f"{name}: item {i}: after another history and poisoning the results changed"


# ---- 7. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        for prompts, states in (([], []), (good * 17, SEEDS + [1]), (None, [1]), (good, None), (good, 5), (good, [1, 2]), (good, [-1]), (good, [1 << 64])):
            with pytest.raises(ValueError):
                dm.decode_sample_batch(prompts, 4, *DEFAULT, states)
        for n in (-1, 2.5):
            with pytest.raises(ValueError):
                dm.decode_sample_batch(good, n, *DEFAULT, [1])
        for bad in ([], [-1, 2], [3, spec.vocab_size], [[1, 2]], [0.5]):
            with pytest.raises(ValueError):
                dm.decode_sample_batch([good[0], bad], 4, *DEFAULT, [1, 2])
        toks, states, served = dm.decode_sample_batch(good * 2, 0, *DEFAULT, [9, 10])  # nothing wanted: no draw
        assert toks.shape == (2, 0) and states == [9, 10] and served == 1
