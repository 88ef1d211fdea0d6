"""calm_b200_decode_sample_n: nseq continuations of one prompt, one short block per step whose rows are the sequences, with
the shared-prompt split-KV attention of sample_n.cuh (k_sn_attn, k_sn_fold).

1. The last step's stages against float64 fed the device's own previous stage: Q, each row's new cache entries, the
   attention output over each row's gathered keys (prompt plus its own interleaved slots), the hidden and residual rows.
2. Batch invariance: a seed's tokens, state, last logit row and own cache entries are bit-identical alone, as row 0 of 5
   and as row 15 of 16; the prompt's cache slots are bit-identical before and after every call.
3. Each row's last token is lib.sample_logits of its logit row with the state before the last draw; states advance by
   n_tokens draws.
4. On a seed whose every coin sits clear of its bin edges, every sequence is decode_sample's stream and state.
5. Temperature 0: every sequence is decode_greedy's stream on a seed whose top-2 margins are clear; states untouched.
6. Fallback shapes give exactly nseq decode_sample runs.  7. No result depends on history.  8. Bad arguments raise."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_score_greedy_gpu import greedy_stream, top2  # noqa: E402
from test_stages_gpu import DECODE, L8B, V4K, check_entries, layer_cache, make_model, pf_tol, report  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402
from test_verify_sample_gpu import DEFAULT, sampled_stream, xs_advance  # noqa: E402,F401  (sampled_stream is a fixture)

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

SEEDS = [0x9E3779B97F4A7C15 + 7919 * i for i in range(16)]


def own_slots(pos0, nseq, b, steps):
    """Cache slots of sequence b's entries after `steps` steps."""
    return pos0 + np.arange(steps) * nseq + b


def gathered(arr, pos0, nseq, b, steps):
    """Sequence b's keys (or values) in virtual order: the prompt's slots, then its own."""
    return arr[:, np.concatenate([np.arange(pos0), own_slots(pos0, nseq, b, steps)])]


# ---- 1. the last step's stages: (spec, kvbits, nseq, n_tokens, pos0)
STAGES = {
    "llama3-8b fp8 kv_mul4 n16 t9 pos 300": (L8B, 16, 16, 9, 300),  # the prompt ends inside chunk 2
    "llama3-8b fp8 e5m2 n5 t1 pos 256": (L8B, 8, 5, 1, 256),  # the prompt ends on a chunk edge
    "llama3-8b fp16 n1 t10 pos 0": (replace(mg.SPECS["llama3-8b-fp16"], n_layers=1, vocab_size=V4K), 16, 1, 10, 0),  # no prompt
    "llama3-70b kv_mul8 n5 t9 pos 37": (replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K), 16, 5, 9, 37),
    "mistral gf4 e5m2 n16 t1 pos 129": (DECODE["mistral-gf4"][0], 8, 16, 1, 129),  # past a chunk edge
    "pf-tiny hd64 kv_mul2 gf4 n5 t12 pos 37": (replace(TINY1, dtype="gf4"), 16, 5, 12, 37),
    "pf-tiny hd64 kv_mul1 fp16 e5m2 n16 t10 pos 250": (replace(TINY1, dtype="fp16", n_kv_heads=4), 8, 16, 10, 250),  # own keys cross 256
    "pf-tiny-hd128 kv_mul4 bias n16 t1 pos 127": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 16, 16, 1, 127),  # 128 keys: one chunk
    "pf-tiny-hd128 kv_mul4 n1 t9 pos 0": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 8, 1, 9, 0),
}


@pytest.mark.parametrize("case", sorted(STAGES))
def test_last_step_every_stage(case, capfd):
    spec, kvbits, nseq, n_tokens, pos0 = STAGES[case]
    tensors, w = make_model(spec, 4)
    with lib.DeviceModel(spec, tensors, seq_len=1024, kvbits=kvbits) as dm, capfd.disabled():
        dm.fill_kv(pos0, seed=6)
        check_last_step(dm, w, kvbits, nseq, n_tokens, pos0, case)


def check_last_step(dm, w, kvbits, nseq, n_tokens, pos0, case, layer=0):
    """decode_sample_n(3, pos0, n_tokens) for the first nseq SEEDS over the prompt in slots [0, pos0), then the last step's
    stages of `layer` (whose input must be the embedding rows) against float64."""
    spec, token0 = w.spec, 3
    hd, kv_mul, j = spec.head_dim, spec.n_heads // spec.n_kv_heads, n_tokens - 1
    toks, states, served = dm.decode_sample_n(token0, pos0, n_tokens, *DEFAULT, SEEDS[:nseq])
    X = dm.read_state("pf_x").reshape(-1, spec.dim)[:nseq]
    Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:nseq]
    A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:nseq]
    H = dm.read_state("pf_hb").reshape(-1, spec.hidden_dim)[:nseq]
    keys, values = layer_cache(dm, spec, layer)
    assert served == 1, f"{case}: the shared-prompt path did not serve this shape"
    assert states == [xs_advance(s, n_tokens) for s in SEEDS[:nseq]]
    label = f"sample_n {case} kv{kvbits}"
    inputs = toks[:, j - 1] if j > 0 else np.full(nseq, token0)
    X0 = w.mat("model.embed.weight")[inputs].astype(np.float64)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, layer, X0, np.full(nseq, pos0 + j))
    report(label, "Q", "k_vf_gemm QKV", Q, q_ref, np.abs(q_ref).max(), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "vf_q", pf_tol(spec.dim))
    slots = pos0 + j * nseq + np.arange(nseq)
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        got = dev[:, slots].transpose(1, 0, 2).reshape(nseq, -1)
        check_entries(label, name, "k_vf_gemm QKV", got, ref, kvbits, lambda i: f"row {i[0]} kv head {i[1] // hd} dim {i[1] % hd}", "vf_kv", pf_tol(spec.dim))
    a_ref, vmax = [], []
    for b in range(nseq):
        K, V = gathered(keys, pos0, nseq, b, j + 1), gathered(values, pos0, nseq, b, j + 1)
        a_ref.append(sr.attention(spec, Q[b], K, V, pos0 + j + 1))
        vmax.append(np.repeat(np.abs(V).max((1, 2)), kv_mul * hd))
    report(label, "A", "k_sn_attn", A, np.stack(a_ref), np.stack(vmax), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")
    x1 = sr.wo(w, layer, X0, A)
    h_ref = sr.ffn_up(w, layer, sr.ffn_input(w, layer, x1, xn))
    report(label, "H", "k_vf_gemm WO+UP", H, h_ref, np.abs(h_ref).max(), lambda i: f"row {i[0]} hidden row {i[1]}", "vf_hb", pf_tol(max(spec.dim, spec.q_dim)))
    x_ref = sr.ffn_down(w, layer, x1, H)
    report(label, "X", "k_vf_gemm DOWN", X, x_ref, np.abs(x_ref).max(), lambda i: f"row {i[0]} row {i[1]}", "vf_x", pf_tol(spec.hidden_dim))
    return toks


# ---- 2 + 3. batch invariance, the prompt's cache, each row's draw
def own_entries(dm, spec, pos0, nseq, b, steps):
    out = []
    for layer in range(spec.n_layers):
        k, v = dm.read_state("keys", layer), dm.read_state("values", layer)
        shape = (spec.n_kv_heads, dm.seq_len, spec.head_dim)
        s = own_slots(pos0, nseq, b, steps)
        out += [k.reshape(shape)[:, s], v.reshape(shape)[:, s]]
    return out


def prompt_cache(dm, spec, pos0):
    return [dm.read_state(which, layer).reshape(spec.n_kv_heads, dm.seq_len, spec.head_dim)[:, :pos0].copy()
            for layer in range(spec.n_layers) for which in ("keys", "values")]


INVARIANCE = {
    "llama-2l fp8 pos 200": (replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K), 16, 200),
    "pf-tiny vocab 4100 e5m2 pos 90": (replace(mg.SPECS["pf-tiny"], vocab_size=4100), 8, 90),
}


@pytest.mark.parametrize("temperature,minp", [(1.0, 0.1), (1.3, 0.0)])
@pytest.mark.parametrize("case", sorted(INVARIANCE))
def test_a_sequence_does_not_depend_on_its_neighbours(case, temperature, minp):
    spec, kvbits, pos0 = INVARIANCE[case]
    tensors = mg.generate(spec, 21, device="cuda")
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, pos0 + 1, start=5), np.int32)
    n, seed = 12, SEEDS[3]
    runs = {}
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        before = prompt_cache(dm, spec, pos0)
        for nseq, b in ((1, 0), (5, 0), (16, 15)):
            states = [SEEDS[(i + 7) % 16] for i in range(nseq)]
            states[b] = seed
            toks, after, served = dm.decode_sample_n(int(prompt[-1]), pos0, n, temperature, minp, states)
            assert served == 1
            L = dm.read_state("pf_logits").reshape(nseq, dm.vocab)
            # 3. every row's last draw and every state
            for r in range(nseq):
                tok, st = lib.sample_logits(L[r], temperature, minp, xs_advance(states[r], n - 1))
                assert tok == toks[r, -1], f"{case} nseq {nseq} row {r}: last token {toks[r, -1]} vs the reference draw {tok}"
                assert st == after[r] == xs_advance(states[r], n)
            runs[nseq] = [toks[b], np.asarray([after[b]], np.uint64), L[b].copy()] + own_entries(dm, spec, pos0, nseq, b, n)
            for i, (x, y) in enumerate(zip(before, prompt_cache(dm, spec, pos0))):
                assert np.array_equal(x, y), f"{case} nseq {nseq}: prompt cache item {i} changed"
    for nseq in (5, 16):
        for i, (x, y) in enumerate(zip(runs[1], runs[nseq])):
            assert np.array_equal(x, y), f"{case}: item {i} of the seed's results differs between nseq 1 and nseq {nseq}"
    assert np.isfinite(runs[1][2]).all()


# ---- 4. against decode_sample, on a seed whose coins clear their bin edges
@pytest.mark.parametrize("nseq", [1, 16])
def test_every_sequence_is_the_decode_sample_stream(sampled_stream, nseq):  # noqa: F811
    spec, tensors, prompt, seed, G, state = sampled_stream
    P = len(prompt)
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        toks, states, served = dm.decode_sample_n(int(prompt[-1]), P - 1, len(G), *DEFAULT, [seed] * nseq)
    assert served == 1
    for b in range(nseq):
        assert np.array_equal(toks[b], G), f"sequence {b}: {toks[b].tolist()} vs decode_sample {G.tolist()}"
    assert states == [state] * nseq


# ---- 5. greedy
@pytest.mark.parametrize("temperature,minp", [(0.0, 0.1), (1.0, 1.0)])
def test_greedy_settings_give_the_greedy_stream(temperature, minp):
    """test_draft_verification_reproduces_the_greedy_stream's model seed: no top-2 margin of the stream inside the tolerance."""
    spec = mg.SPECS["pf-tiny"]
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    P, N = len(prompt), 24
    tensors = mg.generate(spec, 46)
    stream, logits = greedy_stream(spec, tensors, prompt, N)
    best, margin = top2(logits)
    assert (margin > 2 * TOL_SIGMA * logits.std(1)).all()
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        toks, states, served = dm.decode_sample_n(int(prompt[-1]), P - 1, N, temperature, minp, SEEDS[:7])
    assert served == 1 and states == SEEDS[:7]
    for b in range(7):
        assert np.array_equal(toks[b], stream[1:]), f"sequence {b}: {toks[b].tolist()} vs decode_greedy {stream[1:].tolist()}"


# ---- 6. fallback
@pytest.mark.parametrize("name,seq_len,nseq,n,pos0", [("tiny-moe", None, 3, 9, 5), ("pf-tiny", 64, 4, 8, 40)])
def test_fallback_is_decode_sample_per_sequence(name, seq_len, nseq, n, pos0):
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, pos0 + 1), np.int32)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        dm.prefill(prompt[:-1], 0)
        toks, states, served = dm.decode_sample_n(int(prompt[-1]), pos0, n, *DEFAULT, SEEDS[:nseq])
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        dm.prefill(prompt[:-1], 0)
        want = [dm.decode_sample(int(prompt[-1]), pos0, n, *DEFAULT, s) for s in SEEDS[:nseq]]
    assert served == 0
    assert np.array_equal(toks, np.stack([t for t, _ in want])) and states == [s for _, s in want]


# ---- 7. history
HIST = {"pf-tiny-v1000": replace(mg.SPECS["pf-tiny"], vocab_size=1000), "llama-2l": replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K)}


def sample_n_run(dm, prompt, pos0):
    out = []
    for nseq, n in ((16, 6), (5, 13), (1, 3)):
        toks, states, served = dm.decode_sample_n(int(prompt[-1]), pos0, n, *DEFAULT, SEEDS[:nseq])
        assert served == 1
        out += [toks, np.asarray(states, np.uint64), dm.read_state("pf_logits"), dm.read_state("pf_x").reshape(-1, dm.spec.dim)[:nseq],
                dm.read_state("pf_att").reshape(-1, dm.spec.q_dim)[:nseq]]
    return out


@pytest.mark.parametrize("name", sorted(HIST))
def test_decode_sample_n_does_not_depend_on_history(name):
    spec = HIST[name]
    tensors = mg.generate(spec, 31, device="cuda")
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 141, start=4), np.int32)
    other = np.asarray(mg.teacher_tokens(spec.vocab_size, 300, start=9), np.int32)
    pos0 = len(prompt) - 1
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        fresh = sample_n_run(dm, prompt, pos0)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        dm.prefill(other[:250], 0)
        dm.decode_sample_n(int(other[250]), 250, 16, 0.8, 0.02, SEEDS)  # more chunks than the runs need
        dm.verify_sample(other[:16], 200, 1.3, 0.0, 12)
        assert dm.prefill(prompt[:-1], 0) == 1
        dm.poison(pos0)
        dirty = sample_n_run(dm, prompt, pos0)
    for i, (f, d) in enumerate(zip(fresh, dirty)):
        if f.dtype.kind == "f":
            assert np.isfinite(f).all(), f"{name}: item {i} not finite"
        assert np.array_equal(d, f), f"{name}: item {i}: after another history and poisoning the results changed"


# ---- 8. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        for states in ([], SEEDS + [1], None, 5, [1, -1], [1, 1 << 64]):
            with pytest.raises(ValueError):
                dm.decode_sample_n(1, 0, 4, *DEFAULT, states)
        for n in (-1, 2.5):
            with pytest.raises(ValueError):
                dm.decode_sample_n(1, 0, n, *DEFAULT, [1])
        for tok in (-1, spec.vocab_size):
            with pytest.raises(ValueError):
                dm.decode_sample_n(tok, 0, 4, *DEFAULT, [1])
        with pytest.raises(ValueError):
            dm.decode_sample_n(1, -1, 4, *DEFAULT, [1])
        toks, states, served = dm.decode_sample_n(1, 0, 0, *DEFAULT, [9, 10])  # nothing wanted: no draw
        assert toks.shape == (2, 0) and states == [9, 10] and served == 1
