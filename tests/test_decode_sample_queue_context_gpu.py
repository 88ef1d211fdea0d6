"""calm_b200_decode_sample_queue_context: the queue with prompts that share contexts, each context computed once while its
requests are in flight and its whole chunks read once per step for all of them.

1. Every request equals decode_sample_batch over its concatenated prompt alone with n_tokens = its out_len: tokens,
   final state and out_len, bit for bit, across shapes, kv_mul 1 / 2 / 4 / 7 / 8, both caches, max_rows 1 / 3 / 16,
   contexts of 1 .. 2100 tokens (across chunk and prompt-pass block edges), own prompts of 1 token, stops and max_new 0.
2. With every ctx_len 0 the call is decode_sample_queue: the same outputs and steps, and the rows it computed.
3. steps and prompt_rows are the documented rule's, simulated here, including a tight cache where admission waits and a
   context is released and placed again.
4. n samples through the queue (context = prompt[:-1], own = prompt[-1:]) are decode_sample_n of that prompt.
5. The outputs do not depend on what earlier calls left behind.
6. The last step's stages against float64, with each row's keys gathered from its context, its own prompt and its own
   generated slots.  7. The fallback and bad arguments."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from test_decode_sample_queue_gpu import HD128, SEEDS, SETTINGS, Slots, ceil8, greedy_setting, lone, prompts_of, queue  # noqa: E402
from test_stages_gpu import L8B, V4K, check_entries, layer_cache, make_model, pf_tol, report  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402
from test_verify_sample_gpu import xs_advance  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

CHUNK = 128  # SN_CHUNK: a chunk wholly inside a context is shared by the context's rows


def place_round(slots, rs, key, clen, lens, max_new, resident):
    """include/calm_b200.h's placement of a round: ({request: (s, L, t, c, nc)}, rows of the prompt extent) or None."""
    P, placed = 0, {}
    for i in rs:
        if clen[i] and key[i] not in resident and key[i] not in placed:
            placed[key[i]] = P
            P += ceil8(clen[i])
        P += ceil8(lens[i] - 1)
    s0 = slots.take(P, 8) if P else 0
    if s0 < 0:
        return None
    out, seen, s = {}, set(), s0
    for i in rs:
        c = 0
        if clen[i]:
            if key[i] in resident:
                c = resident[key[i]]
            else:
                c = s0 + placed[key[i]]
                if key[i] not in seen:
                    seen.add(key[i])
                    s += ceil8(clen[i])
        t = slots.take(max_new[i], 1)
        if t < 0:
            return None
        out[i] = (s, clen[i] + lens[i] - 1, t, c, clen[i])
        s += ceil8(lens[i] - 1)
    return out, P


def simulate(key, clen, lens, max_new, out_len, max_rows, seq_len):
    """The documented schedule given each request's out_len: (every step's rows [(request, own step)], placement,
    prompt rows, the contexts in the order they were placed, waited, released)."""
    n = len(lens)
    st = dict(slots=Slots(seq_len), head=0, waited=False, released=0)
    resident, place, live, done, steps, placed, rows = {}, {}, [], {}, [], [], 0

    def admit():
        rnd, rp, after, P = [], {}, st["slots"], 0
        while st["head"] < n and len(live) + len(rnd) < max_rows:
            h = st["head"]
            if max_new[h] == 0:
                st["head"] += 1
                continue
            a = st["slots"].copy()
            r = place_round(a, rnd + [h], key, clen, lens, max_new, resident)
            if r is None:
                st["waited"] = True
                break
            rnd, (rp, P), after = rnd + [h], r, a
            st["head"] += 1
        st["slots"] = after
        return rnd, rp, P

    while True:
        rnd, rp, P = admit()
        named = {key[i] for i in live + rnd if clen[i]}
        for k in [k for k in resident if k not in named]:
            st["slots"].give(resident.pop(k), ceil8(k[1]))
            st["released"] += 1
        if not live and not rnd:
            rnd, rp, P = admit()
            if not rnd:
                break
        for i in rnd:
            if clen[i] and key[i] not in resident:
                resident[key[i]] = rp[i][3]
                placed.append(key[i])
        place.update(rp)
        rows += P
        live += rnd
        steps.append([(i, done.get(i, 0)) for i in live])
        keep = []
        for i in live:
            done[i] = done.get(i, 0) + 1
            if done[i] < out_len[i]:
                keep.append(i)
            else:
                s, _, t, _, _ = place[i]
                st["slots"].give(s, ceil8(lens[i] - 1))
                st["slots"].give(t, max_new[i])
        live[:] = keep
    return steps, place, rows, placed, st["waited"], st["released"]


def layout(contexts, ctx_of, prompts):
    """decode_sample_queue_context's keys for the simulation: (key, ctx_len) per request, a context's key its (offset,
    length) in the laid-out tokens."""
    starts = np.concatenate([[0], np.cumsum([len(c) for c in contexts])])
    key = [(int(starts[c]), len(contexts[c])) if c >= 0 else (0, 0) for c in ctx_of]
    return key, [k[1] for k in key]


def concat(contexts, c, p):
    return np.concatenate([contexts[c], p]).astype(np.int32) if c >= 0 else p


def qctx(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows):
    return dm.decode_sample_queue_context(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds)


def shared_groups(steps, key, clen):
    """Whether some step runs two rows of one context with at least one shared chunk at different own steps."""
    for rows in steps:
        by = {}
        for i, j in rows:
            if clen[i] >= CHUNK:
                by.setdefault(key[i], set()).add(j)
        if any(len(js) >= 2 for js in by.values()):
            return True
    return False


# ---- 1. every request equals decode_sample_batch over its concatenated prompt alone
QWEN = replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=1, vocab_size=V4K)
KV1 = replace(mg.SPECS["pf-tiny"], name="kv1", n_kv_heads=4, n_layers=1)
L70 = replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K)
ALL_CTX = [1, 7, 8, 127, 128, 129, 2047, 2048, 2100]
MIXED = {"pf-tiny fp8 kv_mul2 r16", "pf-tiny gf4 e5m2 r3", "llama3-70b widths kv_mul8 e5m2 r3"}  # a group's rows admitted in different rounds
ALONE = {  # (spec, kvbits, max_rows, nreq, context lengths, own lengths, seq_len)
    "pf-tiny fp8 kv_mul2 r16": (mg.SPECS["pf-tiny"], 16, 16, 30, ALL_CTX, [1, 9, 300, 2, 40], 8192),
    "pf-tiny gf4 e5m2 r3": (replace(mg.SPECS["pf-tiny"], dtype="gf4"), 8, 3, 20, [2047, 128, 7], [300, 1, 9, 2], 8192),
    "pf-tiny fp16 r1": (replace(TINY1, dtype="fp16"), 16, 1, 10, [129, 8], [1, 9, 40], 4096),
    "kv1 r3": (KV1, 16, 3, 14, [2048, 1, 127], [9, 1, 300], 8192),
    "hd128 bias e5m2 kv_mul4 r16": (HD128, 8, 16, 20, [2100, 129, 1], [9, 1, 40, 2], 8192),
    "llama3-8b widths kv_mul4 r16": (L8B, 16, 16, 20, [2100, 128, 7], [1, 300, 9, 2], 8192),
    "llama3-70b widths kv_mul8 e5m2 r3": (L70, 8, 3, 10, [129, 2047], [9, 1, 40], 4096),
    "qwen2 widths kv_mul7 r16": (QWEN, 16, 16, 16, [300, 8, 129], [1, 9, 40], 4096),
}


def alone_requests(vocab, nreq, ctx_lens, own_lens):
    contexts = prompts_of(vocab, ctx_lens, start=101)
    ctx_of = [-1 if i % 5 == 3 else i % len(contexts) for i in range(nreq)]
    prompts = prompts_of(vocab, [own_lens[i % len(own_lens)] for i in range(nreq)], start=7)
    max_new = [[0, 1, 7, 40][(3 * i + 1) % 4] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    return contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq]


@pytest.mark.parametrize("case", sorted(ALONE))
def test_each_request_is_its_concatenated_prompt_alone(case):
    spec, kvbits, max_rows, nreq, ctx_lens, own_lens, seq_len = ALONE[case]
    tensors = mg.generate(spec, 17, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = alone_requests(spec.vocab_size, nreq, ctx_lens, own_lens)
    key, clen = layout(contexts, ctx_of, prompts)
    lens = [len(p) for p in prompts]
    cat = [concat(contexts, c, p) for c, p in zip(ctx_of, prompts)]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        full = [lone(dm, p, m, *s, seed) if m else (np.zeros(0, np.int32), seed) for p, m, s, seed in zip(cat, max_new, sets, seeds)]
        long = [i for i in range(nreq) if max_new[i] == 40]
        stop = [int(full[long[0]][0][0]), int(full[long[1]][0][20]), int(full[long[-1]][0][39])]
        for stops in ([], stop):
            want_len = []
            for i in range(nreq):
                hit = [k for k, tok in enumerate(full[i][0]) if tok in stops]
                want_len.append(min(max_new[i], hit[0] + 1) if hit else max_new[i])
            toks, states, served, steps, rows = qctx(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stops, max_rows)
            assert served == 1
            assert [len(x) for x in toks] == want_len, f"{case} stop {stops}: out_len"
            sched, _, want_rows, _, _, _ = simulate(key, clen, lens, max_new, want_len, max_rows, seq_len)
            assert (steps, rows) == (len(sched), want_rows), f"{case} stop {stops}: steps / prompt rows"
            if case in MIXED and not stops:
                assert shared_groups(sched, key, clen), f"{case}: no step ran a context's rows at different own steps"
            for i in range(nreq):
                if want_len[i] < max_new[i]:
                    want = lone(dm, cat[i], want_len[i], *sets[i], seeds[i]) if want_len[i] else (np.zeros(0, np.int32), seeds[i])
                else:
                    want = full[i]
                assert np.array_equal(toks[i], want[0]), f"{case} stop {stops}: request {i} (context {ctx_of[i]}) differs from its prompt alone"
                assert states[i] == want[1], f"{case} stop {stops}: request {i} state"
                assert states[i] == (seeds[i] if greedy_setting(*sets[i]) else xs_advance(seeds[i], want_len[i]))
            if stops:
                assert want_len[long[0]] == 1


# ---- 2. every ctx_len 0 is decode_sample_queue
def test_no_context_is_the_queue():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    tensors = mg.generate(spec, 23, device="cuda")
    lens = [129, 9, 300, 1, 40, 2] * 3
    prompts = prompts_of(spec.vocab_size, lens, start=3)
    max_new = [[13, 1, 40, 7, 0, 25][i % 6] for i in range(len(lens))]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    with lib.DeviceModel(spec, tensors, seq_len=2048) as dm:
        for max_rows in (1, 5, 16):
            want = queue(dm, prompts, max_new, sets, SEEDS[:len(lens)], [], max_rows)
            got = qctx(dm, [np.zeros(0, np.int32)], [0 if i % 2 else -1 for i in range(len(lens))], prompts, max_new, sets, SEEDS[:len(lens)], [], max_rows)
            assert got[1:4] == want[1:4]
            assert all(np.array_equal(x, y) for x, y in zip(got[0], want[0]))
            assert got[4] == sum(ceil8(n - 1) for n, m in zip(lens, max_new) if m)


# ---- 3. steps and prompt_rows are the rule's, with waits, releases and recomputed contexts
def test_schedule_is_the_documented_rule():
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 5, device="cuda")
    contexts = prompts_of(spec.vocab_size, [300, 200, 129], start=11)
    ctx_of = [0, 0, 1, 1, 0, -1, 2, 0, 2, 1, 0, 0]
    lens = [9, 1, 40, 2, 17, 30, 1, 8, 64, 3, 5, 12]
    max_new = [20, 5, 30, 1, 12, 9, 0, 14, 7, 22, 3, 11]
    prompts = prompts_of(spec.vocab_size, lens, start=5)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    key, clen = layout(contexts, ctx_of, prompts)
    tight = max(ceil8(c) + ceil8(n - 1) + m for c, n, m in zip(clen, lens, max_new)) + 24
    for seq_len, max_rows in ((4096, 16), (4096, 3), (tight, 16), (tight, 2)):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            toks, _, served, steps, rows = qctx(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:len(lens)], [], max_rows)
        assert served == 1 and [len(x) for x in toks] == max_new
        sched, _, want_rows, placed, waited, released = simulate(key, clen, lens, max_new, max_new, max_rows, seq_len)
        assert (steps, rows) == (len(sched), want_rows), f"seq_len {seq_len} max_rows {max_rows}"
        if seq_len == tight:
            assert waited and released, "the tight cache never made admission wait or released a context"
            assert len(placed) > len(set(placed)), "no context was placed twice"
            assert rows > sum(ceil8(c) for c in {k[1] for k in key if k[1]}) + sum(ceil8(n - 1) for n, m in zip(lens, max_new) if m)
        if seq_len == 4096 and max_rows == 16:
            assert len(placed) == len(set(placed)), "a context was computed twice in a roomy cache"


# ---- 4. n samples through the queue are decode_sample_n
@pytest.mark.parametrize("plen", [257, 1000])
def test_n_samples_are_decode_sample_n(plen):
    spec = replace(mg.SPECS["pf-tiny"], n_layers=1)
    tensors = mg.generate(spec, 9, device="cuda")
    prompt = prompts_of(spec.vocab_size, [plen], start=2)[0]
    n_tokens, (t, p) = 24, (0.9, 0.05)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        dm.prefill(prompt[:-1], 0)
        want, want_st, served = dm.decode_sample_n(int(prompt[-1]), plen - 1, n_tokens, t, p, SEEDS[:16])
        assert served == 1
        toks, states, served, _, rows = qctx(dm, [prompt[:-1]], [0] * 16, [prompt[-1:]] * 16, [n_tokens] * 16, [(t, p)] * 16, SEEDS[:16], [], 16)
    assert served == 1 and rows == ceil8(plen - 1)
    assert states == want_st
    for b in range(16):
        assert np.array_equal(toks[b], want[b]), f"sample {b} differs from decode_sample_n"


# ---- 5. no dependence on history
def test_outputs_do_not_depend_on_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    tensors = mg.generate(spec, 29, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = alone_requests(spec.vocab_size, 14, [300, 129, 7], [9, 1, 40])
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        fresh = qctx(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], 4)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        toks = prompts_of(spec.vocab_size, [900], start=40)[0]
        dm.score_context(toks, [0, 0], [500, 300], [500, 300], [400, 200])
        other = prompts_of(spec.vocab_size, [700, 33, 2], start=50)
        qctx(dm, [other[0]], [0, 0, -1], other, [60, 5, 30], [(1.1, 0.0)] * 3, SEEDS[20:23], [], 2)
        dm.poison(0)
        dirty = qctx(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], 4)
    assert dirty[1:] == fresh[1:]
    assert all(np.array_equal(x, y) for x, y in zip(dirty[0], fresh[0]))


# ---- 6. the last step's stages against float64
STAGES = {  # (spec, kvbits, contexts, ctx_of, own lengths, max_new, max_rows): later requests shorter, so the last step holds several rows
    "llama3-8b fp8 kv_mul4": (L8B, 16, [300, 129], [0, 0, -1, 1, 0, 1, 0], [9, 1, 130, 2, 40, 1, 17], [29, 26, 23, 20, 17, 14, 11], 4),
    "llama3-8b fp8 kv_mul4 e5m2": (L8B, 8, [2100], [0, -1, 0, 0, 0], [300, 9, 1, 33, 2], [23, 20, 17, 14, 11], 3),
    "pf-tiny hd64 kv_mul2": (TINY1, 16, [256, 37], [0, 1, 0, -1, 0, 1], [1, 9, 250, 2, 64, 1], [26, 23, 20, 17, 14, 11], 4),
}


@pytest.mark.parametrize("case", sorted(STAGES))
def test_last_step_every_stage(case, capfd):
    spec, kvbits, ctx_lens, ctx_of, lens, max_new, max_rows = STAGES[case]
    tensors, w = make_model(spec, 4)
    with lib.DeviceModel(spec, tensors, seq_len=8192, kvbits=kvbits) as dm, capfd.disabled():
        check_last_step(dm, w, kvbits, ctx_lens, ctx_of, lens, max_new, max_rows, case)


def check_last_step(dm, w, kvbits, ctx_lens, ctx_of, lens, max_new, max_rows, case):
    """The queue over contexts and own prompts of these lengths, then the last step's stages against float64."""
    spec, nreq, seq_len = w.spec, len(lens), dm.seq_len
    contexts = prompts_of(spec.vocab_size, ctx_lens, start=61)
    prompts = prompts_of(spec.vocab_size, lens, start=3)
    key, clen = layout(contexts, ctx_of, prompts)
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    toks, _, served, steps, _ = qctx(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], max_rows)
    sched, place, _, _, _, _ = simulate(key, clen, lens, max_new, max_new, max_rows, seq_len)
    rows = sched[-1]
    n = len(rows)
    X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
    Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:n]
    A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:n]
    H = dm.read_state("pf_hb").reshape(-1, spec.hidden_dim)[:n]
    keys, values = layer_cache(dm, spec)
    assert served == 1 and steps == len(sched)
    assert n >= 2 and len({j for _, j in rows}) >= 2, f"{case}: the last step's rows {rows} are not at different own steps"
    assert any(clen[i] >= CHUNK for i, _ in rows), f"{case}: no row of the last step has a shared chunk"
    label = f"sample_queue_context {case} kv{kvbits}"
    inputs = np.asarray([toks[i][j - 1] if j > 0 else prompts[i][-1] for i, j in rows])
    pos = np.asarray([place[i][1] + j for i, j in rows])
    X0 = w.mat("model.embed.weight")[inputs].astype(np.float64)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, 0, X0, pos)
    report(label, "Q", "k_vf_gemm QKV", Q, q_ref, np.abs(q_ref).max(), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "vf_q", pf_tol(spec.dim))
    slots = np.asarray([place[i][2] + j for i, j in rows])
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        got = dev[:, slots].transpose(1, 0, 2).reshape(n, -1)
        check_entries(label, name, "k_vf_gemm QKV_SLOTS", got, ref, kvbits, lambda i: f"row {i[0]} kv head {i[1] // hd} dim {i[1] % hd}", "vf_kv", pf_tol(spec.dim))
    a_ref, vmax = [], []
    for r, (i, j) in enumerate(rows):
        s, L, t, c, nc = place[i]
        idx = np.concatenate([c + np.arange(nc), s + np.arange(L - nc), t + np.arange(j + 1)])
        K, V = keys[:, idx], values[:, idx]
        a_ref.append(sr.attention(spec, Q[r], K, V, L + j + 1))
        vmax.append(np.repeat(np.abs(V).max((1, 2)), kv_mul * hd))
    report(label, "A", "k_sn_attn GROUPS", A, np.stack(a_ref), np.stack(vmax), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")
    x1 = sr.wo(w, 0, X0, A)
    h_ref = sr.ffn_up(w, 0, sr.ffn_input(w, 0, x1, xn))
    report(label, "H", "k_vf_gemm WO+UP", H, h_ref, np.abs(h_ref).max(), lambda i: f"row {i[0]} hidden row {i[1]}", "vf_hb", pf_tol(max(spec.dim, spec.q_dim)))
    x_ref = sr.ffn_down(w, 0, x1, H)
    report(label, "X", "k_vf_gemm DOWN", X, x_ref, np.abs(x_ref).max(), lambda i: f"row {i[0]} row {i[1]}", "vf_x", pf_tol(spec.hidden_dim))


# ---- 7. fallback and bad arguments
@pytest.mark.parametrize("name,seq_len,ctx_lens,lens,max_new", [("tiny-moe", None, [20, 5], [6, 1, 12], [9, 0, 5]),
                                                                ("pf-tiny", 80, [30, 2], [21, 50, 11], [8, 20, 3])])
def test_fallback_is_prefill_and_forward_sample_over_concatenated_prompts(name, seq_len, ctx_lens, lens, max_new):
    """A MoE model, and a served shape with a request whose ceil8(ctx_len) + ceil8(len - 1) + max_new (8 + 56 + 20) passes
    seq_len: forward_prefill_cuda + forward_sample per request over ctx ++ prompt, cut at the stop, steps and prompt_rows 0."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    contexts = prompts_of(spec.vocab_size, ctx_lens, start=8)
    ctx_of = [0, 1, 0]
    prompts = prompts_of(spec.vocab_size, lens, start=1)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    cat = [concat(contexts, c, p) for c, p in zip(ctx_of, prompts)]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        stream = []
        dm.prefill(cat[0][:-1], 0)
        tok, s = int(cat[0][-1]), SEEDS[0]
        for k in range(max_new[0]):
            tok, s = dm.forward_sample(tok, len(cat[0]) - 1 + k, *sets[0], s)
            stream.append(tok)
        stop = [stream[2]]
        want, want_st = [], []
        for p, m, (t, mp), s in zip(cat, max_new, sets, SEEDS):
            dm.prefill(p[:-1], 0)
            tok, out = int(p[-1]), []
            while len(out) < m:
                tok, s = dm.forward_sample(tok, len(p) - 1 + len(out), t, mp, s)
                out.append(tok)
                if tok in stop:
                    break
            want.append(out), want_st.append(s)
        toks, states, served, steps, rows = qctx(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], stop, 16)
    assert (served, steps, rows) == (0, 0, 0)
    assert [x.tolist() for x in toks] == want and states == want_st
    assert len(want[0]) <= 3


def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(contexts=[np.asarray([4, 5], np.int32)], ctx_of=[0], prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4,
                  rng_states=[1])
        bad = [dict(contexts=None), dict(ctx_of=None), dict(ctx_of=[1]), dict(ctx_of=[-2]), dict(ctx_of=[0, 0]), dict(ctx_of=[0.0]),
               dict(contexts=[[-1]]), dict(contexts=[[spec.vocab_size]]), dict(contexts=[[0.5]]), dict(contexts=[[[1]]]),
               dict(prompts=None), dict(rng_states=5), dict(rng_states=[1, 2]), dict(max_new=[-1]), dict(max_rows=0), dict(max_rows=17),
               dict(stop=[spec.vocab_size]), dict(prompts=[np.zeros(0, np.int32)]), dict(prompts=[[3, spec.vocab_size]])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue_context(**{**ok, **b})
        toks, states, served, steps, rows = dm.decode_sample_queue_context(**{**ok, "max_new": [0]})  # never admitted: the context is not placed
        assert len(toks[0]) == 0 and states == [1] and (served, steps, rows) == (1, 0, 0)
        toks, states, served, steps, rows = dm.decode_sample_queue_context([], [], [], [], [], [], [], 4, [])
        assert toks == [] and states == [] and (served, steps, rows) == (1, 0, 0)
