"""calm_b200_decode_sample_queue_logprobs: the queue's tokens with each generated token's log-probability and the k most
likely tokens at its step, from the step's own classifier (a top-k epilogue in k_vf_gemm and the scoring merge).

1. Tokens, out_len, final states, steps and prompt_rows are decode_sample_queue(_context)'s bit for bit at k 0 / 1 / 5 / 20,
   across fp8 / gf4 / fp16, head_dim 128 with bias, Llama-3-8B widths, both caches, max_rows 1 / 3 / 16 (max_rows 1 runs
   all-greedy and all-sampled steps), stops at step 0, mid-stream and on the last step, and contexts shared by rows
   admitted in different rounds.  Every output keeps the invariants: logprobs <= 0, top_logprobs non-increasing, the
   emitted token's top-k entry equal to its logprobs entry bit for bit, a greedy row's first id its token, and logprobs
   the same bits at every k.
2. Exact values: a request run with max_new = j + 1 gives the same first j + 1 outputs, and its last step's logit row
   (PF_LOGITS) in float64 gives its log-probability and top-k: ids exactly (they are chosen from those fp32 logits), values
   within the fp32 merge's bound.  A partial last vocabulary tile, and 128256 tokens (1002 tiles per merge).
3. Slots past out_len keep what the caller put there.
4. Each request's outputs are the same bits alone, among 40 requests, under max_rows 1 / 4 / 16, at a tight seq_len, and
   after other calls and poisoning.
5. Every step against calm_b200_score_context_topk over ctx ++ prompt ++ generated tokens.
6. The fallback (MoE, and a request past seq_len) returns 0 with the queue fallback's tokens and the float64 log-softmax
   of the device logits of a forward_sample replay.  7. Bad arguments raise ValueError (the binding always passes its own
   output arrays, so the C call's NULL-output aborts are not reachable from Python).

Mutations the tests are designed to catch (by the test named): a greedy row's target taken from tile 0 (1: a greedy row's
logprobs differs from its top_logprobs[0]); the tile lists written at a wrong row stride (2: ids differ from the logit
row's); the merge skipped in an all-sampled step (2 and 4: stale log-probabilities); the output slot off by one (2, 3)."""
import ctypes as C
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import TOL_SIGMA  # noqa: E402
from test_decode_sample_queue_context_gpu import concat, qctx  # noqa: E402
from test_decode_sample_queue_gpu import HD128, SEEDS, SETTINGS, ceil8, greedy_setting, prompts_of, queue  # noqa: E402
from test_score_gpu import MERGE_C  # noqa: E402
from test_score_topk_gpu import host_topk  # noqa: E402
from test_stages_gpu import L8B  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

KS = (0, 1, 5, 20)


def qlp(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows, k):
    return dm.decode_sample_queue_logprobs(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds, k)


def plain(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows):
    """The call the log-probability call must match: decode_sample_queue without contexts, else the context call."""
    if contexts is None:  # (decode_sample_queue does not return its prompt rows)
        return queue(dm, prompts, max_new, sets, seeds, stop, max_rows) + (None,)
    return qctx(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def check_invariants(toks, lps, ids, tlps, sets, k, vocab, label):
    for i, (t, lp) in enumerate(zip(toks, lps)):
        assert lp.shape == t.shape and np.isfinite(lp).all(), f"{label}: request {i} logprobs"
        assert (lp <= 0).all(), f"{label}: request {i} has a positive log-probability"
        if not k:
            continue
        d, tl = ids[i], tlps[i]
        assert d.shape == tl.shape == (len(t), k)
        assert ((d >= 0) & (d < vocab)).all() and np.isfinite(tl).all() and (tl <= 0).all(), f"{label}: request {i} top-k"
        assert (np.diff(tl, axis=1) <= 0).all(), f"{label}: request {i} top_logprobs increase"
        s = np.sort(d, axis=1)
        assert (s[:, 1:] != s[:, :-1]).all(), f"{label}: request {i} repeats an id"
        hit = d == t[:, None]
        rows = np.nonzero(hit.any(1))[0]
        assert same_bits(tl[hit], lp[rows]), f"{label}: request {i}: the emitted token's top_logprobs is not its logprobs"
        if greedy_setting(*sets[i]):
            assert np.array_equal(d[:, 0], t), f"{label}: greedy request {i}: top_ids[0] is not its token"
            assert same_bits(tl[:, 0], lp), f"{label}: greedy request {i}: logprobs differ from top_logprobs[0]"


# ---- 1. the same tokens at every k, and the invariants
CASES = {  # (spec, kvbits, max_rows, nreq, context lengths (None: no contexts), own lengths, seq_len)
    "pf-tiny fp8 r16 contexts": (mg.SPECS["pf-tiny"], 16, 16, 24, [300, 129, 7], [1, 9, 40, 2], 4096),
    "pf-tiny gf4 e5m2 r3 contexts": (replace(mg.SPECS["pf-tiny"], dtype="gf4"), 8, 3, 14, [200, 8], [9, 1, 30], 4096),
    "pf-tiny fp16 r1": (replace(TINY1, dtype="fp16"), 16, 1, 8, None, [9, 129, 1, 2], 2048),
    "pf-tiny-hd128 bias e5m2 r16": (HD128, 8, 16, 16, [129], [2, 40, 1, 9], 4096),
    "llama3-8b widths r16 contexts": (L8B, 16, 16, 16, [300], [1, 30, 9, 2], 4096),
}


def case_requests(vocab, nreq, ctx_lens, own_lens):
    contexts = prompts_of(vocab, ctx_lens, start=101) if ctx_lens else None
    ctx_of = [-1 if i % 5 == 3 else i % len(contexts) for i in range(nreq)] if ctx_lens else None
    prompts = prompts_of(vocab, [own_lens[i % len(own_lens)] for i in range(nreq)], start=7)
    max_new = [[0, 1, 7, 24][(3 * i + 1) % 4] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    return contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq]


@pytest.mark.parametrize("case", sorted(CASES))
def test_same_tokens_at_every_k(case):
    spec, kvbits, max_rows, nreq, ctx_lens, own_lens, seq_len = CASES[case]
    tensors = mg.generate(spec, 17, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = case_requests(spec.vocab_size, nreq, ctx_lens, own_lens)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        full = plain(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], max_rows)
        long = [i for i in range(nreq) if max_new[i] == 24]
        stop = [int(full[0][long[0]][0]), int(full[0][long[1]][12]), int(full[0][long[-1]][23])]
        for stops in ([], stop):
            want = plain(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stops, max_rows)
            assert want[2] == 1
            if stops:
                assert len(want[0][long[0]]) == 1, f"{case}: the stop at step 0 did not fire"
            by_k = {}
            for k in KS:
                got = qlp(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stops, max_rows, k)
                label = f"{case} stop {stops} k {k}"
                assert got[1:4] == tuple(want[1:4]), f"{label}: states / served / steps differ"
                assert want[4] is None or got[4] == want[4], f"{label}: prompt_rows differ"
                assert all(np.array_equal(x, y) for x, y in zip(got[0], want[0])), f"{label}: tokens differ"
                check_invariants(got[0], got[5], got[6], got[7], sets, k, spec.vocab_size, label)
                by_k[k] = got
            for k in KS[1:]:
                assert all(same_bits(a, b) for a, b in zip(by_k[k][5], by_k[0][5])), f"{case} stop {stops}: logprobs at k {k} differ from k 0"
                assert all(np.array_equal(a, b[:, :k]) for a, b in zip(by_k[k][6], by_k[20][6])), f"{case}: top ids at k {k} are not a prefix of k 20's"
                assert all(same_bits(a, np.ascontiguousarray(b[:, :k])) for a, b in zip(by_k[k][7], by_k[20][7]))


# ---- 2. exact values against the step's own logit row
EXACT = {  # (spec, prompt lengths (greedy, sampled), steps j checked)
    "pf-tiny vocab 1000 (partial last tile)": (replace(TINY1, vocab_size=1000), [37, 200], [0, 3, 17]),
    "llama3-8b 1 layer vocab 128256": (replace(mg.SPECS["llama3-8b-fp8"], n_layers=1), [129, 9], [0, 5]),
}


def merge_tol(want, lse):
    """The fp32 (M, S) merge and the final subtraction against float64: test_score_gpu's merge bound plus a rounding of
    the result."""
    return MERGE_C * np.maximum(1.0, np.abs(lse)) + 2e-7 * np.abs(want)


@pytest.mark.parametrize("case", sorted(EXACT))
def test_exact_values_from_the_steps_logits(case):
    spec, lens, js = EXACT[case]
    k = 20
    tensors = mg.generate(spec, 5, device="cuda")
    prompts = prompts_of(spec.vocab_size, lens, start=3)
    sets = [(0.0, 0.1), (1.0, 0.05)]  # row 0 greedy, row 1 sampled: the step samples, so PF_LOGITS holds both rows
    seeds = SEEDS[:2]
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        jmax = max(js)
        ref = qlp(dm, None, None, prompts, [jmax + 1] * 2, sets, seeds, [], 2, k)
        for j in js:
            got = qlp(dm, None, None, prompts, [j + 1] * 2, sets, seeds, [], 2, k)
            rows = dm.read_state("pf_logits").reshape(-1, spec.vocab_size)
            assert got[2] == 1 and rows.shape[0] == 2
            for b in range(2):
                label = f"{case} j {j} row {b}"
                assert np.array_equal(got[0][b], ref[0][b][:j + 1]), f"{label}: tokens are not the longer call's"
                assert same_bits(got[5][b], ref[5][b][:j + 1]) and same_bits(got[7][b], ref[7][b][:j + 1]), f"{label}: not the longer call's bits"
                row = rows[b].astype(np.float64)
                lse = np.log(np.exp(row - row.max()).sum()) + row.max()
                tok = int(got[0][b][j])
                if b == 0:
                    assert tok == int(np.argmax(rows[b])), f"{label}: the greedy token is not the row's argmax"
                want = row[tok] - lse
                err = abs(float(got[5][b][j]) - want)
                assert err <= merge_tol(want, lse), f"{label}: logprob {got[5][b][j]!r} vs float64 {want!r}"
                ids = host_topk(rows[b][None], k)[0]
                assert np.array_equal(got[6][b][j], ids), f"{label}: top ids {got[6][b][j].tolist()} vs the row's {ids.tolist()}"
                wt = row[ids] - lse
                assert (np.abs(got[7][b][j].astype(np.float64) - wt) <= merge_tol(wt, lse)).all(), f"{label}: top_logprobs"


# ---- 3. slots past out_len are left untouched
def test_slots_past_out_len_are_untouched():
    spec = mg.SPECS["pf-tiny"]
    k = 5
    with lib.DeviceModel(spec, mg.generate(spec, 3, device="cuda"), seq_len=1024) as dm:
        prompts = prompts_of(spec.vocab_size, [9, 30, 2], start=4)
        max_new, sets, seeds = [12, 12, 6], [SETTINGS[0], SETTINGS[1], SETTINGS[2]], SEEDS[:3]
        free = dm.decode_sample_queue(prompts, max_new, [t for t, _ in sets], [p for _, p in sets], [], 3, seeds)[0]
        stop = [int(free[0][4])]
        toks = np.ascontiguousarray(np.concatenate(prompts), np.int32)
        len_ = np.asarray([len(p) for p in prompts], np.int32)
        off = np.asarray(np.concatenate([[0], np.cumsum(len_)[:-1]]), np.int32)
        total = sum(max_new)
        out = np.full(total, -3, np.int32)
        out_len = np.zeros(3, np.int32)
        lp = np.full(total, -777.25, np.float32)
        ids = np.full((total, k), -9, np.int32)
        tlp = np.full((total, k), -888.5, np.float32)
        ip, fp = C.POINTER(C.c_int), C.POINTER(C.c_float)
        mn, st = np.asarray(max_new, np.int32), np.asarray(stop, np.int32)
        tt, pp = np.asarray([t for t, _ in sets], np.float32), np.asarray([p for _, p in sets], np.float32)
        rng = (C.c_ulonglong * 3)(*seeds)
        steps, prows = C.c_int(-1), C.c_int(-1)
        served = dm.lib.calm_b200_decode_sample_queue_logprobs(C.byref(dm.transformer), toks.ctypes.data_as(ip), len(toks), None, None, off.ctypes.data_as(ip),
                                                               len_.ctypes.data_as(ip), 3, mn.ctypes.data_as(ip), tt.ctypes.data_as(fp), pp.ctypes.data_as(fp),
                                                               st.ctypes.data_as(ip), 1, 3, rng, out.ctypes.data_as(ip), out_len.ctypes.data_as(ip),
                                                               C.byref(steps), C.byref(prows), k, lp.ctypes.data_as(fp), ids.ctypes.data_as(ip),
                                                               tlp.ctypes.data_as(fp))
    assert served == 1 and out_len[0] <= 5
    O = np.concatenate([[0], np.cumsum(max_new)])
    for i in range(3):
        n = int(out_len[i])
        assert (out[O[i]:O[i] + n] >= 0).all() and (lp[O[i]:O[i] + n] <= 0).all() and (ids[O[i]:O[i] + n] >= 0).all()
        assert (out[O[i] + n:O[i + 1]] == -3).all(), f"request {i}: a token slot past out_len was written"
        assert (lp[O[i] + n:O[i + 1]] == np.float32(-777.25)).all(), f"request {i}: a logprobs slot past out_len was written"
        assert (ids[O[i] + n:O[i + 1]] == -9).all() and (tlp[O[i] + n:O[i + 1]] == np.float32(-888.5)).all(), f"request {i}: a top-k slot past out_len"


# ---- 4. independence of the other requests, the schedule, the cache size and history
def test_outputs_do_not_depend_on_schedule_or_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    tensors = mg.generate(spec, 23, device="cuda")
    k = 5
    contexts = prompts_of(spec.vocab_size, [300, 129], start=61)
    nreq = 40
    ctx_of = [[-1, 0, 1, 0][i % 4] for i in range(nreq)]
    lens = [[9, 1, 40, 2, 17][i % 5] for i in range(nreq)]
    prompts = prompts_of(spec.vocab_size, lens, start=3)
    max_new = [[13, 1, 25, 7, 0][(3 * i + 1) % 5] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    clen = [len(contexts[c]) if c >= 0 else 0 for c in ctx_of]
    tight = max(ceil8(c) + ceil8(n - 1) + m for c, n, m in zip(clen, lens, max_new)) + 16
    runs = {}
    for seq_len in (4096, tight):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            for max_rows in ((1, 4, 16) if seq_len == 4096 else (16,)):
                runs[(seq_len, max_rows)] = qlp(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, k)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        alone = {i: qlp(dm, [contexts[ctx_of[i]]] if ctx_of[i] >= 0 else None, [0] if ctx_of[i] >= 0 else None, [prompts[i]], [max_new[i]], [sets[i]],
                        [SEEDS[i]], [], 16, k) for i in (0, 1, 2, 5, 6, 8)}
        other = prompts_of(spec.vocab_size, [700, 33, 2], start=50)
        qlp(dm, [other[0]], [0, 0, -1], other, [60, 5, 30], [(1.1, 0.0)] * 3, SEEDS[20:23], [], 2, 20)
        dm.score_context_topk(np.concatenate(other), [0], [400], [700], [33], 3)
        dm.poison(0)
        runs["dirty"] = qlp(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], 16, k)
    ref = runs[(4096, 16)]
    assert all(len(t) == m for t, m in zip(ref[0], max_new))
    for key, got in runs.items():
        for i in range(nreq):
            assert np.array_equal(got[0][i], ref[0][i]), f"{key}: request {i} tokens"
            for f in (5, 6, 7):
                assert same_bits(got[f][i], ref[f][i]), f"{key}: request {i} output {f} differs"
    for i, got in alone.items():
        assert np.array_equal(got[0][0], ref[0][i])
        for f in (5, 6, 7):
            assert same_bits(got[f][0], ref[f][i]), f"request {i} alone: output {f} differs from the 40-request run"


# ---- 5. against calm_b200_score_context_topk over ctx ++ prompt ++ generated tokens
def test_matches_scoring_the_generated_tokens():
    spec = mg.SPECS["pf-tiny"]
    k = 5
    contexts = prompts_of(spec.vocab_size, [200, 37], start=9)
    ctx_of = [0, 1, -1, 0, 0, 1]
    prompts = prompts_of(spec.vocab_size, [9, 1, 40, 2, 17, 5], start=2)
    max_new = [25, 14, 9, 20, 3, 11]  # the longest request samples: the last step's PF_LOGITS gives the logits' spread
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(prompts))]
    with lib.DeviceModel(spec, mg.generate(spec, 8, device="cuda"), seq_len=4096) as dm:
        toks, _, served, _, _, lps, ids, tlps = qlp(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:6], [], 4, k)
        sigma = float(dm.read_state("pf_logits").reshape(-1, spec.vocab_size).std(1).min())
        assert served == 1
        for i in range(len(prompts)):
            seq = np.concatenate([prompts[i], toks[i]]).astype(np.int32)
            c = contexts[ctx_of[i]] if ctx_of[i] >= 0 else np.zeros(0, np.int32)
            tokens = np.concatenate([c, seq]).astype(np.int32)
            slp, sids, stlp, sserved = dm.score_context_topk(tokens, [0], [len(c)], [len(c)], [len(seq)], k)
            assert sserved == 1
            at = len(c) + len(prompts[i]) - 1 + np.arange(len(toks[i]))  # the slot that scores generated token j
            tol = 2 * 2 * TOL_SIGMA * sigma  # a log-probability moves by at most twice its logits' error
            err = np.abs(lps[i] - slp[at])
            assert (err <= tol).all(), f"request {i}: step {int(np.argmax(err))} logprob {lps[i][np.argmax(err)]} vs scoring {slp[at][np.argmax(err)]}"
            assert (np.abs(tlps[i] - stlp[at]) <= tol).all(), f"request {i}: top_logprobs (rank by rank) differ from scoring's"
            agree = (ids[i] == sids[at]).mean()
            assert agree >= 0.9, f"request {i}: only {agree:.0%} of the top ids agree with scoring's"


# ---- 6. the fallback
@pytest.mark.parametrize("name,seq_len,lens,max_new", [("tiny-moe", None, [6, 1, 12], [9, 0, 5]), ("pf-tiny", 64, [21, 50, 11], [8, 20, 3])])
def test_fallback_is_the_log_softmax_of_the_device_logits(name, seq_len, lens, max_new):
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    k = 5
    contexts = prompts_of(spec.vocab_size, [4], start=8)
    ctx_of = [0, -1, 0]
    prompts = prompts_of(spec.vocab_size, lens, start=1)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    cat = [concat(contexts, c, p) for c, p in zip(ctx_of, prompts)]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        want = qctx(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16)
        got = qlp(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k)
        assert got[2] == 0 and got[1:5] == tuple(want[1:5])
        assert all(np.array_equal(x, y) for x, y in zip(got[0], want[0]))
        for i, (p, m, (t, mp), s) in enumerate(zip(cat, max_new, sets, SEEDS)):
            dm.prefill(p[:-1], 0)
            tok = int(p[-1])
            for j in range(m):
                tok, s = dm.forward_sample(tok, len(p) - 1 + j, t, mp, s)
                assert tok == got[0][i][j]
                row = dm.device_logits().astype(np.float64)
                lse = np.log(np.exp(row - row.max()).sum()) + row.max()
                want_lp = row[tok] - lse
                assert abs(float(got[5][i][j]) - want_lp) <= 1e-6 * max(1.0, abs(want_lp)), f"{name}: request {i} step {j}"
                top = host_topk(row[None], k)[0]
                assert np.array_equal(got[6][i][j], top), f"{name}: request {i} step {j} top ids"
                assert np.allclose(got[7][i][j], row[top] - lse, rtol=1e-6, atol=1e-6)
    check_invariants(got[0], got[5], got[6], got[7], sets, k, spec.vocab_size, name)


# ---- 7. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(contexts=[np.asarray([4, 5], np.int32)], ctx_of=[0], prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4,
                  rng_states=[1], k=5)
        bad = [dict(k=-1), dict(k=lib.TOPK_MAX + 1), dict(k=2.0), dict(k=None), dict(k=True), dict(contexts=None), dict(ctx_of=None), dict(ctx_of=[1]),
               dict(contexts=[[spec.vocab_size]]), dict(prompts=None), dict(rng_states=5), dict(rng_states=[1, 2]), dict(max_new=[-1]), dict(max_rows=0),
               dict(max_rows=17), dict(stop=[spec.vocab_size]), dict(prompts=[np.zeros(0, np.int32)]), dict(prompts=[[3, spec.vocab_size]])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue_logprobs(**{**ok, **b})
        got = dm.decode_sample_queue_logprobs(**{**ok, "max_new": [0]})
        assert len(got[0][0]) == 0 and got[1] == [1] and got[2:5] == (1, 0, 0) and len(got[5][0]) == 0 and got[6][0].shape == (0, 5)
        got = dm.decode_sample_queue_logprobs(None, None, [], [], [], [], [], 4, [], 0)
        assert got[:5] == ([], [], 1, 0, 0) and got[5] == [] and got[6] is None and got[7] is None
    tiny = replace(spec, vocab_size=12)
    with lib.DeviceModel(tiny, mg.generate(tiny, 1)) as dm:
        with pytest.raises(ValueError):
            dm.decode_sample_queue_logprobs(None, None, [[1, 2]], [3], [1.0], [0.1], [], 2, [1], 13)
        got = dm.decode_sample_queue_logprobs(None, None, [[1, 2]], [3], [1.0], [0.1], [], 2, [1], 12)
        assert got[6][0].shape == (3, 12) and sorted(got[6][0][0].tolist()) == list(range(12))
