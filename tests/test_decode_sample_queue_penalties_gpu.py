"""calm_b200_decode_sample_queue_penalties: the queue with per-request logit bias and presence, frequency and repetition
penalties, applied to each vocabulary tile's logits in k_vf_gemm's classifier epilogue from per-request lanes.

1. Neutral requests (all settings NULL, or explicit 0 / 0 / 1 and empty lists) give tokens, states, steps, prompt_rows,
   logprobs and top-k bit for bit equal to decode_sample_queue_logprobs at k 0 / 5 (and the context call's tuple with
   no k), with equal calm_b200_launch_count deltas, across fp8 / gf4 / fp16, head_dim 128 with bias, Llama-3-8B widths,
   both caches and max_rows 1 / 3 / 16; neutral requests that share steps with non-neutral ones keep their outputs.
2. Step 0 exactly: a non-neutral request's PF_LOGITS row is process() of the plain call's row, bit for bit (bias and the
   repetition penalty over ctx ++ prompt); its token and state are calm_b200_sample_logits of that row, and a greedy
   request's token is its argmax.
3. Bookkeeping, by values that dwarf the logits, with 40 requests under max_rows 1 / 3 / 16 (admissions in many rounds,
   lanes reused out of order): bias +1e4 on a set S with presence 2e4 emits a permutation of S and then never S again;
   presence or frequency 1e4 alone never repeats a token; bias -1e4 on the plain step-0 token gives the plain top_ids[1].
4. Every step: a request run with max_new = j + 1 gives the same first j + 1 outputs; its last PF_LOGITS row gives its
   log-probability and top-k (ids exactly, values within the merge's bound), and lies within the logits' bound of
   process() over the raw row of ctx ++ prompt ++ its first j tokens computed by the prompt pass; the greedy token is
   that row's argmax wherever the margin is clear.
5. Each request gives the same bits alone, among 40 requests, under max_rows 1 / 4 / 16, at a tight seq_len, with
   contexts shared by rows admitted in different rounds, and after another call plus poisoning.
6. The fallback (MoE, a request past seq_len) returns 0 and equals a host replay: device logits, process(), then
   calm_b200_sample_logits.  7. Bad arguments raise ValueError.

Mutations the tests are designed to catch (by the test named): the lane indexed by row instead of by request (3 and 5:
rows compact as requests retire, so a row reads another request's counts); the count updated before the step's own
logits are read (2: step 0 would see its own token); prompt tokens left out of seen (2: the repetition penalty over the
prompt); a lane not cleared on admission (3 and 5: a reused lane keeps its previous occupant's counts and bias); neutral
rows processed (1)."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import TOL_SIGMA  # noqa: E402
from test_decode_sample_queue_context_gpu import concat  # noqa: E402
from test_decode_sample_queue_gpu import HD128, SEEDS, SETTINGS, ceil8, greedy_setting, prompts_of  # noqa: E402
from test_decode_sample_queue_logprobs_gpu import merge_tol, same_bits  # noqa: E402
from test_score_topk_gpu import host_topk  # noqa: E402
from test_stages_gpu import L8B  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu


def process(l, seen, c, p, f, r, b):
    """The header's expression in float32: l the raw logits, seen a bool row, c the counts, b the bias row."""
    l, c, b = np.asarray(l, np.float32), np.asarray(c), np.asarray(b, np.float32)
    p, f, r = np.float32(p), np.float32(f), np.float32(r)
    with np.errstate(all="ignore"):
        l1 = np.where(seen & (r != 1), np.where(l > 0, l / r, l * r), l).astype(np.float32)
        a = ((b - f * c.astype(np.float32)).astype(np.float32) - np.where(c > 0, p, np.float32(0))).astype(np.float32)
        return np.where(a == 0, l1, (l1 + a).astype(np.float32)).astype(np.float32)


def host_state(vocab, ctx_prompt, generated, bias):
    """(seen, counts, bias row) of a request after `generated`."""
    c = np.bincount(np.asarray(generated, np.int64), minlength=vocab)[:vocab]
    seen = np.zeros(vocab, bool)
    seen[np.asarray(ctx_prompt, np.int64)] = True
    b = np.zeros(vocab, np.float32)
    for t, v in (bias or {}).items():
        b[t] = v
    return seen | (c > 0), c, b


def qpen(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows, k=None, **pen):
    return dm.decode_sample_queue_penalties(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds, k=k,
                                            **pen)


def qlp(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows, k):
    return dm.decode_sample_queue_logprobs(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds, k)


def launches():
    return lib.load().calm_b200_launch_count()


def assert_same(got, want, label, idx=None):
    """Tuples of the _logprobs (or context) call: every field, bit for bit, for requests idx (default all)."""
    idx = range(len(want[0])) if idx is None else idx
    for i in idx:
        assert np.array_equal(got[0][i], want[0][i]), f"{label}: request {i} tokens"
        assert got[1][i] == want[1][i], f"{label}: request {i} state"
        for f in range(5, len(want)):
            if want[f] is not None:
                assert same_bits(got[f][i], want[f][i]), f"{label}: request {i} output {f}"


def mixed_pen(vocab, nreq, which):
    """Settings for the requests in `which` (the others neutral): bias on a few ids, all three penalties."""
    pres, freq, rep = [0.0] * nreq, [0.0] * nreq, [1.0] * nreq
    bias = [None] * nreq
    for i in which:
        pres[i], freq[i], rep[i] = 0.5, 0.25 * (i % 3), [1.1, 1.3, 0.9][i % 3]
        bias[i] = {(7 * i + 3) % vocab: 2.5, (11 * i + 1) % vocab: -3.0, (13 * i) % vocab: 0.0}
    return dict(presence=pres, frequency=freq, repetition=rep, logit_bias=bias)


# ---- 1. neutral requests are the plain call
CASES = {  # (spec, kvbits, max_rows, nreq, context lengths (None: no contexts), own lengths, seq_len)
    "pf-tiny fp8 r16 contexts": (mg.SPECS["pf-tiny"], 16, 16, 20, [300, 7], [1, 9, 40, 2], 4096),
    "pf-tiny gf4 e5m2 r3 contexts": (replace(mg.SPECS["pf-tiny"], dtype="gf4"), 8, 3, 10, [200], [9, 1, 30], 4096),
    "pf-tiny fp16 r1": (replace(TINY1, dtype="fp16"), 16, 1, 6, None, [9, 129, 1], 2048),
    "pf-tiny-hd128 bias e5m2 r16": (HD128, 8, 16, 12, [129], [2, 40, 1, 9], 4096),
    "llama3-8b widths r16 contexts": (L8B, 16, 16, 12, [300], [1, 30, 9, 2], 4096),
}


def case_requests(vocab, nreq, ctx_lens, own_lens):
    contexts = prompts_of(vocab, ctx_lens, start=101) if ctx_lens else None
    ctx_of = [-1 if i % 5 == 3 else i % len(contexts) for i in range(nreq)] if ctx_lens else None
    prompts = prompts_of(vocab, [own_lens[i % len(own_lens)] for i in range(nreq)], start=7)
    max_new = [[0, 1, 7, 16][(3 * i + 1) % 4] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    return contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq]


@pytest.mark.parametrize("case", sorted(CASES))
def test_neutral_requests_are_the_plain_call(case):
    spec, kvbits, max_rows, nreq, ctx_lens, own_lens, seq_len = CASES[case]
    tensors = mg.generate(spec, 17, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = case_requests(spec.vocab_size, nreq, ctx_lens, own_lens)
    neutral = dict(presence=[0.0] * nreq, frequency=[-0.0] * nreq, repetition=[1.0] * nreq, logit_bias=[{} if i % 2 else None for i in range(nreq)])
    args = (contexts, ctx_of, prompts, max_new, sets, seeds, [], max_rows)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        for k in (None, 0, 5):
            n0 = launches()
            want = qlp(dm, *args, 0 if k is None else k)
            n1 = launches()
            if k is None:  # the context call's tuple, and its launches (no log-probability work)
                want = want[:5]
                ctx = dm.decode_sample_queue_context(contexts or [], ctx_of or [-1] * nreq, prompts, max_new, [t for t, _ in sets], [p for _, p in sets],
                                                     [], max_rows, seeds)
                n1b = launches()
                assert ctx[1:5] == want[1:5]
                n0, n1 = n1, n1b
            assert want[2] == 1
            for label, pen in (("NULL", {}), ("neutral", neutral)):
                m0 = launches()
                got = qpen(dm, *args, k=k, **pen)
                m1 = launches()
                tag = f"{case} k {k} {label}"
                assert len(got) == len(want) and got[2:5] == want[2:5], f"{tag}: served / steps / prompt_rows"
                assert_same(got, want, tag)
                assert m1 - m0 == n1 - n0, f"{tag}: {m1 - m0} launches against {n1 - n0}"
        # neutral requests sharing steps with non-neutral ones keep their outputs
        want = qlp(dm, *args, 5)
        pen = mixed_pen(spec.vocab_size, nreq, [i for i in range(nreq) if i % 2 == 0])
        got = qpen(dm, *args, k=5, **pen)
        assert got[2:5] == want[2:5]
        assert_same(got, want, f"{case} mixed", [i for i in range(nreq) if i % 2])
        assert any(not np.array_equal(got[0][i], want[0][i]) for i in range(0, nreq, 2)), f"{case}: no processed request changed"


# ---- 2. step 0 exactly
@pytest.mark.parametrize("spec", [replace(TINY1, vocab_size=1000), HD128], ids=["pf-tiny vocab 1000", "pf-tiny-hd128 bias"])
def test_step0_is_process_of_the_plain_row(spec):
    tensors = mg.generate(spec, 5, device="cuda")
    V = spec.vocab_size
    contexts = prompts_of(V, [40], start=11)
    prompts = prompts_of(V, [9, 30], start=3)
    sets = [(0.0, 0.1), (1.0, 0.05)]  # row 0 greedy, row 1 sampled: the step samples, so PF_LOGITS holds both rows
    seeds = SEEDS[:2]
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        plain = qlp(dm, contexts, [0, -1], prompts, [1, 1], sets, seeds, [], 2, 5)
        raw = dm.read_state("pf_logits").reshape(-1, V).copy()
        # bias on the plain tokens, on prompt tokens and elsewhere; repetition over ctx ++ prompt
        bias = [{int(plain[0][b][0]): -2.0, int(prompts[b][0]): 1.5, int(prompts[b][-1]): 0.75, (17 * b + 5) % V: 3.0} for b in range(2)]
        pen = dict(presence=[0.5, -0.25], frequency=[0.75, 0.5], repetition=[1.3, 0.8], logit_bias=bias)
        got = qpen(dm, contexts, [0, -1], prompts, [1, 1], sets, seeds, [], 2, k=5, **pen)
        rows = dm.read_state("pf_logits").reshape(-1, V)
        assert got[2] == 1 and rows.shape[0] == 2
        for b in range(2):
            seq = concat(contexts, [0, -1][b], prompts[b])
            seen, c, bv = host_state(V, seq, [], bias[b])
            want = process(raw[b], seen, c, pen["presence"][b], pen["frequency"][b], pen["repetition"][b], bv)
            assert same_bits(rows[b], want), f"row {b}: PF_LOGITS is not process() of the plain row ({int((rows[b] != want).sum())} entries differ)"
            tok = int(got[0][b][0])
            if b == 0:
                assert tok == int(np.argmax(want)), "the greedy token is not the processed row's argmax"
            else:
                t, s = lib.sample_logits(want, *sets[b], seeds[b])
                assert (tok, got[1][b]) == (t, s), "the sampled token / state are not calm_b200_sample_logits of the processed row"
            assert int(host_topk(want[None], 5)[0][0]) == int(got[6][b][0][0])


# ---- 3. bookkeeping that does not depend on the logits
@pytest.mark.parametrize("max_rows", [1, 3, 16])
def test_bookkeeping_by_dominating_values(max_rows):
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 29, device="cuda")
    nreq = 40
    rng = np.random.default_rng(3)
    prompts = prompts_of(V, [[9, 1, 40, 2, 17][i % 5] for i in range(nreq)], start=5)
    sets = [(0.0, 0.1) if i % 2 else (1.0, 0.1) for i in range(nreq)]  # greedy, or min-p 0.1: no negligible token is drawn
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        plain = qlp(dm, None, None, prompts, [1] * nreq, sets, SEEDS[:nreq], [], 16, 2)
        kinds, S, max_new = [], [], []
        pen = dict(presence=[0.0] * nreq, frequency=[0.0] * nreq, repetition=[1.0] * nreq, logit_bias=[None] * nreq)
        for i in range(nreq):
            kind = ["set", "presence", "frequency", "ban", "neutral"][i % 5]
            kinds.append(kind)
            s = [int(x) for x in rng.choice(V, size=3 + i % 4, replace=False)]
            S.append(s)
            if kind == "set":
                pen["logit_bias"][i], pen["presence"][i] = {t: 1e4 for t in s}, 2e4
                max_new.append(len(s) + 4 + i % 3)
            elif kind == "presence":
                pen["presence"][i] = 1e4
                max_new.append(9 + i % 7)
            elif kind == "frequency":
                pen["frequency"][i] = 1e4
                max_new.append(5 + i % 11)
            elif kind == "ban":
                pen["logit_bias"][i] = {int(plain[0][i][0]): -1e4}
                max_new.append(2 + i % 4)
            else:
                max_new.append(3 + i % 6)
        got = qpen(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, **pen)
        ref = qlp(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, 0)
    assert got[2] == 1
    for i, kind in enumerate(kinds):
        t = [int(x) for x in got[0][i]]
        assert len(t) == max_new[i]
        if kind == "set":
            m = len(S[i])
            assert sorted(t[:m]) == sorted(S[i]), f"request {i}: the first {m} tokens {t[:m]} are not a permutation of {S[i]}"
            assert not set(t[m:]) & set(S[i]), f"request {i}: a token of S after the first {m}"
        elif kind in ("presence", "frequency"):
            assert len(set(t)) == len(t), f"request {i} ({kind}): a token repeats: {t}"
        elif kind == "ban" and greedy_setting(*sets[i]):
            assert t[0] == int(plain[6][i][0][1]), f"request {i}: the banned token's runner-up is not the token"
        elif kind == "ban":
            assert t[0] != int(plain[0][i][0]), f"request {i}: the banned token was drawn"
        else:
            assert np.array_equal(got[0][i], ref[0][i]) and got[1][i] == ref[1][i], f"neutral request {i} changed"


# ---- 4. every step
@pytest.mark.parametrize("spec", [replace(TINY1, vocab_size=1000), L8B], ids=["pf-tiny vocab 1000", "llama3-8b widths"])
def test_every_step_against_the_prompt_pass(spec):
    V = spec.vocab_size
    k = 8
    tensors = mg.generate(spec, 41, device="cuda")
    prompts = prompts_of(V, [37, 20], start=2)
    sets = [(0.0, 0.1), (1.0, 0.05)]
    seeds = SEEDS[:2]
    bias = [{int(prompts[0][3]): 1.0, 5: -0.5}, {int(prompts[1][0]): 0.5, 9: 2.0}]
    pen = dict(presence=[0.3, 0.6], frequency=[0.2, 0.4], repetition=[1.2, 1.1], logit_bias=bias)
    js = [0, 3, 11]
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        full = qpen(dm, None, None, prompts, [max(js) + 1] * 2, sets, seeds, [], 2, k=k, **pen)
        for j in js:
            got = qpen(dm, None, None, prompts, [j + 1] * 2, sets, seeds, [], 2, k=k, **pen)
            rows = dm.read_state("pf_logits").reshape(-1, V).copy()
            assert got[2] == 1 and rows.shape[0] == 2
            for b in range(2):
                label = f"j {j} row {b}"
                assert np.array_equal(got[0][b], full[0][b][:j + 1]) and all(same_bits(got[f][b], full[f][b][:j + 1]) for f in (5, 6, 7)), label
                row = rows[b].astype(np.float64)
                lse = np.log(np.exp(row - row.max()).sum()) + row.max()
                tok = int(got[0][b][j])
                want = row[tok] - lse
                assert abs(float(got[5][b][j]) - want) <= merge_tol(want, lse), f"{label}: logprob"
                ids = host_topk(rows[b][None], k)[0]
                assert np.array_equal(got[6][b][j], ids), f"{label}: top ids"
                assert (np.abs(got[7][b][j] - (row[ids] - lse)) <= merge_tol(row[ids] - lse, lse)).all(), f"{label}: top_logprobs"
                # the raw row of the same position from the prompt pass (teacher-forced by the device's tokens)
                seq = np.concatenate([prompts[b], got[0][b][:j]]).astype(np.int32)
                qlp(dm, None, None, [seq, seq], [1, 1], [sets[1]] * 2, seeds, [], 2, 0)
                raw = dm.read_state("pf_logits").reshape(-1, V)[0].copy()
                seen, c, bv = host_state(V, prompts[b], got[0][b][:j], bias[b])
                want_row = process(raw, seen, c, pen["presence"][b], pen["frequency"][b], pen["repetition"][b], bv)
                tol = 2 * TOL_SIGMA * float(raw.std()) * max(1.0, 1.0 / pen["repetition"][b])
                err = np.abs(rows[b] - want_row)
                assert err.max() <= tol, f"{label}: processed row off by {err.max():.3g} at {int(err.argmax())} (bound {tol:.3g})"
                if b == 0:
                    top2 = np.sort(want_row)[-2:]
                    if top2[1] - top2[0] > 2 * tol:
                        assert tok == int(np.argmax(want_row)), f"{label}: the greedy token is not the clear argmax"


# ---- 5. independence of the other requests, the schedule, the cache size and history
def test_outputs_do_not_depend_on_schedule_or_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 23, device="cuda")
    k = 3
    contexts = prompts_of(V, [300, 129], start=61)
    nreq = 40
    ctx_of = [[-1, 0, 1, 0][i % 4] for i in range(nreq)]
    lens = [[9, 1, 40, 2, 17][i % 5] for i in range(nreq)]
    prompts = prompts_of(V, lens, start=3)
    max_new = [[13, 1, 25, 7, 0][(3 * i + 1) % 5] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    pen = mixed_pen(V, nreq, [i for i in range(nreq) if i % 4 != 2])
    clen = [len(contexts[c]) if c >= 0 else 0 for c in ctx_of]
    tight = max(ceil8(c) + ceil8(n - 1) + m for c, n, m in zip(clen, lens, max_new)) + 16
    runs = {}
    for seq_len in (4096, tight):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            for max_rows in ((1, 4, 16) if seq_len == 4096 else (16,)):
                runs[(seq_len, max_rows)] = qpen(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, k=k, **pen)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        alone = {}
        for i in (0, 1, 3, 5, 6, 8, 10):
            one = {key: [v[i]] for key, v in pen.items()}
            alone[i] = qpen(dm, [contexts[ctx_of[i]]] if ctx_of[i] >= 0 else None, [0] if ctx_of[i] >= 0 else None, [prompts[i]], [max_new[i]], [sets[i]],
                            [SEEDS[i]], [], 16, k=k, **one)
        other = prompts_of(V, [700, 33, 2], start=50)
        qpen(dm, [other[0]], [0, 0, -1], other, [60, 5, 30], [(1.1, 0.0)] * 3, SEEDS[20:23], [], 2, k=20, presence=[1.0] * 3, repetition=[2.0] * 3,
             logit_bias=[{t: 5.0 for t in range(0, V, 7)}] * 3)
        dm.poison(0)
        runs["dirty"] = qpen(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], 16, k=k, **pen)
    ref = runs[(4096, 16)]
    assert ref[2] == 1 and all(len(t) == m for t, m in zip(ref[0], max_new))
    for key, got in runs.items():
        assert got[2] == 1
        assert_same(got, ref, str(key))
    for i, got in alone.items():
        assert_same(got, tuple([x[i]] if isinstance(x, list) else x for x in ref), f"request {i} alone", [0])


# ---- 6. the fallback
@pytest.mark.parametrize("name,seq_len,lens,max_new", [("tiny-moe", None, [6, 1, 12], [9, 0, 5]), ("pf-tiny", 64, [21, 50, 11], [8, 20, 3])])
def test_fallback_is_a_host_replay(name, seq_len, lens, max_new):
    spec = mg.SPECS[name]
    V = spec.vocab_size
    tensors = mg.generate(spec, 45)
    k = 3
    contexts = prompts_of(V, [4], start=8)
    ctx_of = [0, -1, 0]
    prompts = prompts_of(V, lens, start=1)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    cat = [concat(contexts, c, p) for c, p in zip(ctx_of, prompts)]
    bias = [{int(cat[0][-1]): 1.5, 3: -2.0}, None, {1: 0.5}]
    pen = dict(presence=[0.5, 0.0, 0.2], frequency=[0.3, 0.0, 0.0], repetition=[1.2, 1.0, 0.9], logit_bias=bias)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        plain = qlp(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k)
        got = qpen(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k=k, **pen)
        assert got[2] == 0 and plain[2] == 0
        assert_same(got, plain, f"{name} neutral request", [1])
        for i in (0, 2):
            p, s = cat[i], SEEDS[i]
            dm.prefill(p[:-1], 0)
            tok = int(p[-1])
            gen = []
            for j in range(max_new[i]):
                dm.forward_sample(tok, len(p) - 1 + j, 0.0, 0.0, 1)
                seen, c, bv = host_state(V, p, gen, bias[i])
                row = process(dm.device_logits(), seen, c, pen["presence"][i], pen["frequency"][i], pen["repetition"][i], bv)
                tok, s = lib.sample_logits(row, *sets[i], s)
                assert tok == got[0][i][j], f"{name}: request {i} step {j}"
                gen.append(tok)
                r64 = row.astype(np.float64)
                lse = np.log(np.exp(r64 - r64.max()).sum()) + r64.max()
                assert abs(float(got[5][i][j]) - (r64[tok] - lse)) <= 1e-6 * max(1.0, abs(r64[tok] - lse)), f"{name}: request {i} step {j} logprob"
                assert np.array_equal(got[6][i][j], host_topk(row[None], k)[0]), f"{name}: request {i} step {j} top ids"
            assert len(got[0][i]) == max_new[i] and (max_new[i] == 0 or greedy_setting(*sets[i]) or got[1][i] == s), f"{name}: request {i} state"


# ---- 7. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    V = spec.vocab_size
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(contexts=None, ctx_of=None, prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4, rng_states=[1],
                  presence=[0.5], frequency=[0.5], repetition=[1.1], logit_bias=[{3: 1.0}], k=2)
        bad = [dict(k=-1), dict(k=lib.TOPK_MAX + 1), dict(k=True), dict(contexts=[np.asarray([4], np.int32)]), dict(ctx_of=[0]),
               dict(presence=[np.nan]), dict(presence=[2e6]), dict(frequency=[-np.inf]), dict(frequency=[0.1, 0.2]), dict(repetition=[0.0]),
               dict(repetition=[5e-7]), dict(repetition=[2e6]), dict(repetition=[np.nan]), dict(logit_bias=[{V: 1.0}]), dict(logit_bias=[{-1: 1.0}]),
               dict(logit_bias=[{2: np.inf}]), dict(logit_bias=[{2: -2e6}]), dict(logit_bias=[{2.0: 1.0}]), dict(logit_bias=[[2, 1.0]]),
               dict(logit_bias=[{}, {}]), dict(max_new=[-1]), dict(max_rows=17), dict(prompts=[[3, V]])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue_penalties(**{**ok, **b})
        got = dm.decode_sample_queue_penalties(**{**ok, "max_new": [0]})
        assert len(got[0][0]) == 0 and got[1] == [1] and got[2:5] == (1, 0, 0)
        got = dm.decode_sample_queue_penalties(**{**ok, "k": None, "repetition": [1e6], "presence": [-1e6], "logit_bias": [{0: 1e6, V - 1: -1e6}]})
        assert len(got) == 5 and got[2] == 1 and len(got[0][0]) == 4
