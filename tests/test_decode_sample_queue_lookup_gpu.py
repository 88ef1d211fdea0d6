"""calm_b200_decode_sample_queue_lookup: the truncated queue with the rows a step leaves free holding prompt-lookup drafts
of each request's own tokens, verified in the same step and accepted where the row before gave the drafted token.

1. Same bits as decode_sample_queue_truncated at max_draft 1 / 7 / 15 over fp8 / gf4 / fp16, head_dim 64 / 128, kv_mul
   1 / 2 / 4 / 8, both caches, shared contexts whose rows cross SN_CHUNK boundaries, max_rows 1 / 3 / 16, stops, k 0 and
   5, truncation, constrained requests and non-neutral penalties; steps never more.  2. max_draft 0 launches exactly
   what _truncated launches and takes its steps.  3. Forced acceptance: requests on a cycling automaton (one allowed
   token per state) accept every draft; steps, drafted and accepted are the documented schedule's, replayed here, and
   each generator advances out_len times.  4. On greedy random-model workloads steps, drafted and accepted equal the
   replay over the plain call's tokens.  5. A draft that holds a stop token or a final-state token ends its request
   exactly there.  6. Slots past out_len are untouched.  7. The same bits after other calls and poison_state.
   8. The fallback is _truncated's, with zero counts.  9. Bad arguments raise ValueError.

Mutations the tests are built to catch: a draft row given the request's own coin instead of the d-th next one (1, 3:
sampled requests diverge); a rejected row's token written to its output slot or its state to the request (1, 6);
drafts kept past a stop or final-state token (5); draft rows taken from rows max_rows reserves (4: the replay's
steps); acceptance that compares a row with its own draft instead of its successor's (3, 4)."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_decode_sample_queue_constrained_gpu import loop_automaton  # noqa: E402
from test_decode_sample_queue_gpu import HD128, SEEDS, SETTINGS, Slots, greedy_setting, place_round, prompts_of  # noqa: E402
from test_decode_sample_queue_penalties_gpu import assert_same, launches, mixed_pen  # noqa: E402
from test_decode_sample_queue_truncated_gpu import qtr  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402
from test_verify_sample_gpu import xs_advance  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.lib import TokenAutomaton  # noqa: E402

pytestmark = pytest.mark.gpu

ROWS = 16  # SQ_ROWS: the rows of a queue step


def qlk(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows, max_draft, k=None, top_k=None, top_p=None, automaton=None, start=None,
        **pen):
    return dm.decode_sample_queue_lookup(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds,
                                         max_draft=max_draft, top_k=top_k, top_p=top_p, automaton=automaton, start=start, k=k, **pen)


def assert_truncated(got, want, label):
    """got (the lookup call's tuple) is want (the _truncated call's) bit for bit, steps at most want's."""
    assert len(got) == len(want) + 2, f"{label}: tuple length"
    assert got[2] == want[2] and got[4] == want[4], f"{label}: served / prompt_rows"
    assert got[3] <= want[3], f"{label}: {got[3]} steps, _truncated takes {want[3]}"
    assert_same(got[:-3], want[:-1], label)
    assert got[-3] == want[-1], f"{label}: out_state"
    assert 0 <= got[-1] <= got[-2], f"{label}: accepted {got[-1]} of {got[-2]} drafts"


def lookup(seq, cap):
    """The draft rule (vf_lookup with source NULL): the key is the last 3, else 2, else 1 tokens; the draft follows the
    key's rightmost occurrence that some token follows."""
    n = len(seq)
    for gl in (3, 2, 1):
        if n < gl:
            continue
        key = seq[n - gl:]
        for i in range(n - gl - 1, -1, -1):
            if seq[i:i + gl] == key:
                return seq[i + gl:i + gl + min(cap, n - i - gl)]
    return []


def cut(draft, stop, aut, s):
    """The draft up to (not including) its first stop token, token its state s disallows, or token leading to a final state."""
    out = []
    for v in draft:
        if v in stop:
            break
        if s >= 0:
            if v not in aut.allowed(s):
                break
            s = aut.next(s, v)
            if aut.final[s]:
                break
        out.append(v)
    return out


def replay(prompts, plain, max_new, max_rows, seq_len, max_draft, stop=(), aut=None, start=None, drafts=None):
    """test_decode_sample_queue_gpu.simulate's schedule (no contexts) with the header's drafts over the plain call's
    tokens: (steps, drafted, accepted).  drafts[i] False: request i never drafts (a non-neutral request)."""
    lens = [len(p) for p in prompts]
    out_len = [len(t) for t in plain]
    nreq = len(prompts)
    slots, place, live, done, head = Slots(seq_len), {}, [], {}, 0
    steps = drafted = accepted = 0
    stop = set(int(x) for x in stop)
    while True:
        rnd, rp, after = [], {}, slots
        while head < nreq and len(live) + len(rnd) < max_rows:
            if max_new[head] == 0:
                head += 1
                continue
            a = slots.copy()
            tp = place_round(a, rnd + [head], lens, max_new)
            if tp is None:
                break
            rnd, rp, after, head = rnd + [head], tp, a, head + 1
        if not live and not rnd:
            break
        slots = after
        place.update(rp)
        live += rnd
        free = ROWS - len(live)
        emitted = {}
        for i in live:
            j = done.get(i, 0)
            d = []
            if max_draft and (drafts is None or drafts[i]):
                s = -1 if start is None else start[i]
                for t in plain[i][:j]:
                    s = aut.next(s, int(t)) if s >= 0 else -1
                seq = [int(x) for x in prompts[i]] + [int(x) for x in plain[i][:j]]
                d = cut(lookup(seq, min(max_draft, max_new[i] - j - 1, free)), stop, aut, s)
                free -= len(d)
            a = 0
            while a < len(d) and j + a < out_len[i] and d[a] == plain[i][j + a]:
                a += 1
            drafted, accepted = drafted + len(d), accepted + a
            emitted[i] = a + 1
        steps += 1
        keep = []
        for i in live:
            done[i] = done.get(i, 0) + emitted[i]
            assert done[i] <= out_len[i]
            if done[i] < out_len[i]:
                keep.append(i)
            else:
                s, L, t = place[i]
                slots.give(s, -(-L // 8) * 8)
                slots.give(t, max_new[i])
        live = keep
    return steps, drafted, accepted


# ---- 1. the _truncated call's bits
KV1 = replace(TINY1, dtype="fp16", n_kv_heads=4)
KV8 = replace(mg.SPECS["pf-tiny"], name="kv8-hd128", dim=512, hidden_dim=1024, n_layers=1, n_heads=8, n_kv_heads=1, head_dim=128, rope_theta=5e5)
MATRIX = {  # (spec, kvbits, max_rows, nreq, context lengths (None: no contexts), own lengths, seq_len)
    "pf-tiny fp8 kv_mul2 r16 contexts": (mg.SPECS["pf-tiny"], 16, 16, 14, [250, 7], [1, 9, 40, 2], 4096),
    "pf-tiny gf4 e5m2 kv_mul2 r3 contexts": (replace(mg.SPECS["pf-tiny"], dtype="gf4"), 8, 3, 8, [120], [9, 1, 30], 4096),
    "pf-tiny fp16 kv_mul1 r1": (KV1, 16, 1, 5, None, [9, 129, 1], 2048),
    "pf-tiny-hd128 bias kv_mul4 e5m2 r16": (HD128, 8, 16, 10, [129], [2, 40, 1, 9], 4096),
    "hd128 kv_mul8 fp8 r3 contexts": (KV8, 16, 3, 8, [250], [1, 20, 5], 4096),
}


def matrix_requests(V, nreq, ctx_lens, own_lens):
    contexts = prompts_of(V, ctx_lens, start=101) if ctx_lens else None
    ctx_of = [-1 if i % 5 == 3 else i % len(contexts) for i in range(nreq)] if ctx_lens else None
    prompts = prompts_of(V, [own_lens[i % len(own_lens)] for i in range(nreq)], start=7)
    max_new = [[24, 40, 9, 0, 40, 1][i % 6] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]  # (request 1 greedy, 40 tokens)
    return contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq]


@pytest.mark.parametrize("case", sorted(MATRIX))
def test_same_bits_as_truncated(case):
    spec, kvbits, max_rows, nreq, ctx_lens, own_lens, seq_len = MATRIX[case]
    V = spec.vocab_size
    tensors = mg.generate(spec, 17, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = matrix_requests(V, nreq, ctx_lens, own_lens)
    args = (contexts, ctx_of, prompts, max_new, sets, seeds)
    aut = loop_automaton(V, [np.arange(V) % 3 != 0])
    tk = [[0, 5, 0, 20][i % 4] for i in range(nreq)]
    tp = [[1.0, 0.9, 0.8, 1.0][i % 4] for i in range(nreq)]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        plain = qtr(dm, *args, [], max_rows)
        stop = sorted({int(t[len(t) // 2]) for t in plain[0] if len(t) > 4})[:2]  # tokens some requests emit midway
        configs = {
            "plain": dict(k=None),
            "stops k5 mixed": dict(k=5, top_k=tk, top_p=tp, automaton=aut, start=[0 if i % 3 == 0 else -1 for i in range(nreq)],
                                   **mixed_pen(V, nreq, range(1, nreq, 4))),
        }
        accepted = 0
        for name, kw in configs.items():
            st = stop if name != "plain" else []
            want = qtr(dm, *args, st, max_rows, **kw)
            assert want[2] == 1
            for md in (1, 7, 15):
                got = qlk(dm, *args, st, max_rows, md, **kw)
                assert_truncated(got, want, f"{case} {name} max_draft {md}")
                accepted += got[-1]
        assert accepted > 0, f"{case}: no draft was accepted"


# ---- 2. max_draft 0
def test_max_draft_0_launches_what_truncated_launches():
    spec = mg.SPECS["pf-tiny"]
    V = spec.vocab_size
    contexts, ctx_of, prompts, max_new, sets, seeds = matrix_requests(V, 12, [250], [1, 9, 40])
    with lib.DeviceModel(spec, mg.generate(spec, 5, device="cuda"), seq_len=4096) as dm:
        for kw in (dict(), dict(k=5, top_k=[5] * 12, **mixed_pen(V, 12, [2, 7]))):
            n0 = launches()
            want = qtr(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [3], 4, **kw)
            n1 = launches()
            got = qlk(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [3], 4, 0, **kw)
            n2 = launches()
            assert_truncated(got, want, f"max_draft 0 {kw.keys()}")
            assert got[3] == want[3] and got[-2:] == (0, 0)
            assert n2 - n1 == n1 - n0, f"{n2 - n1} launches against {n1 - n0}"


# ---- 3. forced acceptance on a cycling automaton
def cycle_automaton(V, cyc):
    """State s allows cyc[s] alone and goes to s + 1 mod len(cyc): every stream is periodic."""
    allow = np.zeros((len(cyc), V), bool)
    allow[np.arange(len(cyc)), cyc] = True
    return TokenAutomaton(V, allow, (np.arange(len(cyc)) + 1) % len(cyc), None)


@pytest.mark.parametrize("max_rows", [1, 4])
def test_forced_acceptance(max_rows):
    spec = replace(TINY1, vocab_size=1000)
    V = spec.vocab_size
    cyc = [17, 250, 3, 99, 401, 3, 640]  # (3 twice: a 1-token key is ambiguous, a 2-token one is not)
    aut = cycle_automaton(V, cyc)
    nreq = 9
    prompts = prompts_of(V, [[5, 30, 1, 12][i % 4] for i in range(nreq)], start=3)
    prompts[2] = np.asarray(cyc * 3, np.int32)  # a prompt that holds the cycle itself: drafts from step 0
    start = [i % len(cyc) for i in range(nreq)]
    max_new = [[40, 13, 2, 30, 1][i % 5] for i in range(nreq)]
    sets = [[(0.0, 0.0), (1.0, 0.1), (0.7, 0.0)][i % 3] for i in range(nreq)]
    want_tok = [np.asarray([cyc[(start[i] + t) % len(cyc)] for t in range(max_new[i])], np.int32) for i in range(nreq)]
    with lib.DeviceModel(spec, mg.generate(spec, 9, device="cuda"), seq_len=2048) as dm:
        want = qtr(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, automaton=aut, start=start)
        for md in (3, 15):
            got = qlk(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, md, automaton=aut, start=start)
            assert_truncated(got, want, f"max_rows {max_rows} max_draft {md}")
            for i in range(nreq):
                assert np.array_equal(got[0][i], want_tok[i]), f"request {i} tokens"
                assert got[1][i] == (SEEDS[i] if greedy_setting(*sets[i]) else xs_advance(SEEDS[i], max_new[i])), f"request {i} state"
                assert got[-3][i] == (start[i] + max_new[i]) % len(cyc), f"request {i} out_state"
            sched = replay(prompts, want_tok, max_new, max_rows, 2048, md, aut=aut, start=start)
            assert got[3:4] + got[-2:] == sched, f"max_draft {md}: (steps, drafted, accepted) {got[3:4] + got[-2:]}, the replay {sched}"
            assert got[-1] == got[-2] > 0 and got[3] < want[3], "every draft of a forced stream is accepted"


# ---- 4. the replay on greedy random-model workloads
@pytest.mark.parametrize("spec,max_rows", [(replace(TINY1, vocab_size=300), 4), (mg.SPECS["pf-tiny"], 16), (HD128, 1)],
                         ids=["pf-tiny vocab 300 r4", "pf-tiny r16", "pf-tiny-hd128 r1"])
def test_schedule_is_the_replay(spec, max_rows):
    V = spec.vocab_size
    nreq = 20
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, V, int(n)).astype(np.int32) for n in rng.integers(1, 120, nreq)]
    max_new = [int(x) for x in rng.integers(0, 60, nreq)]
    sets = [(0.0, 0.0)] * nreq
    pen = mixed_pen(V, nreq, [4, 11])  # two requests that never draft
    drafts = [i not in (4, 11) for i in range(nreq)]
    with lib.DeviceModel(spec, mg.generate(spec, 13, device="cuda"), seq_len=4096) as dm:
        for stop in ([], [int(rng.integers(0, V))]):
            want = qtr(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], stop, max_rows, **pen)
            for md in (1, 7, 15):
                got = qlk(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], stop, max_rows, md, **pen)
                assert_truncated(got, want, f"stop {stop} max_draft {md}")
                sched = replay(prompts, want[0], max_new, max_rows, 4096, md, stop=stop, drafts=drafts)
                assert got[3:4] + got[-2:] == sched, f"stop {stop} max_draft {md}: {got[3:4] + got[-2:]}, the replay {sched}"
                assert got[-1] > 0, "greedy random models repeat themselves: some draft is accepted"


# ---- 5. stops and final states inside a draft
def test_draft_with_a_stop_or_final_token_ends_there():
    spec = replace(TINY1, vocab_size=1000)
    V = spec.vocab_size
    c = [17, 250, 3, 99]
    p, q = 600, 601
    prompt = np.asarray([p] + c + [q, p], np.int32)  # the key p drafts c ++ [q, p]
    cyc = cycle_automaton(V, c)  # c forever: the stop token c[3] ends the stream
    allow = np.zeros((len(c) + 1, V), bool)
    allow[np.arange(len(c)), c] = True
    chain = TokenAutomaton(V, allow, list(range(1, len(c) + 1)) + [-1], None)  # c[3] leads to a final state
    with lib.DeviceModel(spec, mg.generate(spec, 2, device="cuda"), seq_len=1024) as dm:
        for label, aut, stop in (("stop", cyc, [c[3]]), ("final", chain, [])):
            for t, mp in ((0.0, 0.0), (1.0, 0.1)):
                args = (None, None, [prompt], [20], [(t, mp)], [SEEDS[0]], stop, 1)
                want = qtr(dm, *args, automaton=aut, start=[0])
                got = qlk(dm, *args, 15, automaton=aut, start=[0])
                assert_truncated(got, want, f"{label} T {t}")
                assert np.array_equal(got[0][0], c), f"{label} T {t}: {got[0][0]}"
                assert got[3] == 1 and got[-2:] == (3, 3), f"{label} T {t}: steps {got[3]}, drafted / accepted {got[-2:]}"
                assert got[1][0] == (SEEDS[0] if t == 0.0 else xs_advance(SEEDS[0], 4))
                assert got[-3][0] == (0 if label == "stop" else len(c))


# ---- 6. untouched slots
def test_slots_past_out_len_are_untouched():
    spec = mg.SPECS["pf-tiny"]
    V = spec.vocab_size
    nreq = 10
    prompts = prompts_of(V, [[30, 9, 1][i % 3] for i in range(nreq)], start=5)
    sets = [(0.0, 0.0)] * nreq
    seen = {}
    with lib.DeviceModel(spec, mg.generate(spec, 8, device="cuda"), seq_len=4096) as dm:
        plain = qtr(dm, None, None, prompts, [40] * nreq, sets, SEEDS[:nreq], [], 16)
        stop = sorted({int(t[10]) for t in plain[0]})[:3]
        real = dm.lib.calm_b200_decode_sample_queue_lookup

        def spy(*args):  # the wrapper's own output arrays, read before it slices them
            r = real(*args)
            total = 40 * nreq
            seen["out"] = np.ctypeslib.as_array(args[23], (total,)).copy()
            seen["lp"] = np.ctypeslib.as_array(args[28], (total,)).copy()
            seen["ids"] = np.ctypeslib.as_array(args[29], (total * 3,)).copy()
            return r

        dm.lib.calm_b200_decode_sample_queue_lookup = spy
        try:
            got = qlk(dm, None, None, prompts, [40] * nreq, sets, SEEDS[:nreq], stop, 16, 15, k=3)
        finally:
            dm.lib.calm_b200_decode_sample_queue_lookup = real
        want = qtr(dm, None, None, prompts, [40] * nreq, sets, SEEDS[:nreq], stop, 16, k=3)
    assert_truncated(got, want, "stops")
    assert got[-2] > got[-1] > 0, "some drafts were rejected"
    assert any(len(t) < 40 for t in got[0]), "a stop fired"
    for i, t in enumerate(got[0]):
        o, n = 40 * i, len(t)
        assert (seen["out"][o + n:o + 40] == -1).all(), f"request {i}: a token past out_len"
        assert np.isnan(seen["lp"][o + n:o + 40]).all(), f"request {i}: a log-probability past out_len"
        assert (seen["ids"][3 * (o + n):3 * (o + 40)] == -1).all(), f"request {i}: a top id past out_len"


# ---- 7. history
def test_same_bits_after_other_calls_and_poison():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 23, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = matrix_requests(V, 16, [250, 40], [9, 1, 40, 2])
    kw = dict(k=3, top_k=[[0, 5][i % 2] for i in range(16)], **mixed_pen(V, 16, [5]))
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        ref = qlk(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], 16, 7, **kw)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        other = prompts_of(V, [700, 33, 2], start=50)
        qlk(dm, [other[0]], [0, 0, -1], other, [60, 5, 30], [(1.1, 0.0), (0.0, 0.0), (0.9, 0.1)], SEEDS[20:23], [], 2, 15, k=20)
        dm.decode_sample_batch(other, 9, 0.9, 0.05, SEEDS[:3])
        dm.poison(0)
        got = qlk(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], 16, 7, **kw)
    assert got[2:5] == ref[2:5] and got[-3:] == ref[-3:]
    assert_same(got[:-3], ref[:-3], "dirty engine")


# ---- 8. the fallback
@pytest.mark.parametrize("name,seq_len,lens,max_new", [("tiny-moe", None, [6, 1, 12], [9, 0, 5]), ("pf-tiny", 64, [21, 50, 11], [8, 20, 3])])
def test_fallback_is_the_truncated_fallback(name, seq_len, lens, max_new):
    spec = mg.SPECS[name]
    V = spec.vocab_size
    contexts = prompts_of(V, [4], start=8)
    ctx_of = [0, -1, 0]
    prompts = prompts_of(V, lens, start=1)
    sets = [(1.0, 0.0), (0.0, 0.1), (0.7, 0.05)]
    kw = dict(k=3, top_k=[5, 3, 0], top_p=[0.9, 0.5, 0.8], presence=[0.5, 0.0, 0.0])
    with lib.DeviceModel(spec, mg.generate(spec, 45), seq_len=seq_len) as dm:
        want = qtr(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, **kw)
        got = qlk(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, 7, **kw)
    assert want[2] == 0 and got[2:5] == want[2:5] and got[3] == 0 and got[-2:] == (0, 0)
    assert_same(got[:-3], want[:-1], name)
    assert got[-3] == want[-1]


# ---- 9. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(contexts=None, ctx_of=None, prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4, rng_states=[1],
                  max_draft=7, top_k=[3], top_p=[0.9], k=2)
        bad = [dict(max_draft=-1), dict(max_draft=16), dict(max_draft=1.5), dict(max_draft=True), dict(max_draft=None), dict(top_k=[-1]),
               dict(top_p=[1.5]), dict(k=-1), dict(max_rows=17), dict(start=[0]), dict(max_new=[-1])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue_lookup(**{**ok, **b})
        got = dm.decode_sample_queue_lookup(**ok)
        assert got[2] == 1 and len(got[0][0]) == 4 and got[-2] >= got[-1] >= 0
