"""calm_b200_decode_sample_queue_truncated: the queue with per-request top-k / top-p truncation of sampled rows, applied
by k_sample_trunc_rows (an 8-CTA cluster radix select per row) between the classifier and the masked sampler scan.

1. Neutral requests (top_k / top_p None, or all (0, 1)) give the _constrained call's bits and launch counts over the
   penalties tests' case matrix, with and without penalties, an automaton and k.
2. Step 0 exactly: the PF_LOGITS row is the _constrained row with -inf at exactly the ids test_truncation_rule's
   restatement drops (a neighbouring nucleus boundary only where expf's ulp explains it, and rarely); the token and
   state are masked_algorithm on the device's own row.
3. The kernel at 32000 / 128256 / 151936 / 262144 tokens through sample_logits_truncated: flat, peaked, all-equal,
   tie groups and boundaries across the 8 CTA segment edges, many -inf entries.
4. Invariants over many steps from each step's own top_ids / top_logprobs at k = 20.  5. Independence of the other
   requests, max_rows, seq_len, shared contexts and call history.  6. Qwen2-style defaults mixed with greedy and neutral
   requests.  7. The fallback equals a host replay on sample_logits_truncated.  8. Bad arguments raise ValueError.

Mutations the tests are built to catch (by the test named): ties broken by the highest id (2, 3: the all-equal and
tie-group rows keep the lowest ids); a nucleus normalised over all tokens instead of the top-k set (2, 3: rows with
both K and P); a prefix that stops one token early, > instead of >= (3: P = j/n over n equal logits hits the target
exactly); masses at temperature 1 instead of T (2: T 0.6 and 2 rows); a row's settings indexed by row instead of by
request (5: rows compact as requests retire); a CTA's histogram left out of the cluster merge (3: boundaries in every
segment); truncation applied to greedy rows (1, 6: greedy requests with top_k / top_p keep their bits)."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_decode_sample_queue_constrained_gpu import loop_automaton, masked_algorithm, qcon  # noqa: E402
from test_decode_sample_queue_context_gpu import concat  # noqa: E402
from test_decode_sample_queue_gpu import HD128, SEEDS, ceil8, greedy_setting, prompts_of  # noqa: E402
from test_decode_sample_queue_logprobs_gpu import merge_tol, same_bits  # noqa: E402
from test_decode_sample_queue_penalties_gpu import CASES, assert_same, case_requests, host_state, launches, mixed_pen, process  # noqa: E402
from test_truncation_rule import boundary_slack, kept, rank_order  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu


def qtr(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows, k=None, top_k=None, top_p=None, automaton=None, start=None, **pen):
    return dm.decode_sample_queue_truncated(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds,
                                            top_k=top_k, top_p=top_p, automaton=automaton, start=start, k=k, **pen)


def check_row(src, got, T, K, P, label):
    """got is src truncated by the rule: a rank prefix of src's allowed tokens, of the rule's length (or, for top-p, one
    whose boundary expf's ulp explains).  Returns whether the length differed."""
    order = rank_order(src)
    fin = np.isfinite(got)
    assert (fin <= np.isfinite(src)).all(), f"{label}: an id the row did not allow"
    assert same_bits(got[fin], src[fin]), f"{label}: a kept logit changed"
    n_got = int(fin.sum())
    assert fin[order[:n_got]].all(), f"{label}: the kept ids are not a rank prefix"
    n, _ = kept(src, T, K, P)
    assert boundary_slack(src, T, K, P, n_got), f"{label}: {n_got} ranks kept, the rule keeps {n}"
    return n_got != n


def sample_row(row, T, minp, K, P, state):
    tok, st, out = lib.sample_logits_truncated(row, T, minp, K, P, state)
    return tok, st, out


# ---- 1. neutral requests are the _constrained call
@pytest.mark.parametrize("case", sorted(CASES))
def test_neutral_is_the_constrained_call(case):
    spec, kvbits, max_rows, nreq, ctx_lens, own_lens, seq_len = CASES[case]
    V = spec.vocab_size
    tensors = mg.generate(spec, 17, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = case_requests(V, nreq, ctx_lens, own_lens)
    args = (contexts, ctx_of, prompts, max_new, sets, seeds, [], max_rows)
    aut = loop_automaton(V, [np.arange(V) % 3 != 0])
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        for k, pen, con in ((None, {}, {}), (5, mixed_pen(V, nreq, range(0, nreq, 2)), {}),
                            (3, {}, dict(automaton=aut, start=[0 if i % 3 == 0 else -1 for i in range(nreq)]))):
            n0 = launches()
            want = qcon(dm, *args, k=k, **con, **pen)
            n1 = launches()
            for label, kw in (("None", {}), ("neutral", dict(top_k=[0] * nreq, top_p=[1.0] * nreq))):
                m0 = launches()
                got = qtr(dm, *args, k=k, **kw, **con, **pen)
                m1 = launches()
                tag = f"{case} k {k} {label} pen {bool(pen)} aut {bool(con)}"
                assert got[2:5] == want[2:5], f"{tag}: served / steps / prompt_rows"
                assert_same(got[:-1], want[:-1], tag)
                assert got[-1] == want[-1], f"{tag}: out_state"
                assert m1 - m0 == n1 - n0, f"{tag}: {m1 - m0} launches against {n1 - n0}"
        # greedy requests with truncation settings, neutral ones beside truncated ones: their bits stay
        tk = [[0, 5, 1, 20][i % 4] for i in range(nreq)]
        tp = [[1.0, 0.9, 0.5, 1.0][i % 4] for i in range(nreq)]
        want = qcon(dm, *args, k=3)
        got = qtr(dm, *args, k=3, top_k=tk, top_p=tp)
        keep = [i for i in range(nreq) if greedy_setting(*sets[i]) or (tk[i] == 0 and tp[i] == 1.0)]
        assert_same(got[:-1], want[:-1], f"{case} greedy / neutral among truncated", keep)
        for i in range(nreq):  # logprobs describe the distribution before truncation: top-k still lists it
            for j, t in enumerate(got[0][i]):
                if tk[i] and not greedy_setting(*sets[i]):
                    assert t in got[6][i][j][:3] or tk[i] > 3, f"{case}: request {i} step {j} emitted a token outside its top-{tk[i]}"


# ---- 2. step 0 exactly
@pytest.mark.parametrize("spec", [replace(TINY1, vocab_size=1000), HD128], ids=["pf-tiny vocab 1000", "pf-tiny-hd128 bias"])
def test_step0_is_the_truncated_constrained_row(spec):
    tensors = mg.generate(spec, 5, device="cuda")
    V = spec.vocab_size
    rng = np.random.default_rng(7)
    grid = [(T, mp, K, P) for T in (0.6, 1.0, 2.0) for mp in (0.0, 0.1) for K, P in
            ((1, 1.0), (2, 0.9), (20, 0.8), (50, 1.0), (V - 1, 0.5), (V + 7, 0.9), (0, 1e-30), (0, 0.5), (20, 0.9), (0, 0.8))]
    nreq = 8
    prompts = prompts_of(V, [9, 30, 5, 1, 17, 2, 40, 3], start=3)
    allowed = rng.random((2, V)) < 0.4
    aut = loop_automaton(V, allowed)
    start = [0, -1, 1, -1, -1, 0, -1, -1]
    pen = mixed_pen(V, nreq, [0, 3, 6])
    slack = 0
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        for g0 in range(0, len(grid), nreq):
            g = [grid[(g0 + i) % len(grid)] for i in range(nreq)]
            sets = [(T, mp) for T, mp, _, _ in g]
            seeds = SEEDS[g0 % 40:g0 % 40 + nreq]
            base = qcon(dm, None, None, prompts, [1] * nreq, sets, seeds, [], nreq, k=5, automaton=aut, start=start, **pen)
            src = dm.read_state("pf_logits").reshape(-1, V).copy()
            got = qtr(dm, None, None, prompts, [1] * nreq, sets, seeds, [], nreq, k=5, top_k=[x[2] for x in g], top_p=[x[3] for x in g],
                      automaton=aut, start=start, **pen)
            rows = dm.read_state("pf_logits").reshape(-1, V)
            assert got[2] == 1
            for b in range(nreq):
                T, mp, K, P = g[b]
                label = f"T {T} minp {mp} K {K} P {P} row {b}"
                slack += check_row(src[b], rows[b], T, K, P, label)
                tok, st = masked_algorithm(rows[b], T, mp, seeds[b])
                assert int(got[0][b][0]) == tok and got[1][b] == st, f"{label}: token / state"
                # log-probabilities are the untruncated distribution's: top-k lists unchanged, the token's from src
                assert np.array_equal(got[6][b], base[6][b]) and same_bits(got[7][b], base[7][b]), f"{label}: top-k changed"
                r64 = src[b][np.isfinite(src[b])].astype(np.float64)
                lse = np.log(np.exp(r64 - r64.max()).sum()) + r64.max()
                want_lp = float(src[b][tok]) - lse
                assert abs(float(got[5][b][0]) - want_lp) <= merge_tol(want_lp, lse), f"{label}: logprob"
    assert slack <= len(grid) // 10, f"{slack} rows needed the ulp slack"


# ---- 3. the kernel at real vocabularies
def rows_for(V, rng):
    S = -(-V // 8)
    flat = rng.normal(0, 0.05, V).astype(np.float32)
    peaked = rng.normal(0, 3.0, V).astype(np.float32)
    peaked[rng.integers(V)] = 25.0
    equal = np.zeros(V, np.float32)
    ties = np.round(rng.normal(0, 1.0, V), 1).astype(np.float32)  # ~60 distinct values: every group crosses segments
    edges = np.full(V, -3.0, np.float32)
    for c in range(1, 8):  # equal tops straddling each segment edge
        edges[c * S - 2:c * S + 2] = 4.0
    sparse = np.full(V, -np.inf, np.float32)
    on = rng.random(V) < 0.01
    sparse[on] = rng.normal(0, 2.0, int(on.sum())).astype(np.float32)
    return dict(flat=flat, peaked=peaked, equal=equal, ties=ties, edges=edges, sparse=sparse)


@pytest.mark.parametrize("V", [32000, 128256, 151936, 262144])
def test_kernel_at_real_vocabularies(V):
    rng = np.random.default_rng(V)
    slack = total = 0
    settings = [(1.0, 0.0, 1, 1.0), (1.0, 0.0, 50, 1.0), (0.6, 0.0, 0, 0.9), (0.7, 0.0, 20, 0.8), (2.0, 0.0, 0, 0.5), (1.0, 0.1, 5000, 0.95),
                (1.0, 0.0, V // 8 + 3, 1.0), (1.0, 0.0, 0, 1e-30)]
    for name, row in rows_for(V, rng).items():
        for T, mp, K, P in settings:
            label = f"V {V} {name} T {T} K {K} P {P}"
            s0 = SEEDS[total % len(SEEDS)]
            tok, st, out = sample_row(row, T, mp, K, P, s0)
            slack += check_row(row, out, T, K, P, label)
            total += 1
            want = masked_algorithm(out, T, mp, s0)
            assert (tok, st) == want, f"{label}: token / state"
            if name == "equal":
                n = int(np.isfinite(out).sum())
                assert np.isfinite(out[:n]).all(), f"{label}: the lowest ids are kept"
            if name == "edges" and K == 1:
                assert np.isfinite(out).sum() == 1 and np.isfinite(out[-(-V // 8) - 2]), f"{label}: the first of the tied top"
    # P = j / n over n equal logits: the prefix stops exactly at the target
    for n, j in ((64, 16), (1024, 1023), (4096, 1)):
        row = np.full(V, -np.inf, np.float32)
        row[np.linspace(0, V - 1, n).astype(int)] = 0.5
        _, _, out = sample_row(row, 1.0, 0.0, 0, j / n, 1)
        assert int(np.isfinite(out).sum()) == j, f"V {V}: {n} equal, P {j}/{n}"
    assert slack <= total // 10


# ---- 4. invariants over many steps
def test_invariants_over_many_steps():
    spec = replace(TINY1, vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 31, device="cuda")
    nreq = 64
    prompts = prompts_of(V, [[9, 1, 30, 4][i % 4] for i in range(nreq)], start=5)
    max_new = [24] * nreq
    with lib.DeviceModel(spec, tensors, seq_len=2048) as dm:
        got = qtr(dm, None, None, prompts, max_new, [(2.0, 0.0)] * nreq, SEEDS[:nreq] + SEEDS[:16], [], 16, k=20, top_k=[5] * nreq)
        for i in range(nreq):
            for j, t in enumerate(got[0][i]):
                assert t in got[6][i][j][:5], f"top_k 5: request {i} step {j}"
        for P in (0.5, 0.9):
            got = qtr(dm, None, None, prompts, max_new, [(1.0, 0.0)] * nreq, SEEDS[:nreq] + SEEDS[:16], [], 16, k=20, top_p=[P] * nreq)
            for i in range(nreq):
                for j, t in enumerate(got[0][i]):
                    ids, lps = got[6][i][j], got[7][i][j].astype(np.float64)
                    r = list(ids).index(t) if t in ids else len(ids)  # past rank 20: the whole list lies above it
                    assert np.exp(lps[:r]).sum() < P + 1e-4, f"top_p {P}: request {i} step {j}"


# ---- 5. independence
def test_outputs_do_not_depend_on_schedule_or_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 23, device="cuda")
    contexts = prompts_of(V, [300, 129], start=61)
    nreq = 40
    ctx_of = [[-1, 0, 1, 0][i % 4] for i in range(nreq)]
    lens = [[9, 1, 40, 2, 17][i % 5] for i in range(nreq)]
    prompts = prompts_of(V, lens, start=3)
    max_new = [[13, 1, 25, 7, 0][(3 * i + 1) % 5] for i in range(nreq)]
    sets = [[(1.0, 0.0), (0.7, 0.05), (0.0, 0.1), (2.0, 0.0), (1.3, 0.1)][i % 5] for i in range(nreq)]
    tk = [[0, 5, 20, 1, 0, 50, 2][i % 7] for i in range(nreq)]
    tp = [[0.9, 1.0, 0.8, 1.0, 0.5, 0.95][i % 6] for i in range(nreq)]
    pen = mixed_pen(V, nreq, [i for i in range(nreq) if i % 4 == 1])
    clen = [len(contexts[c]) if c >= 0 else 0 for c in ctx_of]
    tight = max(ceil8(c) + ceil8(n - 1) + m for c, n, m in zip(clen, lens, max_new)) + 16
    kw = dict(k=3, top_k=tk, top_p=tp, **pen)
    runs = {}
    for seq_len in (4096, tight):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            for max_rows in ((1, 3, 16) if seq_len == 4096 else (16,)):
                runs[(seq_len, max_rows)] = qtr(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, **kw)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        alone = {}
        for i in (1, 2, 3, 5, 6, 9, 10, 12):
            one = {key: [v[i]] for key, v in kw.items() if isinstance(v, list)}
            alone[i] = qtr(dm, [contexts[ctx_of[i]]] if ctx_of[i] >= 0 else None, [0] if ctx_of[i] >= 0 else None, [prompts[i]], [max_new[i]], [sets[i]],
                           [SEEDS[i]], [], 16, k=3, **one)
        other = prompts_of(V, [700, 33, 2], start=50)
        qtr(dm, [other[0]], [0, 0, -1], other, [60, 5, 30], [(1.1, 0.0)] * 3, SEEDS[20:23], [], 2, k=20, top_k=[3, 0, 9], top_p=[0.5, 0.7, 1.0])
        dm.poison(0)
        runs["dirty"] = qtr(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], 16, **kw)
    ref = runs[(4096, 16)]
    assert ref[2] == 1 and all(len(t) == m for t, m in zip(ref[0], max_new))
    for key, got in runs.items():
        assert got[2] == 1
        assert_same(got[:-1], ref[:-1], str(key))
    for i, got in alone.items():
        assert_same(got[:-1], tuple([x[i]] if isinstance(x, list) else x for x in ref[:-1]), f"request {i} alone", [0])


# ---- 6. Qwen2-style defaults
@pytest.mark.parametrize("name", ["tiny-qwen", "qwen2-0.5b-fp16"])
def test_qwen2_style_defaults(name):
    spec = mg.SPECS[name]
    if name != "tiny-qwen":
        spec = replace(spec, n_layers=2)  # the 151936-token classifier at Qwen2-0.5B's widths, two layers
    V = spec.vocab_size
    tensors = mg.generate(spec, 3, device="cuda")
    nreq = 12
    prompts = prompts_of(V, [[7, 20, 1][i % 3] for i in range(nreq)], start=9)
    sets = [[(0.7, 0.0), (0.0, 0.0), (0.7, 0.0), (1.0, 0.1)][i % 4] for i in range(nreq)]
    qwen = [i % 4 in (0, 1) for i in range(nreq)]  # the greedy ones carry the settings too; i % 4 == 2 / 3 are neutral
    tk = [20 if q else 0 for q in qwen]
    tp = [0.8 if q else 1.0 for q in qwen]
    rep = [1.05 if q else 1.0 for q in qwen]
    max_new = [12] * nreq
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        want = qcon(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], 16, k=20, repetition=rep)
        got = qtr(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], 16, k=20, top_k=tk, top_p=tp, repetition=rep)
    assert got[2] == want[2]  # (tiny-qwen's shapes decode on the fallback)
    assert_same(got[:-1], want[:-1], name, [i for i in range(nreq) if not (qwen[i] and not greedy_setting(*sets[i]))])
    for i in range(nreq):
        if qwen[i] and not greedy_setting(*sets[i]):
            for j, t in enumerate(got[0][i]):
                assert t in got[6][i][j], f"{name}: request {i} step {j} past its top 20"


# ---- 7. the fallback
@pytest.mark.parametrize("name,seq_len,lens,max_new", [("tiny-moe", None, [6, 1, 12], [9, 0, 5]), ("pf-tiny", 64, [21, 50, 11], [8, 20, 3])])
def test_fallback_is_a_host_replay(name, seq_len, lens, max_new):
    spec = mg.SPECS[name]
    V = spec.vocab_size
    tensors = mg.generate(spec, 45)
    contexts = prompts_of(V, [4], start=8)
    ctx_of = [0, -1, 0]
    prompts = prompts_of(V, lens, start=1)
    sets = [(1.0, 0.0), (0.0, 0.1), (0.7, 0.05)]
    tk, tp = [5, 3, 0], [0.9, 0.5, 0.8]
    cat = [concat(contexts, c, p) for c, p in zip(ctx_of, prompts)]
    pen = dict(presence=[0.5, 0.0, 0.0], frequency=[0.3, 0.0, 0.0], repetition=[1.2, 1.0, 1.0], logit_bias=[{3: -2.0}, None, None])
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        plain = qcon(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k=3, **pen)
        got = qtr(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k=3, top_k=tk, top_p=tp, **pen)
        assert got[2] == 0 and plain[2] == 0
        assert_same(got[:-1], plain[:-1], f"{name} greedy request", [1])
        for i in (0, 2):
            p, s = cat[i], SEEDS[i]
            dm.prefill(p[:-1], 0)
            tok = int(p[-1])
            gen = []
            for j in range(max_new[i]):
                dm.forward_sample(tok, len(p) - 1 + j, 0.0, 0.0, 1)
                seen, c, bv = host_state(V, p, gen, pen["logit_bias"][i])
                row = process(dm.device_logits(), seen, c, pen["presence"][i], pen["frequency"][i], pen["repetition"][i], bv)
                tok, s, _ = sample_row(row, *sets[i], tk[i], tp[i], s)
                assert tok == got[0][i][j], f"{name}: request {i} step {j}"
                gen.append(tok)
            assert len(got[0][i]) == max_new[i] and (max_new[i] == 0 or got[1][i] == s), f"{name}: request {i}"


# ---- 8. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(contexts=None, ctx_of=None, prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4, rng_states=[1],
                  top_k=[3], top_p=[0.9], k=2)
        bad = [dict(top_k=[-1]), dict(top_k=[1, 2]), dict(top_k=[1.5]), dict(top_p=[0.0]), dict(top_p=[1.5]), dict(top_p=[np.nan]),
               dict(top_p=[np.inf]), dict(top_p=[-0.1]), dict(top_p=[0.5, 0.5]), dict(k=-1), dict(max_rows=17), dict(start=[0])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue_truncated(**{**ok, **b})
        got = dm.decode_sample_queue_truncated(**ok)
        assert got[2] == 1 and len(got[0][0]) == 4
    row = np.zeros(10, np.float32)
    for K, P in ((-1, 0.5), (1, 0.0), (1, 2.0), (1, float("nan")), (True, 0.5)):
        with pytest.raises(ValueError):
            lib.sample_logits_truncated(row, 1.0, 0.0, K, P, 1)
    with pytest.raises(ValueError):
        lib.sample_logits_truncated(np.zeros(TRUNC_BIG, np.float32), 1.0, 0.0, 5, 1.0, 1)
    tok, st, out = lib.sample_logits_truncated(np.zeros(TRUNC_BIG, np.float32), 0.0, 0.0, 5, 0.5, 1)  # greedy: accepted, unchanged
    assert tok == 0 and st == 1 and np.array_equal(out, np.zeros(TRUNC_BIG, np.float32))


TRUNC_BIG = lib.TRUNC_VOCAB_MAX + 1
