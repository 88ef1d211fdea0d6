"""calm_b200_decode_sample_queue_constrained: the queue with requests constrained to a token automaton (structured
output), each step's disallowed tokens set to -inf in k_vf_gemm's classifier epilogue from the state the host follows.

1. Unconstrained requests (start None, or every start -1) give tokens, states, steps, prompt_rows, logprobs and top-k
   bit for bit equal to decode_sample_queue_penalties, with equal calm_b200_launch_count deltas, over the penalties
   tests' case matrix (fp8 / gf4 / fp16, head_dim 128 with bias, Llama-3-8B widths, both caches, max_rows 1 / 3 / 16).
2. A one-state automaton that allows every token and loops gives the unconstrained bits (neutral, penalised, greedy).
3. Step 0 exactly: a constrained request's PF_LOGITS row is the _penalties row with -inf at exactly the masked ids; its
   token and state are the masked device sampler (test_sampler's _device_algorithm with masked tokens never surviving)
   on that row at minp 0 and 0.1; a greedy request's token is the first allowed maximum.
4. Sampler and tile edges: one allowed token (forced, one draw), two, more than 2048 survivors (chunk path), every
   allowed token inside one 128-token tile, allowed tokens only in the partial last tile, many fully masked tiles; 64
   sampled requests at T = 2, minp 0 never emit a masked token.  5. Top-k past the allowed set is -1 / -inf, the
   allowed ranks host_topk of the masked row.
6. guided_choice: 40 requests on choices tries under max_rows 1 / 4 / 16 mixed with unconstrained and penalised ones
   emit exactly one choice each, with out_len its length and a final out_state; unconstrained requests keep their
   bits; each step of a greedy constrained request matches a prompt-pass recomputation, processed and masked.
7. Each request gives the same bits alone, among 40 requests, at a tight seq_len, with shared contexts, and after
   another call plus poisoning.  8. The fallback (MoE, a request past seq_len) returns 0 and equals a host replay.
9. Bad arguments raise ValueError.

Mutations the tests are designed to catch (by the test named): the state indexed by row instead of by request (6 and 7:
rows compact as requests retire, so a row would read another request's state); the state advanced before the step's
mask is read (6 and 7: their states change with every token, so a step masked by the state after its own token emits
tokens the automaton's walk does not allow; test 3's states loop, so it cannot see this); masked tokens surviving at minp 0 (3,
4: the survivor count and fallback change, and a masked token can be drawn); top-k past the allowed set emitting
INT_MAX (5); a final state not retiring the request (6: out_len would exceed the choice's length)."""
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
from test_decode_sample_queue_penalties_gpu import CASES, assert_same, case_requests, host_state, launches, mixed_pen, process, qpen  # noqa: E402
from test_score_topk_gpu import host_topk  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.lib import TokenAutomaton  # noqa: E402

pytestmark = pytest.mark.gpu


def qcon(dm, contexts, ctx_of, prompts, max_new, sets, seeds, stop, max_rows, k=None, automaton=None, start=None, **pen):
    return dm.decode_sample_queue_constrained(contexts, ctx_of, prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds,
                                              automaton=automaton, start=start, k=k, **pen)


def masked_algorithm(logits, temperature, minp, rng_state, chunk=1024, exact=2048):
    """test_sampler's _device_algorithm (k_sample_scan + k_sample_pick) where a -inf logit never survives the cut:
    k_sample_scan_rows_masked + k_sample_pick_rows.  Returns (token, state)."""
    f = np.float32
    s = rng_state
    s ^= s >> 12
    s ^= (s << 25) & 0xFFFFFFFFFFFFFFFF
    s ^= s >> 27
    coin = f(((s * 0x2545F4914F6CDD1D & 0xFFFFFFFFFFFFFFFF) >> 32) >> 8) / f(16777216.0)
    mx = f(logits.max())
    with np.errstate(divide="ignore"):
        cutoff = f(mx + f(f(np.log(f(minp))) * f(temperature)))
    chunks = []
    for c0 in range(0, len(logits), chunk):
        l = logits[c0:c0 + chunk]
        keep = np.nonzero((l >= cutoff) & (l != -np.inf))[0]
        probs = np.exp(((l[keep] - mx) / f(temperature)).astype(f)).astype(f)
        csum = f(0)
        for p in probs:
            csum = f(csum + p)
        chunks.append((keep + c0, probs, csum))
    total = sum(len(k) for k, _, _ in chunks)
    fallback = max((int(k[-1]) for k, _, _ in chunks if len(k)), default=0)
    cum = f(0)
    if total <= exact:
        for _, probs, _ in chunks:
            for p in probs:
                cum = f(cum + p)
    else:
        for _, _, cs in chunks:
            cum = f(cum + cs)
    r = f(coin * cum)
    cdf = f(0)
    for idx, probs, cs in chunks:
        if total > exact and not (r < f(cdf + cs)):
            cdf = f(cdf + cs)
            continue
        for i, p in zip(idx, probs):
            cdf = f(cdf + p)
            if r < cdf:
                return int(i), s
    return fallback, s


def pick(row, temperature, minp, state):
    """The token (and state) the queue draws from a masked row: the first maximum when greedy."""
    if greedy_setting(temperature, minp):
        return int(np.argmax(row)), state
    return masked_algorithm(row, temperature, minp, state)


def mask_row(row, allowed):
    return np.where(allowed, row, np.float32(-np.inf)).astype(np.float32)


def loop_automaton(V, allowed_rows):
    """One state per bool row, each looping to itself."""
    a = np.asarray(allowed_rows, bool)
    return TokenAutomaton(V, a, np.arange(len(a)), None)


def edge_automaton(V, allowed_rows):
    """One state per bool row, each going to one final state after any token."""
    a = np.zeros((len(allowed_rows) + 1, V), bool)
    a[:-1] = allowed_rows
    n = len(allowed_rows)
    return TokenAutomaton(V, a, [n] * n + [-1], None)


# ---- 1. unconstrained requests are the _penalties call
@pytest.mark.parametrize("case", sorted(CASES))
def test_unconstrained_is_the_penalties_call(case):
    spec, kvbits, max_rows, nreq, ctx_lens, own_lens, seq_len = CASES[case]
    tensors = mg.generate(spec, 17, device="cuda")
    contexts, ctx_of, prompts, max_new, sets, seeds = case_requests(spec.vocab_size, nreq, ctx_lens, own_lens)
    args = (contexts, ctx_of, prompts, max_new, sets, seeds, [], max_rows)
    aut = TokenAutomaton.choices([[1, 2], [3]], spec.vocab_size)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        for k in (None, 5):
            for pen in ({}, mixed_pen(spec.vocab_size, nreq, range(0, nreq, 2))):
                n0 = launches()
                want = qpen(dm, *args, k=k, **pen)
                n1 = launches()
                for label, kw in (("start None", {}), ("all -1", dict(automaton=aut, start=[-1] * nreq))):
                    m0 = launches()
                    got = qcon(dm, *args, k=k, **kw, **pen)
                    m1 = launches()
                    tag = f"{case} k {k} {label} pen {bool(pen)}"
                    assert len(got) == len(want) + 1 and got[2:5] == want[2:5], f"{tag}: served / steps / prompt_rows"
                    assert_same(got[:-1], want, tag)
                    assert got[-1] == [-1] * nreq, f"{tag}: out_state"
                    assert m1 - m0 == n1 - n0, f"{tag}: {m1 - m0} launches against {n1 - n0}"


# ---- 2. an automaton that allows everything changes nothing
@pytest.mark.parametrize("spec", [replace(TINY1, vocab_size=1000), mg.SPECS["pf-tiny"]], ids=["pf-tiny vocab 1000", "pf-tiny"])
def test_allow_all_is_unconstrained(spec):
    V = spec.vocab_size
    tensors = mg.generate(spec, 9, device="cuda")
    nreq = 12
    contexts, ctx_of, prompts, max_new, sets, seeds = case_requests(V, nreq, [40], [9, 1, 30])
    pen = mixed_pen(V, nreq, range(0, nreq, 3))
    aut = loop_automaton(V, [np.ones(V, bool)])
    start = [0 if i % 2 == 0 else -1 for i in range(nreq)]
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        for k in (None, 5):
            want = qpen(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], 16, k=k, **pen)
            got = qcon(dm, contexts, ctx_of, prompts, max_new, sets, seeds, [], 16, k=k, automaton=aut, start=start, **pen)
            assert got[2:5] == want[2:5]
            assert_same(got[:-1], want, f"k {k}")
            assert got[-1] == [0 if s == 0 else -1 for s in start]


# ---- 3. step 0 exactly
@pytest.mark.parametrize("minp", [0.0, 0.1])
@pytest.mark.parametrize("spec", [replace(TINY1, vocab_size=1000), HD128], ids=["pf-tiny vocab 1000", "pf-tiny-hd128 bias"])
def test_step0_is_the_masked_penalties_row(spec, minp):
    tensors = mg.generate(spec, 5, device="cuda")
    V = spec.vocab_size
    rng = np.random.default_rng(7)
    contexts = prompts_of(V, [40], start=11)
    prompts = prompts_of(V, [9, 30, 5], start=3)
    sets = [(0.0, 0.1), (1.0, minp), (2.0, minp)]  # greedy, sampled, sampled flat
    seeds = SEEDS[:3]
    pen = dict(presence=[0.5, 0.0, 0.3], frequency=[0.25, 0.0, 0.0], repetition=[1.2, 1.0, 0.9],
               logit_bias=[{int(prompts[0][0]): 1.5}, None, {4: -2.0}])
    allowed = rng.random((3, V)) < 0.3
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        plain = qpen(dm, contexts, [0, -1, 0], prompts, [1] * 3, sets, seeds, [], 3, k=5, **pen)
        raw = dm.read_state("pf_logits").reshape(-1, V).copy()
        plain_row0 = raw[0].copy()
        # the plain greedy token is masked for request 0, so the constraint moves it
        allowed[0, int(plain[0][0][0])] = False
        aut = loop_automaton(V, allowed)
        got = qcon(dm, contexts, [0, -1, 0], prompts, [1] * 3, sets, seeds, [], 3, k=5, automaton=aut, start=[0, 1, 2], **pen)
        rows = dm.read_state("pf_logits").reshape(-1, V)
    assert got[2] == 1 and rows.shape[0] == 3
    for b in range(3):
        want = mask_row(raw[b], allowed[b])
        assert same_bits(rows[b], want), f"row {b}: PF_LOGITS is not the masked _penalties row ({int((rows[b] != want).sum())} entries differ)"
        tok, st = pick(want, *sets[b], seeds[b])
        assert int(got[0][b][0]) == tok and allowed[b, tok], f"row {b}: token {int(got[0][b][0])}, want {tok}"
        if not greedy_setting(*sets[b]):
            assert got[1][b] == st, f"row {b}: generator state"
        assert got[-1][b] == b
        r64 = want.astype(np.float64)
        lse = np.log(np.exp(r64 - r64.max()).sum()) + r64.max()
        assert abs(float(got[5][b][0]) - (r64[tok] - lse)) <= merge_tol(r64[tok] - lse, lse), f"row {b}: logprob"
        assert np.array_equal(got[6][b][0], host_topk(want[None], 5)[0]), f"row {b}: top ids"
    assert int(got[0][0][0]) == int(np.argmax(mask_row(plain_row0, allowed[0])))


# ---- 4 / 5. sampler and tile edges, top-k past the allowed set
def test_sampler_and_tile_edges():
    spec = replace(TINY1, vocab_size=5000)  # 40 tiles, the last one 8 entries
    V = spec.vocab_size
    tensors = mg.generate(spec, 13, device="cuda")
    rows = np.zeros((7, V), bool)
    rows[0, 777] = True                       # forced
    rows[1, [5, 4321]] = True                 # two, in distant tiles
    rows[2, ::2] = True                       # 2500 survivors at minp 0: the chunk path
    rows[3, 1280:1408] = True                 # one whole tile
    rows[4, 4992:5000] = True                 # only the partial last tile
    rows[5, [3, 2600, 4999]] = True           # many fully masked tiles
    rows[6, 1300:1303] = True                 # fewer than k allowed, greedy
    aut = edge_automaton(V, rows)
    n = len(rows)
    prompts = prompts_of(V, [9, 17, 3, 30, 1, 12, 5], start=21)
    sets = [(1.0, 0.0), (2.0, 0.0), (2.0, 0.0), (1.0, 0.0), (1.0, 0.05), (2.0, 0.0), (0.0, 0.1)]
    seeds = SEEDS[:n]
    k = 5
    with lib.DeviceModel(spec, tensors, seq_len=1024) as dm:
        plain = qpen(dm, None, None, prompts, [1] * n, sets, seeds, [], 16, k=k)
        raw = dm.read_state("pf_logits").reshape(-1, V).copy()
        got = qcon(dm, None, None, prompts, [3] * n, sets, seeds, [], 16, k=k, automaton=aut, start=list(range(n)))
        out = dm.read_state("pf_logits").reshape(-1, V)
    assert got[2] == 1 and plain[2] == 1 and out.shape[0] == n
    for b in range(n):
        want = mask_row(raw[b], rows[b])
        assert same_bits(out[b], want), f"state {b}: masked row"
        tok, st = pick(want, *sets[b], seeds[b])
        assert [int(x) for x in got[0][b]] == [tok], f"state {b}: tokens {got[0][b]}, want [{tok}] (then the final state retires it)"
        assert got[-1][b] == n, f"state {b}: out_state {got[-1][b]}"
        if not greedy_setting(*sets[b]):
            assert got[1][b] == st, f"state {b}: one draw"
        n_allowed = int(rows[b].sum())
        ids, tlp = got[6][b][0], got[7][b][0]
        m = min(k, n_allowed)
        assert np.array_equal(ids[:m], host_topk(want[None], k)[0][:m]), f"state {b}: allowed top ids"
        assert (ids[m:] == -1).all() and (tlp[m:] == -np.inf).all(), f"state {b}: ranks past the allowed set {ids}, {tlp}"
        assert np.isfinite(tlp[:m]).all() and np.isfinite(got[5][b][0])
    assert got[0][0][0] == 777


def test_flat_sampling_never_emits_a_masked_token():
    spec = replace(TINY1, vocab_size=3000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 19, device="cuda")
    allowed = np.zeros(V, bool)
    allowed[1::2] = True
    aut = loop_automaton(V, [allowed])
    nreq = 64
    prompts = prompts_of(V, [[9, 1, 4, 30][i % 4] for i in range(nreq)], start=2)
    with lib.DeviceModel(spec, tensors, seq_len=2048) as dm:
        seeds = [(SEEDS[i % len(SEEDS)] + i) % (1 << 64) for i in range(nreq)]
        got = qcon(dm, None, None, prompts, [8] * nreq, [(2.0, 0.0)] * nreq, seeds, [], 16, automaton=aut, start=[0] * nreq)
    assert got[2] == 1
    toks = np.concatenate(got[0])
    assert len(toks) == 8 * nreq and allowed[toks].all(), f"masked tokens emitted: {toks[~allowed[toks]]}"


# ---- 6. guided_choice
def choice_seqs(V, rng):
    """Nine random token sequences of 1 .. 6 ids and two that share a first token with the last one; no proper prefixes."""
    seqs = [[int(t) for t in rng.choice(V, size=1 + j % 6, replace=False)] for j in range(9)]
    seqs += [[seqs[-1][0], 7, 8], [seqs[-1][0], 7, 9]]
    return [q for q in seqs if not any(len(o) > len(q) and o[:len(q)] == q for o in seqs)]


@pytest.mark.parametrize("max_rows", [1, 4, 16])
def test_choices(max_rows):
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 31, device="cuda")
    rng = np.random.default_rng(11)
    nreq = 40
    seqs = choice_seqs(V, rng)
    aut = TokenAutomaton.choices(seqs, V)
    prompts = prompts_of(V, [[9, 1, 40, 2, 17][i % 5] for i in range(nreq)], start=5)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    kind = ["free", "free-pen", "choice", "choice-pen"]
    start = [0 if kind[i % 4].startswith("choice") else -1 for i in range(nreq)]
    max_new = [[7, 3, 12][i % 3] if start[i] < 0 else 6 + i % 5 for i in range(nreq)]
    pen = mixed_pen(V, nreq, [i for i in range(nreq) if kind[i % 4].endswith("pen")])
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        free = qpen(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, k=3, **pen)
        got = qcon(dm, None, None, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, k=3, automaton=aut, start=start, **pen)
        assert got[2] == 1
        assert_same(got[:-1], free, f"r{max_rows} unconstrained", [i for i in range(nreq) if start[i] < 0])
        chosen = set()
        for i in range(nreq):
            if start[i] < 0:
                assert got[-1][i] == -1
                continue
            t = [int(x) for x in got[0][i]]
            assert t in seqs, f"request {i}: {t} is not a choice"
            s = 0
            for x in t:
                s = aut.next(s, x)
            assert got[-1][i] == s and aut.final[s], f"request {i}: out_state {got[-1][i]}"
            chosen.add(tuple(t))
            assert np.isfinite(got[5][i]).all() and (got[5][i] <= 0).all()
        assert len(chosen) > 1, "every constrained request chose the same sequence"
        # each step of the greedy constrained requests against the prompt pass, processed and masked
        for i in [i for i in range(nreq) if start[i] >= 0 and greedy_setting(*sets[i])][:3]:
            s = 0
            for j, tok in enumerate(int(x) for x in got[0][i]):
                seq = np.concatenate([prompts[i], got[0][i][:j]]).astype(np.int32)
                qpen(dm, None, None, [seq, seq], [1, 1], [(1.0, 0.1)] * 2, SEEDS[:2], [], 2, k=0)
                raw = dm.read_state("pf_logits").reshape(-1, V)[0].copy()
                seen, c, bv = host_state(V, prompts[i], got[0][i][:j], pen["logit_bias"][i])
                row = mask_row(process(raw, seen, c, pen["presence"][i], pen["frequency"][i], pen["repetition"][i], bv), np.isin(np.arange(V), aut.allowed(s)))
                tol = 2 * TOL_SIGMA * float(raw.std()) * max(1.0, 1.0 / pen["repetition"][i])
                fin = np.isfinite(row)
                top2 = np.sort(row[fin])[-2:]
                if len(top2) < 2 or top2[1] - top2[0] > 2 * tol:
                    assert tok == int(np.argmax(row)), f"request {i} step {j}: not the clear allowed argmax"
                r64 = row[fin].astype(np.float64)
                lse = np.log(np.exp(r64 - r64.max()).sum()) + r64.max()
                assert abs(float(got[5][i][j]) - (float(row[tok]) - lse)) <= 4 * tol + 1e-5, f"request {i} step {j}: logprob"
                s = aut.next(s, tok)
            assert aut.final[s] and s == got[-1][i]


# ---- 7. independence of the other requests, the schedule, the cache size and history
def test_outputs_do_not_depend_on_schedule_or_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    V = spec.vocab_size
    tensors = mg.generate(spec, 23, device="cuda")
    rng = np.random.default_rng(5)
    k = 3
    contexts = prompts_of(V, [300, 129], start=61)
    nreq = 40
    ctx_of = [[-1, 0, 1, 0][i % 4] for i in range(nreq)]
    lens = [[9, 1, 40, 2, 17][i % 5] for i in range(nreq)]
    prompts = prompts_of(V, lens, start=3)
    max_new = [[13, 1, 25, 7, 0][(3 * i + 1) % 5] for i in range(nreq)]
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    pen = mixed_pen(V, nreq, [i for i in range(nreq) if i % 4 == 1])
    # a loop over three states with different allowed sets, and a choice trie: states differ from step to step
    allow = rng.random((3, V)) < 0.2
    aut = TokenAutomaton(V, allow, [1, 2, 0], None)
    start = [[-1, 0, 1, 2][i % 4] for i in range(nreq)]
    clen = [len(contexts[c]) if c >= 0 else 0 for c in ctx_of]
    tight = max(ceil8(c) + ceil8(n - 1) + m for c, n, m in zip(clen, lens, max_new)) + 16
    runs = {}
    for seq_len in (4096, tight):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            for max_rows in ((1, 4, 16) if seq_len == 4096 else (16,)):
                runs[(seq_len, max_rows)] = qcon(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], max_rows, k=k, automaton=aut,
                                                 start=start, **pen)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        alone = {}
        for i in (1, 2, 3, 5, 6, 9, 10):
            one = {key: [v[i]] for key, v in pen.items()}
            alone[i] = qcon(dm, [contexts[ctx_of[i]]] if ctx_of[i] >= 0 else None, [0] if ctx_of[i] >= 0 else None, [prompts[i]], [max_new[i]], [sets[i]],
                            [SEEDS[i]], [], 16, k=k, automaton=aut, start=[start[i]], **one)
        other = prompts_of(V, [700, 33, 2], start=50)
        qcon(dm, [other[0]], [0, 0, -1], other, [60, 5, 30], [(1.1, 0.0)] * 3, SEEDS[20:23], [], 2, k=20,
             automaton=TokenAutomaton.choices([[1, 2, 3], [4]], V), start=[0, -1, 0])
        dm.poison(0)
        runs["dirty"] = qcon(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:nreq], [], 16, k=k, automaton=aut, start=start, **pen)
    ref = runs[(4096, 16)]
    assert ref[2] == 1 and all(len(t) == m for t, m in zip(ref[0], max_new))
    for i in range(nreq):
        s = start[i]
        for t in ref[0][i]:
            assert s < 0 or allow[s, int(t)], f"request {i}: a masked token"
            s = s if s < 0 else aut.next(s, int(t))
        assert ref[-1][i] == s
    for key, got in runs.items():
        assert got[2] == 1
        assert_same(got[:-1], ref[:-1], str(key))
        assert got[-1] == ref[-1], str(key)
    for i, got in alone.items():
        assert_same(got[:-1], tuple([x[i]] if isinstance(x, list) else x for x in ref[:-1]), f"request {i} alone", [0])
        assert got[-1] == [ref[-1][i]]


# ---- 8. the fallback
@pytest.mark.parametrize("name,seq_len,lens,max_new", [("tiny-moe", None, [6, 1, 12], [9, 0, 5]), ("pf-tiny", 64, [21, 50, 11], [8, 20, 3])])
def test_fallback_is_a_host_replay(name, seq_len, lens, max_new):
    spec = mg.SPECS[name]
    V = spec.vocab_size
    tensors = mg.generate(spec, 45)
    k = 3
    rng = np.random.default_rng(2)
    contexts = prompts_of(V, [4], start=8)
    ctx_of = [0, -1, 0]
    prompts = prompts_of(V, lens, start=1)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    cat = [concat(contexts, c, p) for c, p in zip(ctx_of, prompts)]
    pen = dict(presence=[0.5, 0.0, 0.0], frequency=[0.3, 0.0, 0.0], repetition=[1.2, 1.0, 1.0], logit_bias=[{3: -2.0}, None, None])
    allow = rng.random((2, V)) < 0.1
    allow[1, :] = False
    allow[1, [2, 5]] = True  # fewer than k
    aut = TokenAutomaton(V, allow, [1, 0], None)
    start = [0, -1, 1]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        plain = qpen(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k=k, **pen)
        got = qcon(dm, contexts, ctx_of, prompts, max_new, sets, SEEDS[:3], [], 16, k=k, automaton=aut, start=start, **pen)
        assert got[2] == 0 and plain[2] == 0
        assert_same(got[:-1], plain, f"{name} unconstrained request", [1])
        for i in (0, 2):
            p, s, st = cat[i], SEEDS[i], start[i]
            dm.prefill(p[:-1], 0)
            tok = int(p[-1])
            gen = []
            for j in range(max_new[i]):
                dm.forward_sample(tok, len(p) - 1 + j, 0.0, 0.0, 1)
                seen, c, bv = host_state(V, p, gen, pen["logit_bias"][i])
                row = mask_row(process(dm.device_logits(), seen, c, pen["presence"][i], pen["frequency"][i], pen["repetition"][i], bv), allow[st])
                tok, s = pick(row, *sets[i], s)
                assert tok == got[0][i][j], f"{name}: request {i} step {j}"
                gen.append(tok)
                fin = np.isfinite(row)
                r64 = row[fin].astype(np.float64)
                lse = np.log(np.exp(r64 - r64.max()).sum()) + r64.max()
                assert abs(float(got[5][i][j]) - (float(row[tok]) - lse)) <= 1e-6 * max(1.0, abs(float(row[tok]) - lse)), f"{name}: request {i} step {j} logprob"
                m = min(k, int(fin.sum()))
                assert np.array_equal(got[6][i][j][:m], host_topk(row[None], k)[0][:m]) and (got[6][i][j][m:] == -1).all(), f"{name}: request {i} step {j} top ids"
                st = aut.next(st, tok)
            assert len(got[0][i]) == max_new[i] and got[-1][i] == st, f"{name}: request {i} length / out_state"
            assert max_new[i] == 0 or greedy_setting(*sets[i]) or got[1][i] == s, f"{name}: request {i} state"


# ---- 9. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    V = spec.vocab_size
    good = [np.asarray([1, 2, 3], np.int32)]
    aut = TokenAutomaton.choices([[4, 5], [6]], V)
    fin = aut.next(0, 6)
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(contexts=None, ctx_of=None, prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4, rng_states=[1],
                  automaton=aut, start=[0], presence=[0.5], logit_bias=[{3: 1.0}], k=2)
        bad = [dict(start=[aut.n_states]), dict(start=[-2]), dict(start=[0, 0]), dict(start=[0.0]), dict(start=[True]),
               dict(automaton=None),                                  # a start >= 0 with no automaton
               dict(automaton="trie"), dict(automaton=TokenAutomaton.choices([[1]], V + 1)),
               dict(start=[fin]),                                     # starts in a final state
               dict(k=-1), dict(presence=[np.nan]), dict(logit_bias=[{V: 1.0}]), dict(max_new=[-1]), dict(max_rows=17), dict(prompts=[[3, V]])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue_constrained(**{**ok, **b})
        got = dm.decode_sample_queue_constrained(**{**ok, "max_new": [0], "start": [fin]})  # nothing to generate: a final start is fine
        assert len(got[0][0]) == 0 and got[-1] == [fin] and got[2:5] == (1, 0, 0)
        got = dm.decode_sample_queue_constrained(**{**ok, "k": None})
        assert len(got) == 6 and got[2] == 1 and [int(t) for t in got[0][0]] in ([4, 5], [6]) and got[-1] == [fin]
