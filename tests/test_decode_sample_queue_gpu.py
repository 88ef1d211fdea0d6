"""calm_b200_decode_sample_queue: a queue of requests, at most max_rows in flight, each with its own prompt, max_new,
temperature / min-p and generator, shared stop tokens, and new requests admitted as rows finish.

1. Every request equals decode_sample_batch over its prompt alone with n_tokens = its out_len: tokens, final state and
   out_len, bit for bit, across shapes, cache types, max_rows, prompt lengths, max_new, mixed settings and stop tokens.
2. The same requests give the same outputs under max_rows 1 / 4 / 16, at a seq_len tight enough that admission waits
   for space and reuses freed extents, and on an engine that ran another call and was poisoned.
3. The step count is the documented policy's, simulated here (continuous admission, not waves).
4. The last step's stages against float64, with rows at different own-step counts: Q, each row's new cache entries at
   the slots the documented placement gives, attention over each row's gathered keys, hidden and residual rows.
5. Fallback shapes give the forward_prefill_cuda + forward_sample loop cut at the stop, with steps 0.  6. Bad arguments raise."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from test_stages_gpu import L8B, V4K, check_entries, layer_cache, make_model, pf_tol, report  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402
from test_verify_sample_gpu import DEFAULT, xs_advance  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

SEEDS = [(0x9E3779B97F4A7C15 * (i + 3) + 12345) % (1 << 64) for i in range(48)]
SETTINGS = [(1.0, 0.1), (0.0, 0.1), (1.3, 0.0), (0.8, 1.0), (0.7, 0.05)]  # (0, .) and (., 1) are greedy


def ceil8(x):
    return -(-x // 8) * 8


def greedy_setting(t, p):
    return t == 0.0 or p >= 1.0


class Slots:
    """First-fit over [0, seq_len), coalescing on release: include/calm_b200.h's placement."""

    def __init__(self, n):
        self.free = [(0, n)]

    def take(self, n, align):
        for k, (s, e) in enumerate(self.free):
            a = ceil8(s) if align == 8 else s
            if a + n <= e:
                pieces = [(x, y) for x, y in ((s, a), (a + n, e)) if x < y]
                self.free[k:k + 1] = pieces
                return a
        return -1

    def give(self, s, n):
        if n:
            out = []
            for x, y in sorted(self.free + [(s, s + n)]):
                if out and out[-1][1] == x:
                    out[-1] = (out[-1][0], y)
                else:
                    out.append((x, y))
            self.free = out

    def copy(self):
        c = Slots(0)
        c.free = list(self.free)
        return c


def place_round(slots, rs, lens, max_new):
    P = sum(ceil8(lens[i] - 1) for i in rs)
    s = slots.take(P, 8) if P else 0
    if s < 0:
        return None
    out = {}
    for i in rs:
        t = slots.take(max_new[i], 1)
        if t < 0:
            return None
        out[i] = (s, lens[i] - 1, t)
        s += ceil8(lens[i] - 1)
    return out


def simulate(lens, max_new, out_len, max_rows, seq_len):
    """The documented schedule given each request's out_len: (every step's rows [(request, own step)], placement, waited),
    waited = some admission found a free row but no room for the next request."""
    slots, place, live, done, steps, head, waited = Slots(seq_len), {}, [], {}, [], 0, False
    n = len(lens)
    while True:
        rnd, rp, after = [], {}, slots
        while head < n and len(live) + len(rnd) < max_rows:
            if max_new[head] == 0:
                head += 1
                continue
            a = slots.copy()
            tp = place_round(a, rnd + [head], lens, max_new)
            if tp is None:
                waited = True
                break
            rnd, rp, after, head = rnd + [head], tp, a, head + 1
        if not live and not rnd:
            break
        slots = after
        place.update(rp)
        live += rnd
        steps.append([(i, done.get(i, 0)) for i in live])
        keep = []
        for i in live:
            done[i] = done.get(i, 0) + 1
            if done[i] < out_len[i]:
                keep.append(i)
            else:
                s, L, t = place[i]
                slots.give(s, ceil8(L))
                slots.give(t, max_new[i])
        live = keep
    return steps, place, waited


def prompts_of(vocab, lens, start=0):
    return [np.asarray(mg.teacher_tokens(vocab, n, start=start + 31 * b), np.int32) for b, n in enumerate(lens)]


def requests(vocab, nreq, lens, max_new, start=0):
    lens = [lens[i % len(lens)] for i in range(nreq)]
    return (prompts_of(vocab, lens, start), [max_new[(3 * i + 1) % len(max_new)] for i in range(nreq)],
            [SETTINGS[i % len(SETTINGS)] for i in range(nreq)], SEEDS[:nreq])


def lone(dm, prompt, n, t, p, seed):
    toks, states, served = dm.decode_sample_batch([prompt], n, t, p, [seed])
    assert served == 1
    return toks[0], states[0]


def queue(dm, prompts, max_new, sets, seeds, stop, max_rows):
    return dm.decode_sample_queue(prompts, max_new, [t for t, _ in sets], [p for _, p in sets], stop, max_rows, seeds)


# ---- 1. every request equals decode_sample_batch over its prompt alone
HD128 = replace(mg.SPECS["pf-tiny-hd128"], n_layers=1)
ALONE = {  # (spec, kvbits, max_rows, nreq, prompt lengths, seq_len)
    "pf-tiny fp8 r16 n40": (mg.SPECS["pf-tiny"], 16, 16, 40, [1, 2, 9, 129, 300], 4096),
    "pf-tiny gf4 e5m2 r3 n24": (replace(mg.SPECS["pf-tiny"], dtype="gf4"), 8, 3, 24, [300, 1, 2100, 9, 129, 2], 4096),
    "pf-tiny fp16 r1 n12": (replace(TINY1, dtype="fp16"), 16, 1, 12, [9, 129, 1, 2], 2048),
    "pf-tiny-hd128 bias e5m2 r16 n20": (HD128, 8, 16, 20, [129, 2, 300, 1, 9], 4096),
    "llama3-8b widths r16 n20": (L8B, 16, 16, 20, [300, 1, 2100, 9, 129, 2], 4096),
    "llama3-70b widths e5m2 r3 n12": (replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K), 8, 3, 12, [129, 9, 1], 2048),
}


@pytest.mark.parametrize("case", sorted(ALONE))
def test_each_request_is_itself_alone(case):
    spec, kvbits, max_rows, nreq, lens, seq_len = ALONE[case]
    tensors = mg.generate(spec, 17, device="cuda")
    prompts, max_new, sets, seeds = requests(spec.vocab_size, nreq, lens, [0, 1, 7, 40])
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        full = [lone(dm, p, m, *s, seed) if m else (np.zeros(0, np.int32), seed) for p, m, s, seed in zip(prompts, max_new, sets, seeds)]
        # stop ids that fire at known steps: step 0 of one request, the middle of another, the last allowed step of a third
        long = [i for i in range(nreq) if max_new[i] == 40]
        stop = [int(full[long[0]][0][0]), int(full[long[1]][0][20]), int(full[long[2]][0][39])]
        for stops in ([], stop):
            want_len = []
            for i in range(nreq):
                hit = [k for k, tok in enumerate(full[i][0]) if tok in stops]
                want_len.append(min(max_new[i], hit[0] + 1) if hit else max_new[i])
            toks, states, served, steps = queue(dm, prompts, max_new, sets, seeds, stops, max_rows)
            assert served == 1
            assert [len(x) for x in toks] == want_len, f"{case} stop {stops}: out_len"
            assert steps == len(simulate([len(p) for p in prompts], max_new, want_len, max_rows, seq_len)[0])
            for i in range(nreq):
                if want_len[i] < max_new[i]:  # the lone call with n_tokens = out_len
                    want = lone(dm, prompts[i], want_len[i], *sets[i], seeds[i]) if want_len[i] else (np.zeros(0, np.int32), seeds[i])
                else:
                    want = full[i]
                assert np.array_equal(toks[i], want[0]), f"{case} stop {stops}: request {i} tokens differ from the request alone"
                assert states[i] == want[1], f"{case} stop {stops}: request {i} state"
                if greedy_setting(*sets[i]):
                    assert states[i] == seeds[i]
                else:
                    assert states[i] == xs_advance(seeds[i], want_len[i])
            if stops:  # the stops fired where they were placed
                assert want_len[long[0]] == 1 and want_len[long[1]] <= 21 and want_len[long[2]] <= 40


# ---- 2. no dependence on schedule or history; 3. the step count is the policy's
def test_outputs_do_not_depend_on_schedule_or_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    tensors = mg.generate(spec, 23, device="cuda")
    prompts, max_new, sets, seeds = requests(spec.vocab_size, 18, [129, 9, 300, 1, 40, 2], [13, 1, 40, 7, 0, 25], start=3)
    lens = [len(p) for p in prompts]
    tight = max(ceil8(n - 1) + m for n, m in zip(lens, max_new))  # the largest request just fits an empty cache
    runs = {}
    for seq_len in (4096, tight):
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            for max_rows in (1, 4, 16):
                toks, states, served, steps = queue(dm, prompts, max_new, sets, seeds, [], max_rows)
                assert served == 1
                out_len = [len(x) for x in toks]
                assert out_len == max_new
                sched, place, waited = simulate(lens, max_new, out_len, max_rows, seq_len)
                assert steps == len(sched), f"seq_len {seq_len} max_rows {max_rows}: {steps} steps, the policy runs {len(sched)}"
                if seq_len == tight and max_rows == 16:
                    assert waited, "the tight cache never made admission wait"
                    order = sorted(place, key=lambda i: place[i][2])
                    assert order != sorted(order), "no freed extent was reused by a later request"
                runs[(seq_len, max_rows)] = (toks, states)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        other = prompts_of(spec.vocab_size, [700, 33, 2], start=50)
        queue(dm, other, [60, 5, 30], [(1.1, 0.0)] * 3, SEEDS[20:23], [], 2)
        dm.decode_sample_batch(other, 9, 0.9, 0.05, SEEDS[:3])
        dm.poison(0)
        runs["dirty"] = queue(dm, prompts, max_new, sets, seeds, [], 16)[:2]
    ref = runs[(4096, 16)]
    for k, (toks, states) in runs.items():
        assert states == ref[1], f"{k}: states differ"
        for i, (x, y) in enumerate(zip(toks, ref[0])):
            assert np.array_equal(x, y), f"{k}: request {i} differs"


def test_admission_is_continuous():
    spec = mg.SPECS["pf-tiny"]
    with lib.DeviceModel(spec, mg.generate(spec, 5), seq_len=1024) as dm:
        prompts = prompts_of(spec.vocab_size, [5, 9, 3, 12, 7], start=1)
        toks, _, served, steps = queue(dm, prompts, [1, 10, 1, 1, 1], [DEFAULT] * 5, SEEDS[:5], [], 2)
        assert served == 1 and [len(x) for x in toks] == [1, 10, 1, 1, 1]
        assert steps == 10, f"{steps} steps: waves of 2 would run 12, continuous admission 10"
        rng = np.random.default_rng(3)
        for max_rows in (1, 3, 7, 16):
            nreq = 30
            lens = [int(x) for x in rng.integers(1, 200, nreq)]
            max_new = [int(x) for x in rng.integers(0, 30, nreq)]
            prompts = prompts_of(spec.vocab_size, lens, start=9)
            toks, _, served, steps = queue(dm, prompts, max_new, [DEFAULT] * nreq, SEEDS[:nreq], [], max_rows)
            assert served == 1 and [len(x) for x in toks] == max_new
            assert steps == len(simulate(lens, max_new, max_new, max_rows, 1024)[0])


# ---- 4. the last step's stages against float64
STAGES = {  # (spec, kvbits, prompt lengths, max_new, max_rows): later requests shorter, so the last step holds several rows
    "llama3-8b fp8 kv_mul4": (L8B, 16, [301, 1, 130, 2101, 40, 9, 257], [29, 26, 23, 20, 17, 14, 11], 4),
    "llama3-8b fp8 kv_mul4 e5m2": (L8B, 8, [129, 9, 700, 1, 33], [23, 20, 17, 14, 11], 3),
    "pf-tiny hd64 kv_mul2": (TINY1, 16, [37, 1, 250, 129, 2, 64], [26, 23, 20, 17, 14, 11], 4),
}


@pytest.mark.parametrize("case", sorted(STAGES))
def test_last_step_every_stage(case, capfd):
    spec, kvbits, lens, max_new, max_rows = STAGES[case]
    nreq, seq_len = len(lens), 4096
    tensors, w = make_model(spec, 4)
    prompts = prompts_of(spec.vocab_size, lens, start=3)
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(nreq)]
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm, capfd.disabled():
        toks, _, served, steps = queue(dm, prompts, max_new, sets, SEEDS[:nreq], [], max_rows)
        sched, place, _ = simulate(lens, max_new, max_new, max_rows, seq_len)
        rows = sched[-1]
        n = len(rows)
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
        Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:n]
        A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:n]
        H = dm.read_state("pf_hb").reshape(-1, spec.hidden_dim)[:n]
        keys, values = layer_cache(dm, spec)
    assert served == 1 and steps == len(sched)
    assert n >= 2 and len({j for _, j in rows}) >= 2, f"{case}: the last step's rows {rows} are not at different own steps"
    label = f"sample_queue {case} kv{kvbits}"
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
        s, L, t = place[i]
        idx = np.concatenate([s + np.arange(L), t + np.arange(j + 1)])
        K, V = keys[:, idx], values[:, idx]
        a_ref.append(sr.attention(spec, Q[r], K, V, L + j + 1))
        vmax.append(np.repeat(np.abs(V).max((1, 2)), kv_mul * hd))
    report(label, "A", "k_sn_attn QUEUE", A, np.stack(a_ref), np.stack(vmax), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")
    x1 = sr.wo(w, 0, X0, A)
    h_ref = sr.ffn_up(w, 0, sr.ffn_input(w, 0, x1, xn))
    report(label, "H", "k_vf_gemm WO+UP", H, h_ref, np.abs(h_ref).max(), lambda i: f"row {i[0]} hidden row {i[1]}", "vf_hb", pf_tol(max(spec.dim, spec.q_dim)))
    x_ref = sr.ffn_down(w, 0, x1, H)
    report(label, "X", "k_vf_gemm DOWN", X, x_ref, np.abs(x_ref).max(), lambda i: f"row {i[0]} row {i[1]}", "vf_x", pf_tol(spec.hidden_dim))


# ---- 5. fallback
@pytest.mark.parametrize("name,seq_len,lens,max_new", [("tiny-moe", None, [6, 1, 12], [9, 0, 5]), ("pf-tiny", 64, [21, 50, 11], [8, 20, 3])])
def test_fallback_is_prefill_and_forward_sample_per_request(name, seq_len, lens, max_new):
    """A MoE model, and a served shape with a request whose ceil8(L) + max_new (56 + 20) passes seq_len."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    prompts = prompts_of(spec.vocab_size, lens, start=1)
    sets = [SETTINGS[i % len(SETTINGS)] for i in range(len(lens))]
    streams = []
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        for p, m, (t, mp), s in zip(prompts, max_new, sets, SEEDS):
            dm.prefill(p[:-1], 0)
            tok, out = int(p[-1]), []
            for k in range(m):
                tok, s = dm.forward_sample(tok, len(p) - 1 + k, t, mp, s)
                out.append(tok)
            streams.append(out)
    stop = [streams[0][2]]
    want, want_st = [], []
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        for p, m, (t, mp), s in zip(prompts, max_new, sets, SEEDS):
            dm.prefill(p[:-1], 0)
            tok, out = int(p[-1]), []
            while len(out) < m:
                tok, s = dm.forward_sample(tok, len(p) - 1 + len(out), t, mp, s)
                out.append(tok)
                if tok in stop:
                    break
            want.append(out), want_st.append(s)
        toks, states, served, steps = queue(dm, prompts, max_new, sets, SEEDS[:len(lens)], stop, 16)
    assert served == 0 and steps == 0
    assert [x.tolist() for x in toks] == want and states == want_st
    assert len(want[0]) <= 3


# ---- 6. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    good = [np.asarray([1, 2, 3], np.int32)]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        ok = dict(prompts=good, max_new=[4], temperature=[1.0], minp=[0.1], stop=[], max_rows=4, rng_states=[1])
        bad = [dict(prompts=None), dict(rng_states=None), dict(rng_states=5), dict(rng_states=[1, 2]), dict(rng_states=[-1]), dict(rng_states=[1 << 64]),
               dict(max_new=[-1]), dict(max_new=[2.5]), dict(max_new=[1, 2]), dict(temperature=[1.0, 1.0]), dict(minp=[]),
               dict(max_rows=0), dict(max_rows=17), dict(max_rows=2.0), dict(stop=[-1]), dict(stop=[spec.vocab_size]), dict(stop=[[1]]),
               dict(prompts=[np.zeros(0, np.int32)]), dict(prompts=[[-1, 2]]), dict(prompts=[[3, spec.vocab_size]]), dict(prompts=[[0.5]])]
        for b in bad:
            with pytest.raises(ValueError):
                dm.decode_sample_queue(**{**ok, **b})
        toks, states, served, steps = dm.decode_sample_queue(**{**ok, "max_new": [0]})  # nothing wanted: no draw
        assert len(toks[0]) == 0 and states == [1] and served == 1 and steps == 0
        toks, states, served, steps = dm.decode_sample_queue([], [], [], [], [], 4, [])
        assert toks == [] and states == [] and served == 1 and steps == 0
