"""calm_b200_decode_beam: beam search over one prompt, every step one short block whose rows are the live beams, each
reading its generated keys through its ancestry (k_sn_attn<.., BEAM>), the classifier's top-K lists walked by k_bm_select.

1. Replay: tests/beam_ref.py over the call's own candidate lists (read_state) gives its outputs and ancestry bit for bit.
2. The candidates are the model's: each row's lists against float64 logits teacher-forced along the row's history.
3. The last step's attention of every row against float64 over its keys gathered through the ancestry.
4. num_beams 1 is the greedy stream of decode_sample_n, with the queue's log-probabilities.
5. The prompt's slots and every slot past the call's are left as they were.  6. No result depends on history.
7. MoE and calls past seq_len are not served and touch no output.  8. Bad arguments raise."""
import ctypes as C
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_ref as br  # noqa: E402
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_stages_gpu import L8B, layer_cache, make_model, report  # noqa: E402
from test_verify_gpu import TINY1  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu


def trace(dm, B, K, max_new):
    """The last call's per-step lists [(ids, lps)] and the ancestry its last step read."""
    ids = dm.read_state("beam_ids").reshape(-1, B, K).astype(np.int64)
    lps = dm.read_state("beam_logprobs").reshape(-1, B, K)
    anc = dm.read_state("beam_anc").reshape(B, max_new).astype(np.int64)
    return list(zip(ids, lps)), anc


def beam(dm, token0, pos0, max_new, B, stop=(), lpen=1.0, early=0, R=None):
    hyps, served, steps = dm.decode_beam(token0, pos0, max_new, B, stop, lpen, early, R)
    assert served == 1
    K = br.n_candidates(B, len(stop))
    lists, anc = trace(dm, B, K, max_new)
    assert len(lists) == steps
    return hyps, steps, lists, anc


def check_replay(hyps, steps, lists, anc, B, stop, lpen, early, max_new, R, label):
    ref = br.replay(lists, B, stop, lpen, early, max_new)
    assert steps == ref["steps"], f"{label}: {steps} steps, the rule {ref['steps']}"
    assert len(hyps) == R
    for r, ((t, lp, s), (rt, rlp, rs)) in enumerate(zip(hyps, ref["hyps"])):
        assert np.array_equal(t, rt), f"{label}: hypothesis {r}: {t.tolist()} vs the rule's {rt.tolist()}"
        assert np.array_equal(lp.view(np.uint32), rlp.view(np.uint32)), f"{label}: hypothesis {r}'s log-probabilities"
        assert np.float32(s).view(np.uint32) == rs.view(np.uint32), f"{label}: hypothesis {r}: score {s} vs {rs}"
    rows = 1 if steps == 1 else B
    assert np.array_equal(anc[:rows, :steps], ref["anc"][:rows, :steps]), f"{label}: ancestry differs from the rule's"
    return ref


def frequent(lists, n):
    """n ids that rank high in many rows of a trace: stop ids the search will meet."""
    ids = np.concatenate([x[:, :3].reshape(-1) for x, _ in lists])
    ids = ids[ids >= 0]
    vals, counts = np.unique(ids, return_counts=True)
    return [int(v) for v in vals[np.argsort(-counts, kind="stable")][:n]]


# ---- 1. replay: (spec, kvbits, B, n_stop, early, R, length_penalty, pos0, max_new)
REPLAY = {
    "tiny B1 no stop": (TINY1, 16, 1, 0, 0, 1, 1.0, 37, 12),
    "tiny B3 4 stops": (TINY1, 16, 3, 4, 0, 2, 1.0, 130, 20),
    "tiny B3 1 stop early lp2 pos0 0": (TINY1, 8, 3, 1, 1, 3, 2.0, 0, 16),
    "tiny B8 1 stop lp0": (TINY1, 16, 8, 1, 0, 5, 0.0, 256, 10),
    "tiny B10 no stop": (TINY1, 16, 10, 0, 0, 10, 1.0, 60, 9),
    "tiny B1 4 stops early": (TINY1, 16, 1, 4, 1, 1, 1.0, 90, 24),
    "llama3-8b B10 1 stop early": (L8B, 16, 10, 1, 1, 4, 1.0, 300, 6),
    "llama3-8b B3 4 stops lp0.5": (L8B, 8, 3, 4, 0, 1, 0.5, 127, 8),
}


@pytest.mark.parametrize("case", sorted(REPLAY))
def test_replay_of_the_candidate_lists_gives_every_output(case):
    spec, kvbits, B, n_stop, early, R, lpen, pos0, max_new = REPLAY[case]
    tensors = mg.generate(spec, 11, device="cuda")
    with lib.DeviceModel(spec, tensors, seq_len=1024, kvbits=kvbits) as dm:
        dm.fill_kv(pos0, seed=3)
        _, _, lists, _ = beam(dm, 5, pos0, max_new, B)
        stop = frequent(lists, n_stop)
        hyps, steps, lists, anc = beam(dm, 5, pos0, max_new, B, stop, lpen, early, R)
    ref = check_replay(hyps, steps, lists, anc, B, stop, lpen, early, max_new, R, case)
    for t, lp, _ in hyps:
        assert len(t) <= max_new and (len(t) == max_new or t[-1] in stop)
    for r, (t, lp, _) in enumerate(hyps):
        assert br.fsum(lp) == ref["raw"][r], f"{case}: hypothesis {r}'s log-probabilities do not sum to its raw sum"


# ---- 2. the candidates are the model's
def test_candidates_are_the_float64_models():
    spec, B, pos0, max_new = TINY1, 3, 70, 6
    stop = []
    tensors, w = make_model(spec, 9)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=16) as dm:
        dm.fill_kv(pos0, seed=4)
        hyps, steps, lists, _ = beam(dm, 7, pos0, max_new, B, stop)
        keys, values = layer_cache(dm, spec)
    K = br.n_candidates(B, 0)
    ref = br.replay(lists, B, stop, 1.0, 0, max_new)
    worst = 0.0
    for j in range(steps):
        for b, hist in enumerate(ref["beams"][j]):
            cache = sr.Cache(spec, 512, 16)
            cache.k[0, :, :pos0], cache.v[0, :, :pos0] = keys[:, :pos0], values[:, :pos0]
            for i, tok in enumerate([7] + hist):
                logits = sr.forward(w, cache, tok, pos0 + i)[0]
            sigma = float(logits.std())
            lp64 = logits - (logits.max() + np.log(np.exp(logits - logits.max()).sum()))
            ids, lps = lists[j][0][b], lists[j][1][b]
            tol = 2 * 2 * TOL_SIGMA * sigma  # a log-probability moves by at most twice its logits' error
            err = np.abs(lps - lp64[ids])
            worst = max(worst, float(err.max() / tol))
            assert (err <= tol).all(), f"step {j} row {b}: lp {lps[np.argmax(err)]} vs float64 {lp64[ids][np.argmax(err)]}"
            order = np.lexsort((np.arange(len(logits)), -logits))
            srt = logits[order]
            for r in range(K):
                gap = min(srt[r - 1] - srt[r] if r else np.inf, srt[r] - srt[r + 1])
                if gap > 2 * TOL_SIGMA * sigma:
                    assert ids[r] == order[r], f"step {j} row {b} rank {r}: id {ids[r]} vs float64 {order[r]}"
    print(f"  beam candidates: worst lp error {worst:.2f} of the bound")


# ---- 3. the last step's attention through the ancestry: (spec, kvbits, B, pos0, max_new)
ATTN = {
    "llama3-8b B4 prompt ends inside a chunk": (L8B, 16, 4, 300, 5),
    "llama3-8b e5m2 B3 prompt on a chunk edge": (L8B, 8, 3, 256, 4),
    "tiny B5 pos0 0": (TINY1, 16, 5, 0, 9),
    "tiny kv_mul1 B10 own keys cross a chunk edge": (replace(TINY1, n_kv_heads=4), 16, 10, 120, 14),
    "tiny-hd128 B2 pos0 127": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 8, 2, 127, 7),
}


@pytest.mark.parametrize("case", sorted(ATTN))
def test_last_step_attention_reads_each_rows_ancestry(case, capfd):
    spec, kvbits, B, pos0, max_new = ATTN[case]
    tensors, w = make_model(spec, 4)
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    with lib.DeviceModel(spec, tensors, seq_len=1024, kvbits=kvbits) as dm, capfd.disabled():
        dm.fill_kv(pos0, seed=6)
        hyps, steps, lists, anc = beam(dm, 3, pos0, max_new, B)
        assert steps == max_new
        Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:B]
        A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:B]
        keys, values = layer_cache(dm, spec)
    j = steps - 1
    a_ref, vmax = [], []
    for b in range(B):
        slots = np.concatenate([np.arange(pos0), pos0 + np.arange(j + 1) * B + anc[b, :j + 1]])
        K, V = keys[:, slots], values[:, slots]
        a_ref.append(sr.attention(spec, Q[b], K, V, pos0 + j + 1))
        vmax.append(np.repeat(np.abs(V).max((1, 2)), kv_mul * hd))
    assert len({tuple(anc[b, :j + 1]) for b in range(B)}) > 1 or B == 1 or max_new == 1, f"{case}: no two rows differ in ancestry"
    report(f"beam {case}", "A", "k_sn_attn BEAM", A, np.stack(a_ref), np.stack(vmax), lambda i: f"row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")


# ---- 4. one beam is greedy
def test_one_beam_is_the_greedy_stream():
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 46, device="cuda")
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    P, N = len(prompt), 24
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        greedy, _, served = dm.decode_sample_n(int(prompt[-1]), P - 1, N, 0.0, 0.1, [1])
        assert served == 1
        greedy = greedy[0]
        free, steps, _, _ = beam(dm, int(prompt[-1]), P - 1, N, 1)
        stop = [int(greedy[N // 2])]
        cut = int(np.argmax(greedy == stop[0])) + 1
        early, esteps, _, _ = beam(dm, int(prompt[-1]), P - 1, N, 1, stop, 1.0, 1)
        q = dm.decode_sample_queue_logprobs(None, None, [prompt], [N], [0.0], [0.1], [], 1, [1], k=2)
    assert q[2] == 1 and np.array_equal(q[0][0], greedy)
    assert steps == N and np.array_equal(free[0][0], greedy), f"{free[0][0].tolist()} vs greedy {greedy.tolist()}"
    assert np.array_equal(free[0][1].view(np.uint32), q[5][0].view(np.uint32))
    assert esteps == cut and np.array_equal(early[0][0], greedy[:cut])
    assert np.array_equal(early[0][1].view(np.uint32), q[5][0][:cut].view(np.uint32))
    assert np.float32(free[0][2]) == np.float32(br.fsum(q[5][0]) / np.float32(N))


# ---- 5. the cache
def test_prompt_and_later_slots_are_untouched():
    spec, B, pos0, max_new, seq_len = replace(mg.SPECS["pf-tiny"], n_layers=2), 4, 45, 9, 256
    with lib.DeviceModel(spec, mg.generate(spec, 7, device="cuda"), seq_len=seq_len) as dm:
        dm.fill_kv(seq_len, seed=8)
        before = [dm.read_state(x, l).copy() for l in range(spec.n_layers) for x in ("keys", "values")]
        beam(dm, 2, pos0, max_new, B, [3], 1.0, 0)
        after = [dm.read_state(x, l) for l in range(spec.n_layers) for x in ("keys", "values")]
    shape = (spec.n_kv_heads, seq_len, spec.head_dim)
    for i, (x, y) in enumerate(zip(before, after)):
        x, y = x.reshape(shape), y.reshape(shape)
        assert np.array_equal(x[:, :pos0].view(np.uint32), y[:, :pos0].view(np.uint32)), f"item {i}: a prompt slot changed"
        end = pos0 + B * max_new
        assert np.array_equal(x[:, end:].view(np.uint32), y[:, end:].view(np.uint32)), f"item {i}: a slot past {end} changed"
        assert not np.array_equal(x[:, pos0:end], y[:, pos0:end]), f"item {i}: the call wrote nothing"


# ---- 6. history
def beam_runs(dm, pos0):
    out = []
    for B, stop, early, max_new in ((3, [4, 9], 0, 11), (10, [], 0, 5), (2, [1, 2, 3, 4], 1, 14)):
        hyps, steps, lists, anc = beam(dm, 6, pos0, max_new, B, stop, 1.0, early)
        out += [np.asarray(steps), np.concatenate([np.asarray(x[0]) for x in lists]), np.concatenate([x[1] for x in lists]), anc[:, :steps],
                dm.read_state("pf_att").reshape(-1, dm.spec.q_dim)[:B]]
        for t, lp, s in hyps:
            out += [t, lp, np.asarray([s], np.float32)]
    return out


def test_decode_beam_does_not_depend_on_history():
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    tensors = mg.generate(spec, 31, device="cuda")
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 141, start=4), np.int32)
    other = np.asarray(mg.teacher_tokens(spec.vocab_size, 300, start=9), np.int32)
    pos0 = len(prompt) - 1
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        fresh = beam_runs(dm, pos0)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        dm.prefill(other[:250], 0)
        dm.decode_beam(int(other[250]), 250, 25, 10)  # a longer ancestry than the runs need
        dm.decode_sample_n(int(other[250]), 250, 16, 0.8, 0.02, list(range(1, 17)))
        assert dm.prefill(prompt[:-1], 0) == 1
        dm.poison(pos0)
        dirty = beam_runs(dm, pos0)
    for i, (f, d) in enumerate(zip(fresh, dirty)):
        if f.dtype.kind == "f":
            assert np.isfinite(f[f != -np.inf]).all(), f"item {i} not finite"
        assert np.array_equal(np.asarray(d), np.asarray(f)), f"item {i}: after another history and poisoning the results changed"


# ---- 7. not served
def raw_call(dm, token0, pos0, max_new, B, R):
    ip, fp = C.POINTER(C.c_int), C.POINTER(C.c_float)
    toks, lps = np.full(R * max_new, -7, np.int32), np.full(R * max_new, 7.5, np.float32)
    lens, scores, steps = np.full(R, -7, np.int32), np.full(R, 7.5, np.float32), C.c_int(-7)
    served = dm.lib.calm_b200_decode_beam(C.byref(dm.transformer), token0, pos0, max_new, B, None, 0, 1.0, 0, R, toks.ctypes.data_as(ip),
                                          lens.ctypes.data_as(ip), lps.ctypes.data_as(fp), scores.ctypes.data_as(fp), C.byref(steps))
    return served, steps.value, toks, lps, lens, scores


@pytest.mark.parametrize("name,seq_len,B,max_new,pos0", [("tiny-moe", None, 3, 5, 4), ("pf-tiny", 64, 4, 8, 40)])
def test_unserved_calls_return_0_and_touch_no_output(name, seq_len, B, max_new, pos0):
    spec = mg.SPECS[name]
    with lib.DeviceModel(spec, mg.generate(spec, 45), seq_len=seq_len) as dm:
        dm.fill_kv(pos0)
        served, steps, toks, lps, lens, scores = raw_call(dm, 1, pos0, max_new, B, 2)
        assert dm.decode_beam(1, pos0, max_new, B) == ([], 0, 0)
    assert served == 0 and steps == 0
    assert (toks == -7).all() and (lens == -7).all() and (lps == 7.5).all() and (scores == 7.5).all()


# ---- 8. bad arguments
def test_bad_arguments_raise():
    spec = mg.SPECS["pf-tiny"]
    with lib.DeviceModel(spec, mg.generate(spec, 1)) as dm:
        bad = [dict(num_beams=0), dict(num_beams=11), dict(num_beams=2.0), dict(num_beams=7, stop=[1, 2]),  # K = 21
               dict(num_beams=1, stop=list(range(20))), dict(num_return=0), dict(num_beams=2, num_return=3),
               dict(max_new=-1), dict(stop=[-1]), dict(stop=[spec.vocab_size]), dict(token0=-1), dict(token0=spec.vocab_size), dict(pos0=-1),
               dict(length_penalty=float("nan")), dict(length_penalty=float("inf")), dict(early_stopping=2)]
        for kw in bad:
            args = dict(token0=1, pos0=0, max_new=4, num_beams=2)
            args.update(kw)
            with pytest.raises(ValueError):
                dm.decode_beam(**args)
        assert dm.decode_beam(1, 0, 0, 3) == ([], 1, 0)  # nothing wanted
