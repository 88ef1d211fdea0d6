"""calm_b200_score_greedy, calm_b200_score_batch_greedy and calm_b200_score_context_greedy: the scoring calls that also
return the greedy token (the argmax of the logits, lowest index on ties) at every scored position.  On the tensor-core
pass it comes from the classifier's epilogue (k_pf_gemm PF_CLS_GREEDY: each tile's first maximum) and the merge
(k_pf_logprob<true>), whose log-softmax records are the same bits as the plain call's.

1. The stage against float64 from the device's own classifier input: logprobs equal score()'s bit for bit, the greedy
   token's float64 logit is within the GEMM bound of the maximum, and it is the float64 argmax wherever the top-2 margin
   exceeds that bound.
2. Exact ties, by construction: classifier rows with one nonzero weight give bit-identical logits whatever the order of
   accumulation, so the lowest index must win inside a lane, across a quad, across vocabulary tiles and merge lanes, and in
   a partial last tile; and through the decode path's host argmax.
3. The packed calls equal the lone call per sequence, bit for bit, in logprobs and greedy tokens.
4. Against calm_b200_forward_argmax: where the serial logits' top-2 margin exceeds the pass's tolerance, and exactly on the
   decode-path shapes.
5. Draft verification on a live cache reproduces a calm_b200_decode_greedy stream.
6. No result depends on what earlier calls left behind; repeated calls agree; empty calls write nothing."""
import ctypes as C
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from conftest import TOL_SIGMA  # noqa: E402
from test_score_context_gpu import layout  # noqa: E402
from test_score_gpu import STAGE, log_softmax_at  # noqa: E402
from test_stages_gpu import make_model, pf_tol  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL_LP = np.float32(-12345.5)
SENTINEL_G = np.int32(-7)
worst = {}


def top2(logits):
    """(first index of the maximum, margin between the largest and the second largest value) per row."""
    L = np.asarray(logits, np.float64)
    s = np.sort(L, axis=1)
    return L.argmax(1), s[:, -1] - s[:, -2]


# ---- 1. the stage, from the device's own input
@pytest.mark.parametrize("case", sorted(STAGE))
def test_greedy_stage_against_float64(case):
    spec, kvbits, n = STAGE[case]
    tensors, w = make_model(spec, 7)
    toks = mg.teacher_tokens(spec.vocab_size, n)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        plain, _ = dm.score(toks, 0)
        lp, greedy, served = dm.score_greedy(toks, 0)
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n - 1]
    assert served == 1, f"{case}: the tensor-core pass did not serve this shape"
    assert np.array_equal(lp, plain), f"{case}: logprobs differ from calm_b200_score's"
    xn = torch.as_tensor(sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, spec.norm_type != "rmsnorm"), device="cuda")
    W = w.classifier()
    logits = torch.empty((n - 1, spec.vocab_size), dtype=torch.float64, device="cuda")
    for r in range(0, W.shape[0], 16384):
        logits[:, r:r + 16384] = xn @ torch.as_tensor(W[r:r + 16384], device="cuda").to(torch.float64).T
    ref = logits.cpu().numpy()
    assert ((greedy >= 0) & (greedy < spec.vocab_size)).all(), f"{case}: a greedy token outside the vocabulary"
    bound = 2 * pf_tol(spec.dim) * np.abs(ref).max(1)
    best, margin = top2(ref)
    short = ref.max(1) - ref[np.arange(n - 1), greedy]
    share = short / bound
    i = int(np.argmax(share))
    clear = margin > bound
    worst[case] = float(share[i])
    print(f"\n  {case}: greedy logit below the float64 maximum by at most {short.max():.2e} = {share[i]:.2f} of its bound"
          f" (position {i}); {int((~clear).sum())} of {n - 1} positions have a top-2 margin inside the bound")
    assert (short <= bound).all(), f"{case}: position {i}: greedy {greedy[i]} is {short[i]:.3e} below the maximum (bound {bound[i]:.3e})"
    bad = np.nonzero(clear & (greedy != best))[0]
    assert len(bad) == 0, f"{case}: position {bad[0]}: greedy {greedy[bad[0]]} vs float64 argmax {best[bad[0]]} (margin {margin[bad[0]]:.3e})"


# ---- 2. exact ties
C_W = 1.0  # a power of two: c and c / 2 are exact in fp16, e5m2 and gf4 (a gf4 group's scale element decodes to itself)
K_COL = 5
# (vocabulary, name, family P, family N): rows of +c e_k and -c e_k; the lowest member of each family must win
TIES = {
    1000: [("one lane", [256 + 3, 256 + 11, 256 + 19, 256 + 2], [256 + 40, 256 + 41]),  # (j, e) ascending in one lane; + the neighbour lane
           ("quad", [384 + 14, 384 + 16, 384 + 20], [384 + 5, 384 + 9]),  # lowest member on a higher lane of its quad
           ("tiles", [128 * 5 + 7, 128 + 100, 128 * 6], [128 * 7 + 50, 128 * 4 + 3]),
           ("partial last tile", [999], [998, 900, 997])],
    4200: [("merge lanes", [31 * 128 + 5, 4096 + 2], [100, 4096 + 50]),  # tile 31 (lane 31) vs tile 32 (lane 0); tiles 0 and 32 on lane 0
           ("partial last tile", [4199, 4096 + 7], [4197, 2 * 128 + 1, 4096])],
}


def tie_model(spec, fam_p, fam_n, seed, k=K_COL):
    assert not set(fam_p) & set(fam_n)
    tensors = mg.generate(spec, seed)
    W = torch.zeros((spec.vocab_size, spec.dim), dtype=torch.float32)
    W[:, k] = torch.where(torch.arange(spec.vocab_size) % 2 == 0, C_W / 2, -C_W / 2)
    W[fam_p, k] = C_W
    W[fam_n, k] = -C_W
    tensors["model.output.weight"] = mg.quantize(W, spec.dtype)
    return tensors


def tie_check(greedy, xk, fam_p, fam_n, label):
    live = xk != 0
    assert (xk > 0).any() and (xk < 0).any(), f"{label}: x_k took one sign only: the test does not cover both families"
    want = np.where(xk > 0, min(fam_p), min(fam_n))
    bad = np.nonzero(live & (greedy != want))[0]
    assert len(bad) == 0, f"{label}: position {bad[0]}: greedy {greedy[bad[0]]}, want {want[bad[0]]} (x_k {xk[bad[0]]:.3e})"


@pytest.mark.parametrize("dtype", ["fp8", "fp16", "gf4"])
@pytest.mark.parametrize("vocab", sorted(TIES))
def test_exact_ties_go_to_the_lowest_index(vocab, dtype):
    spec = replace(mg.SPECS["pf-tiny"], dtype=dtype, vocab_size=vocab, n_layers=1)
    toks = mg.teacher_tokens(vocab, 120)
    for name, fam_p, fam_n in TIES[vocab]:
        tensors = tie_model(spec, fam_p, fam_n, 31)
        w = sr.Weights(spec, tensors)
        with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
            plain, _ = dm.score(toks, 0)
            lp, greedy, served = dm.score_greedy(toks, 0)
            X = dm.read_state("pf_x").reshape(-1, spec.dim)[:len(toks) - 1]
        assert served == 1 and np.array_equal(lp, plain)
        xk = sr.norm(X, w.vec("model.norm.weight"), spec.norm_eps, False)[:, K_COL]
        tie_check(greedy, np.where(np.abs(xk) > 1e-6 * np.abs(xk).max(), xk, 0), fam_p, fam_n, f"vocab {vocab} {dtype} {name}")


def test_exact_ties_on_the_decode_path():
    """tiny-fp8 (head_dim 32) scores on the decode path: the host argmax of the same logits must also keep the lowest index.
    The logits forward_cuda returns show the ties and give the sign of x_k."""
    spec = mg.SPECS["tiny-fp8"]
    fam_p, fam_n = [200 + 14, 200 + 16, 7], [300, 0 + 9, 511]
    toks = mg.teacher_tokens(spec.vocab_size, 40)
    # the column k whose normed value takes both signs most evenly: a probe classifier with row r = e_r returns x[:dim]
    # (the classifier does not feed back into the hidden state)
    probe = mg.generate(spec, 32)
    W = torch.zeros((spec.vocab_size, spec.dim), dtype=torch.float32)
    W[torch.arange(spec.dim), torch.arange(spec.dim)] = 1.0
    probe["model.output.weight"] = mg.quantize(W, spec.dtype)
    with lib.DeviceModel(spec, probe) as dm:
        xs = np.stack([dm.forward(int(t), i)[:spec.dim] for i, t in enumerate(toks[:-1])])
    k = int(np.argmax(np.minimum((xs > 0).sum(0), (xs < 0).sum(0))))
    tensors = tie_model(spec, fam_p, fam_n, 32, k)
    with lib.DeviceModel(spec, tensors) as dm:
        lp, greedy, served = dm.score_greedy(toks, 0)
    assert served == 0
    with lib.DeviceModel(spec, tensors) as dm:
        logits = np.stack([dm.forward(int(t), i) for i, t in enumerate(toks[:-1])])
    assert (logits[:, fam_p] == logits[:, fam_p[:1]]).all() and (logits[:, fam_n] == logits[:, fam_n[:1]]).all(), "the families do not tie"
    tie_check(greedy, logits[:, fam_p[0]], fam_p, fam_n, "tiny-fp8 decode path")
    assert np.array_equal(greedy, logits.argmax(1))


# ---- 3. the packed calls equal the lone call
def outputs(n):
    return np.full(n, SENTINEL_LP, np.float32), np.full(n, SENTINEL_G, np.int32)


def lone(dm, tokens, co, cl, off, lens):
    want = []
    for c0, c, o, n in zip(co, cl, off, lens):
        if n < 2:
            want.append(None)
            continue
        lp, g, _ = dm.score_greedy(np.concatenate([tokens[c0:c0 + c], tokens[o:o + n]]), 0)
        want.append((lp[c:], g[c:]))
    return want


def assert_matches(got, want, tokens, off, lens, vocab, label):
    lp, g = got
    written = np.zeros(len(tokens), bool)
    for i, (o, n) in enumerate(zip(off, lens)):
        if n < 2:
            continue
        wl, wg = want[i]
        assert np.array_equal(lp[o:o + n - 1], wl), f"{label}: sequence {i} (len {n}): logprobs differ from the lone call"
        assert np.array_equal(g[o:o + n - 1], wg), f"{label}: sequence {i} (len {n}): greedy tokens differ from the lone call"
        assert ((wg >= 0) & (wg < vocab)).all()
        written[o:o + n - 1] = True
    assert (lp[~written] == SENTINEL_LP).all() and (g[~written] == SENTINEL_G).all(), f"{label}: a slot no sequence writes was changed"


CTX_LENS = [0, 1, 9, 32, 33, 300]
SEQ_LENS = [2, 9, 40, 129]


@pytest.mark.parametrize("name,dtype,kvbits", [("pf-tiny", "fp8", 16), ("pf-tiny", "fp16", 8), ("pf-tiny", "gf4", 16), ("pf-tiny", "gf4", 8),
                                               ("pf-tiny-hd128", "fp8", 8), ("pf-tiny-hd128", "fp16", 16)])
def test_packed_calls_equal_the_lone_call(name, dtype, kvbits):
    """Contexts shared within a block and, at seq_len 512, across blocks; filler rows; score_batch_greedy on the sequences
    alone; all contexts empty equals score_batch_greedy; a permuted input order gives the same values."""
    spec = replace(mg.SPECS[name], dtype=dtype)
    tensors = mg.generate(spec, 41)
    tokens, co, cl, off, lens = layout(spec.vocab_size, [(c, SEQ_LENS) for c in CTX_LENS], 2)
    zero = np.zeros(len(off), np.int32)
    label = f"{name}/{dtype}/kv{kvbits}"
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        want_ctx = lone(dm, tokens, co, cl, off, lens)
        want_seq = lone(dm, tokens, zero, zero, off, lens)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        got = dm.score_context_greedy(tokens, co, cl, off, lens, *outputs(len(tokens)))
        assert got[2] == 1
        assert_matches(got[:2], want_ctx, tokens, off, lens, spec.vocab_size, f"{label} context")
        batch = dm.score_batch_greedy(tokens, off, lens, *outputs(len(tokens)))
        assert batch[2] == 1
        assert_matches(batch[:2], want_seq, tokens, off, lens, spec.vocab_size, f"{label} batch")
        empty = dm.score_context_greedy(tokens, zero, zero, off, lens, *outputs(len(tokens)))
        assert np.array_equal(empty[0], batch[0]) and np.array_equal(empty[1], batch[1]), f"{label}: empty contexts differ from score_batch_greedy"
        order = np.random.default_rng(3).permutation(len(off))
        perm = dm.score_context_greedy(tokens, co[order], cl[order], off[order], lens[order], *outputs(len(tokens)))
        assert np.array_equal(perm[0], got[0]) and np.array_equal(perm[1], got[1]), f"{label}: the input order changed the results"


@pytest.mark.parametrize("seq_len,items,served", [
    (4096, [(2100, [9]), (5, [2100]), (40, [9, 20])], 1),  # units larger than a block: alone, across the 2048-row split
    (512, [(400, [200]), (40, [9, 20])], 0),  # past seq_len: the decode path
])
def test_units_larger_than_a_block(seq_len, items, served):
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 42)
    tokens, co, cl, off, lens = layout(spec.vocab_size, items, 4)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        want = lone(dm, tokens, co, cl, off, lens)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        got = dm.score_context_greedy(tokens, co, cl, off, lens, *outputs(len(tokens)))
        assert got[2] == served
        assert_matches(got[:2], want, tokens, off, lens, spec.vocab_size, f"seq_len {seq_len}")
        if served:  # the same units without their contexts through score_batch_greedy
            zero = np.zeros(len(off), np.int32)
            want = lone(dm, tokens, zero, zero, off, lens)
            got = dm.score_batch_greedy(tokens, off, lens, *outputs(len(tokens)))
            assert got[2] == 1
            assert_matches(got[:2], want, tokens, off, lens, spec.vocab_size, f"seq_len {seq_len} batch")


def test_llama3_8b_widths_packed():
    """Two blocks of 128256-vocabulary rows, k_pf_attn<., 128, 4, true, true>: context and batch calls equal the lone call."""
    spec = replace(mg.SPECS["llama3-8b-fp8"], n_layers=2)
    tensors = mg.generate(spec, 43, device="cuda")
    torch.cuda.synchronize()
    tokens, co, cl, off, lens = layout(spec.vocab_size, [(500, [21] * 4)] * 4, 5)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        want = lone(dm, tokens, co, cl, off, lens)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        got = dm.score_context_greedy(tokens, co, cl, off, lens, *outputs(len(tokens)))
    assert got[2] == 1
    assert_matches(got[:2], want, tokens, off, lens, spec.vocab_size, "llama3-8b widths")


# ---- 4. against calm_b200_forward_argmax
def serial_argmax(dm, toks, pos0=0):
    """forward_argmax per position, and the logits it computed from."""
    am, logits = [], []
    for i, t in enumerate(toks[:-1]):
        am.append(dm.forward_argmax(int(t), pos0 + i))
        logits.append(dm.logits_view().copy())
    return np.asarray(am), np.stack(logits)


@pytest.mark.parametrize("name,dtype,kvbits,n", [("pf-tiny", "fp8", 16, 300), ("pf-tiny", "gf4", 8, 129), ("pf-tiny-hd128", "fp16", 16, 200),
                                                 ("pf-tiny-hd128", "fp8", 8, 150)])
def test_greedy_matches_forward_argmax(name, dtype, kvbits, n):
    spec = replace(mg.SPECS[name], dtype=dtype)
    tensors = mg.generate(spec, 44)
    toks = mg.teacher_tokens(spec.vocab_size, n + 1)
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        _, greedy, served = dm.score_greedy(toks, 0)
    assert served == 1
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm:
        am, logits = serial_argmax(dm, toks)
    best, margin = top2(logits)
    assert np.array_equal(am, best), "forward_argmax is not the first maximum of its own logits"
    clear = margin > 2 * (TOL_SIGMA if kvbits == 16 else 4e-2) * logits.std(1)
    print(f"  {name}/{dtype}/kv{kvbits}: {int(clear.sum())} of {n} positions outside the tolerance, "
          f"{int((greedy != am).sum())} differ in all")
    bad = np.nonzero(clear & (greedy != am))[0]
    assert len(bad) == 0, f"position {bad[0]}: greedy {greedy[bad[0]]} vs forward_argmax {am[bad[0]]}"


@pytest.mark.parametrize("name,seq_len,n", [("tiny-moe", None, 20), ("tiny-fp8", None, 20), ("pf-tiny", 64, 80)])
def test_decode_path_greedy_is_forward_argmax(name, seq_len, n):
    """MoE, head_dim 32 and a block past seq_len: served 0, and the host argmax of the same logits is forward_argmax."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 45)
    toks = mg.teacher_tokens(spec.vocab_size, n)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        lp, greedy, served = dm.score_greedy(toks, 0)
        plain, _ = dm.score(toks, 0)
    assert served == 0 and np.array_equal(lp, plain)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
        am, _ = serial_argmax(dm, toks)
    assert np.array_equal(greedy, am)


# ---- 5. draft verification on a live cache
# (step, drafts k, index of the corrupted draft or None): full acceptance, the first draft rejected, rejection mid-way
VERIFY_STEPS = [(3, None), (1, None), (4, 0), (7, 3), (15, None), (2, 1), (7, 6), (15, 9), (3, 0), (7, None)]


def greedy_stream(spec, tensors, prompt, N):
    """calm_b200_decode_greedy after the prompt (stream[e] sits at position len(prompt) - 1 + e), and the serial logits
    behind it."""
    P = len(prompt)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        stream = np.concatenate([[prompt[-1]], dm.decode_greedy(int(prompt[-1]), P - 1, N)])
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        logits = np.stack([dm.forward(int(stream[e]), P - 1 + e) for e in range(N)])
    return stream, logits


def test_draft_verification_reproduces_the_greedy_stream():
    """The model seed is chosen so that no step's top-2 margin lies inside the prompt pass's tolerance: the pass's argmax
    must then be the stream's at every step."""
    spec = mg.SPECS["pf-tiny"]
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 60, start=11), np.int32)
    P, N = len(prompt), 48
    tensors = mg.generate(spec, 46)
    stream, logits = greedy_stream(spec, tensors, prompt, N)
    best, margin = top2(logits)
    assert np.array_equal(best, stream[1:]), "the stream is not the argmax of the serial logits"
    tol = 2 * TOL_SIGMA * logits.std(1)
    assert (margin > tol).all(), f"step {int(np.argmin(margin / tol))}: a top-2 margin inside the tolerance; the seed no longer qualifies"

    out, e, seen = [], 0, set()
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        assert dm.prefill(prompt[:-1], 0) == 1
        for step in range(len(VERIFY_STEPS) * 3):
            k, bad = VERIFY_STEPS[step % len(VERIFY_STEPS)]
            if e + k + 1 >= N:
                break
            drafts = stream[e + 1:e + 1 + k].copy()
            if bad is not None:
                drafts[bad] = (drafts[bad] + 1) % spec.vocab_size
            lp, greedy, served = dm.score_greedy(np.concatenate([[stream[e]], drafts, [0]]), P - 1 + e)
            assert served == 1 and len(greedy) == k + 1
            acc = 0
            while acc < k and greedy[acc] == drafts[acc]:
                acc += 1
            assert acc == (k if bad is None else bad), f"step {step}: accepted {acc} of {k} drafts (corrupted: {bad})"
            seen.add("all" if acc == k else ("first" if acc == 0 else "mid"))
            out += drafts[:acc].tolist() + [int(greedy[acc])]
            e += acc + 1  # slots past P - 1 + e hold rejected drafts; the next call overwrites them
        assert seen == {"all", "first", "mid"}
        assert np.array_equal(out, stream[1:e + 1]), "the verify loop does not reproduce the stream"
        nxt = dm.forward(int(stream[e]), P - 1 + e)
    err = float(np.abs(nxt - logits[e]).max())
    sigma = float(logits[e].std())
    print(f"  {e} tokens verified; next logits |verify - serial| {err:.2e} = {err / sigma:.1e} sigma")
    assert err <= TOL_SIGMA * sigma


# ---- 6. history and edges
HIST_ITEMS = [(100, [40, 9]), (0, [129]), (33, [2, 65]), (7, [20])]


def hist_calls(dm, case):
    tokens, co, cl, off, lens = case
    single = dm.score_greedy(tokens[:200], 0)
    batch = dm.score_batch_greedy(tokens, off, lens, *outputs(len(tokens)))
    ctx = dm.score_context_greedy(tokens, co, cl, off, lens, *outputs(len(tokens)))
    return [single, batch, ctx]


@pytest.mark.parametrize("before", ["poison", "score_greedy", "score_greedy+poison", "score+poison"])
def test_greedy_calls_do_not_depend_on_history(before):
    spec = replace(mg.SPECS["pf-tiny"], vocab_size=1000)
    tensors = mg.generate(spec, 47)
    case = layout(spec.vocab_size, HIST_ITEMS, 6)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        fresh = hist_calls(dm, case)
        again = hist_calls(dm, case)
    long = np.asarray(mg.teacher_tokens(spec.vocab_size, 500, start=3), np.int32)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        if before.startswith("score_greedy"):
            dm.score_greedy(long, 0)
        elif before.startswith("score"):
            dm.score(long, 0)
        if "poison" in before:
            dm.poison(0)
        dirty = hist_calls(dm, case)
    for name, f, a, d in zip(("score_greedy", "score_batch_greedy", "score_context_greedy"), fresh, again, dirty):
        assert f[2] == 1 and d[2] == 1
        lp, g = f[0], f[1]
        written = lp != SENTINEL_LP
        assert np.isfinite(lp[written]).all() and ((g[written] >= 0) & (g[written] < spec.vocab_size)).all(), f"{name}: a value out of range"
        assert np.array_equal(a[0], lp) and np.array_equal(a[1], g), f"{name}: a repeated call differs"
        assert np.array_equal(d[0], lp) and np.array_equal(d[1], g), f"{name}: after {before} the results changed"


def test_empty_calls_write_nothing():
    """n < 2 and nseq == 0 leave logprobs, greedy and the cache untouched."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 48)
    toks = np.asarray(mg.teacher_tokens(spec.vocab_size, 40), np.int32)
    ip, fp = C.POINTER(C.c_int), C.POINTER(C.c_float)
    with lib.DeviceModel(spec, tensors) as dm:
        dm.prefill(toks[:20], 0)
        before = dm.forward(int(toks[20]), 20)
        T = C.byref(dm.transformer)
        lp, g = np.full(4, 7.0, np.float32), np.full(4, 9, np.int32)
        for k in (0, 1):
            assert dm.lib.calm_b200_score_greedy(T, toks.ctypes.data_as(ip), k, 5, lp.ctypes.data_as(fp), g.ctypes.data_as(ip)) == 1
        z = np.zeros(1, np.int32)
        assert dm.lib.calm_b200_score_batch_greedy(T, toks.ctypes.data_as(ip), 40, z.ctypes.data_as(ip), z.ctypes.data_as(ip), 0,
                                                   lp.ctypes.data_as(fp), g.ctypes.data_as(ip)) == 1
        assert dm.lib.calm_b200_score_context_greedy(T, toks.ctypes.data_as(ip), 40, z.ctypes.data_as(ip), z.ctypes.data_as(ip),
                                                     z.ctypes.data_as(ip), z.ctypes.data_as(ip), 0, lp.ctypes.data_as(fp), g.ctypes.data_as(ip)) == 1
        assert (lp == 7.0).all() and (g == 9).all()
        after = dm.forward(int(toks[20]), 20)
    assert np.array_equal(before, after)


def test_zz_summary_of_stage_greedy():
    """Runs last in this file: the largest share of its bound the greedy token's shortfall showed in each stage case."""
    if not worst:
        pytest.skip("the stage cases did not run in this session")
    print("\n  greedy stage: " + ", ".join(f"{k} {r:.2f} of bound" for k, r in sorted(worst.items())))
