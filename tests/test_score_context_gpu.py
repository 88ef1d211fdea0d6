"""calm_b200_score_context: sequences that continue contexts, packed into shared prompt-pass blocks with each context
computed once per block.

A context's rows are a packed sequence of their own; a sequence's rows attend over one virtual key sequence, its context's
rows then its own (k_pf_attn<.., SEG, CTX>), whose tile j holds the keys of tile j of ctx ++ sequence scored alone.  So
the claim is exact: each sequence's log-probabilities equal, bit for bit, calm_b200_score(ctx ++ sequence, 0)[ctx_len:].

- Context lengths that put the context / sequence boundary inside a 32-key tile, on a tile edge and tiles away; every
  weight format, both caches, both head sizes, and Llama-3-8B widths at vocabulary 128256.
- Contexts shared by adjacent and non-adjacent sequences, a shared group that spills into a second block, equal contents
  at two offsets; one placement per block shows in the launch count.
- All contexts empty equals calm_b200_score_batch, in values and in launches; input order does not matter; units too big
  for a block and the decode-path shapes give the lone values.
- No result depends on what earlier calls left behind, and nothing after a call depends on it either.

calm_b200_score_batch is this call with every context empty, and test_score_batch_gpu.py checks it with the helpers
defined here (`batch=True`), on cases whose contexts are all empty."""
from dataclasses import replace

import numpy as np
import pytest
import torch

from calm_b200 import lib
from calm_b200 import modelgen as mg
from calm_b200.cstructs import FF_UPDATE_KV_ONLY

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-12345.5)


def layout(vocab, items, seed):
    """items: [(ctx_len, [sequence lengths])].  Each item's context is stored once, followed by its sequences:
    (tokens, ctx_off, ctx_len, off, len)."""
    rng = np.random.default_rng(seed)
    parts, co, cl, off, ln, at = [], [], [], [], [], 0
    for c, lens in items:
        parts.append(rng.integers(0, vocab, c))
        c0, at = at, at + c
        for n in lens:
            parts.append(rng.integers(0, vocab, n))
            co.append(c0), cl.append(c), off.append(at), ln.append(n)
            at += n
    i32 = lambda x: np.asarray(x, np.int32)  # noqa: E731
    return i32(np.concatenate(parts)), i32(co), i32(cl), i32(off), i32(ln)


def lone(dm, tokens, co, cl, off, lens):
    """calm_b200_score of each ctx ++ sequence on its own from position 0, the context's positions dropped."""
    want, served = [], 1
    for c0, c, o, n in zip(co, cl, off, lens):
        if n < 2:
            want.append(None)
            continue
        lp, s = dm.score(np.concatenate([tokens[c0:c0 + c], tokens[o:o + n]]), 0)
        want.append(lp[c:])
        served &= s
    return want, served


def run(dm, tokens, co, cl, off, lens, batch=False):
    """The context call, or with `batch` calm_b200_score_batch of the same sequences (co and cl unused), into an output
    that holds the sentinel."""
    out = np.full(len(tokens), SENTINEL, np.float32)
    got, served = dm.score_batch(tokens, off, lens, out) if batch else dm.score_context(tokens, co, cl, off, lens, out)
    assert got is out
    return got, served


def assert_matches(got, want, tokens, off, lens, label):
    """Sequence by sequence bit for bit; every written value finite, every other slot still the sentinel."""
    written = np.zeros(len(tokens), bool)
    for i, (o, n) in enumerate(zip(off, lens)):
        if n < 2:
            continue
        part = got[o:o + n - 1]
        assert np.isfinite(part).all(), f"{label}: sequence {i} (len {n}) has a value that is not finite"
        if not np.array_equal(part, want[i]):
            j = int(np.argmax(part != want[i]))
            raise AssertionError(f"{label}: sequence {i} (len {n}), position {j}: packed {part[j]!r} vs alone {want[i][j]!r} "
                                 f"({int((part != want[i]).sum())} of {n - 1} positions differ)")
        written[o:o + n - 1] = True
    assert (got[~written] == SENTINEL).all(), f"{label}: a slot no sequence writes was changed"


def check(spec, tensors, case, label, seq_len=None, kvbits=16, served=1, batch=False):
    tokens, co, cl, off, lens = case
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        want, s_lone = lone(dm, tokens, co, cl, off, lens)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        got, s_packed = run(dm, tokens, co, cl, off, lens, batch)
    assert s_packed == served and s_lone == served, f"{label}: served {s_packed} (alone {s_lone}), expected {served}"
    assert_matches(got, want, tokens, off, lens, label)
    return got


def assert_order_does_not_matter(spec, tensors, case, batch=False):
    tokens, co, cl, off, lens = case
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        base, served = run(dm, *case, batch)
        assert served == 1
        for order in (np.arange(len(off))[::-1], np.random.default_rng(5).permutation(len(off))):
            got, served = run(dm, tokens, co[order], cl[order], off[order], lens[order], batch)
            assert served == 1 and np.array_equal(got, base), f"order {order.tolist()} changed the results"


# ---- history independence, from each call's module-scoped fixture
def fresh_results(tensor_seed, make_case, batch=False):
    """A pf-tiny model, a case and the call's results on a fresh engine at seq_len 512."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, tensor_seed)
    case = make_case(spec.vocab_size)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        fresh, served = run(dm, *case, batch)
    assert served == 1
    return spec, tensors, case, fresh


def assert_independent_of_history(hist, before, batch=False):
    spec, tensors, case, fresh = hist
    long = np.asarray(mg.teacher_tokens(spec.vocab_size, 500, start=3), np.int32)
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        if "score" in before:
            dm.score(long, 0)
        if before == "prefill":
            dm.prefill(long, 0)
        if "poison" in before:
            dm.poison(0)
        got, served = run(dm, *case, batch)
    assert served == 1
    assert np.isfinite(got[got != SENTINEL]).all() and np.array_equal(got, fresh), f"after {before}: the results changed"


def assert_nothing_after_depends_on_it(hist, batch=False):
    """forward_prefill_cuda and forward_cuda from position 0 after a call equal the fresh engine's, bit for bit."""
    spec, tensors, case, _ = hist
    prompt = np.asarray(mg.teacher_tokens(spec.vocab_size, 200, start=9), np.int32)
    runs = []
    for dirty in (False, True):
        with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
            if dirty:
                run(dm, *case, batch)
            assert dm.prefill(prompt[:150], 0) == 1
            after_pf = [dm.forward(int(prompt[p]), p) for p in range(150, 160)]
            if dirty:
                run(dm, *case, batch)
            dm.forward(int(prompt[0]), 0, FF_UPDATE_KV_ONLY)
            serial = [dm.forward(int(prompt[p]), p) for p in range(1, 12)]
            runs.append(after_pf + serial)
    for i, (a, b) in enumerate(zip(*runs)):
        assert np.isfinite(a).all() and np.array_equal(a, b), f"logits {i} after a call differ from the fresh engine's"


# Boundaries inside a 32-key tile (1, 7, 8, 9, 31, 33, 100, 300), on a tile edge (32) and none (0); each context with every
# continuation length.  At seq_len 512 (capacity 512 rows) that is several blocks, most holding more than one context.
CTX_LENS = [0, 1, 7, 8, 9, 31, 32, 33, 100, 300]
SEQ_LENS = [2, 3, 9, 40, 129]


@pytest.mark.parametrize("name,dtype,kvbits", [("pf-tiny", "fp8", 16), ("pf-tiny", "fp8", 8), ("pf-tiny", "fp16", 16), ("pf-tiny", "fp16", 8),
                                               ("pf-tiny", "gf4", 16), ("pf-tiny", "gf4", 8), ("pf-tiny-hd128", "fp8", 16), ("pf-tiny-hd128", "gf4", 8)])
def test_each_sequence_equals_its_concatenation_alone(name, dtype, kvbits):
    spec = replace(mg.SPECS[name], dtype=dtype)
    tensors = mg.generate(spec, 21)
    case = layout(spec.vocab_size, [(c, SEQ_LENS) for c in CTX_LENS], 1)
    check(spec, tensors, case, f"{name}/{dtype}/kv{kvbits}", seq_len=512, kvbits=kvbits)


def test_sharing_within_and_across_blocks():
    """Context A shared by adjacent sequences and by one after another context's; A's contents again at a second offset
    (not shared, scored correctly); then eight more of A's sequences of 64 rows, which spill into a second block where A
    is placed again."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 22)
    rng = np.random.default_rng(2)
    a, b = rng.integers(0, spec.vocab_size, 100), rng.integers(0, spec.vocab_size, 37)
    segs = [a, b, a.copy()]
    seqs = [(0, 20), (0, 9), (1, 40), (0, 3), (2, 20)] + [(0, 65)] * 8
    parts, starts, at = [], [], 0
    for s in segs:
        parts.append(s), starts.append(at)
        at += len(s)
    co, cl, off, ln = [], [], [], []
    for k, n in seqs:
        parts.append(rng.integers(0, spec.vocab_size, n))
        co.append(starts[k]), cl.append(len(segs[k])), off.append(at), ln.append(n)
        at += n
    i32 = lambda x: np.asarray(x, np.int32)  # noqa: E731
    check(spec, tensors, (i32(np.concatenate(parts)), i32(co), i32(cl), i32(off), i32(ln)), "sharing", seq_len=512)


def test_a_shared_context_is_computed_once_per_block():
    """Eight 21-token sequences after one 300-token context: 304 + 8 x 24 = 496 rows, one block, so exactly the launches
    of one calm_b200_score of a single block.  The same concatenations through calm_b200_score_batch take 320 rows each,
    one block apiece."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 23)
    tokens, co, cl, off, lens = layout(spec.vocab_size, [(300, [21] * 8)], 3)
    L = lib.load()
    with lib.DeviceModel(spec, tensors, seq_len=512) as dm:
        n0 = L.calm_b200_launch_count()
        _, served = run(dm, tokens, co, cl, off, lens)
        n1 = L.calm_b200_launch_count()
        assert served == 1 and dm.score(tokens[:200], 0)[1] == 1
        n2 = L.calm_b200_launch_count()
        cat = np.concatenate([np.concatenate([tokens[c0:c0 + c], tokens[o:o + n]]) for c0, c, o, n in zip(co, cl, off, lens)])
        bo = np.arange(0, len(cat), 321, dtype=np.int32)
        assert dm.score_batch(cat, bo, np.full(8, 321, np.int32))[1] == 1
        n3 = L.calm_b200_launch_count()
    assert n1 - n0 == n2 - n1, f"one shared block launched {n1 - n0} kernels, one calm_b200_score block {n2 - n1}"
    assert n3 - n2 == 8 * (n2 - n1), f"the unshared batch launched {n3 - n2} kernels"


def test_all_contexts_empty_equals_score_batch():
    """ctx_len 0 everywhere: calm_b200_score_batch's values and launches, on its LENS layout and on study() chunks of a
    3000-token text."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 24)
    lens = np.asarray([2, 3, 9, 40, 129, 257, 513, 1, 257, 129, 40, 0], np.int32)
    rng = np.random.default_rng(4)
    lens_tokens = rng.integers(0, spec.vocab_size, int(lens.sum())).astype(np.int32)
    lens_off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
    n = 3000
    text = np.asarray(mg.teacher_tokens(spec.vocab_size, n), np.int32)
    study_off = np.arange(0, n - 1, 256, dtype=np.int32)
    study_len = np.minimum(257, n - study_off).astype(np.int32)
    L = lib.load()
    for label, (tokens, off, ln), seq_len in (("LENS", (lens_tokens, lens_off, lens), 512), ("study", (text, study_off, study_len), 4096)):
        zero = np.zeros(len(off), np.int32)
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            want = np.full(len(tokens), SENTINEL, np.float32)
            n0 = L.calm_b200_launch_count()
            s_batch = dm.score_batch(tokens, off, ln, want)[1]
            n_batch = L.calm_b200_launch_count() - n0
        with lib.DeviceModel(spec, tensors, seq_len=seq_len) as dm:
            n0 = L.calm_b200_launch_count()
            got, s_ctx = run(dm, tokens, zero, zero, off, ln)
            n_ctx = L.calm_b200_launch_count() - n0
        assert s_ctx == s_batch, f"{label}: served {s_ctx}, score_batch {s_batch}"
        assert np.isfinite(got[got != SENTINEL]).all() and np.array_equal(got, want), f"{label}: differs from calm_b200_score_batch"
        assert n_ctx == n_batch, f"{label}: {n_ctx} launches, score_batch {n_batch}"


def test_order_does_not_matter():
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 25)
    assert_order_does_not_matter(spec, tensors, layout(spec.vocab_size, [(100, [7, 40]), (0, [65]), (33, [2, 129, 17]), (300, [21, 21]), (9, [90])], 5))


@pytest.mark.parametrize("seq_len,items,served", [
    (4096, [(2100, [9]), (5, [2100]), (40, [9, 20])], 1),  # 2104 + 8 and 8 + 2104 rows: more than a block, alone in 2048-row blocks
    (512, [(400, [200]), (40, [9, 20])], 0),  # 599 positions past seq_len 512: the decode path
])
def test_units_larger_than_a_block(seq_len, items, served):
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 26)
    check(spec, tensors, layout(spec.vocab_size, items, 6), f"seq_len {seq_len}", seq_len=seq_len, served=served)


@pytest.mark.parametrize("name", ["tiny-moe", "tiny-fp8"])
def test_falls_back_to_the_decode_path(name):
    """MoE and head_dim 32 score every ctx ++ sequence on the decode path: the call returns 0 and the lone values."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 27)
    check(spec, tensors, layout(spec.vocab_size, [(20, [2, 9]), (0, [12]), (9, [5])], 7), name, served=0)


def test_llama3_8b_widths():
    """Four items of a 500-token context with four 21-token sequences: 600 rows each, two blocks (three items, then one),
    k_pf_attn<., 128, 4, true, true>, 1002 vocabulary tiles, the last partial."""
    spec = replace(mg.SPECS["llama3-8b-fp8"], n_layers=2)
    tensors = mg.generate(spec, 28, device="cuda")
    torch.cuda.synchronize()
    check(spec, tensors, layout(spec.vocab_size, [(500, [21] * 4)] * 4, 8), "llama3-8b widths", seq_len=4096)


# ---- history independence
HIST_ITEMS = [(100, [40, 9]), (0, [129]), (33, [2, 65]), (7, [20])]


@pytest.fixture(scope="module")
def hist():
    return fresh_results(29, lambda vocab: layout(vocab, HIST_ITEMS, 9))


@pytest.mark.parametrize("before", ["poison", "score", "prefill", "score+poison"])
def test_context_call_does_not_depend_on_history(hist, before):
    assert_independent_of_history(hist, before)


def test_nothing_after_a_context_call_depends_on_it(hist):
    assert_nothing_after_depends_on_it(hist)
