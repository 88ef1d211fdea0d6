"""No result may depend on what earlier calls left behind.

Decode and the prompt pass are deterministic (DESIGN.md s.2 "History independence"), so the claim needs no tolerance: the
same calls give bit-identical output whether the engine was freshly prepared (a zeroed cache, zeroed prompt-pass
matrices, zero token parameters) or had another history first, and whatever bytes its scratch memory held.  Every case
runs one scenario twice, on a fresh DeviceModel and on a dirty one (other calls first and / or calm_b200_poison_state,
which puts NaN into every scratch buffer and the unused cache slots), and compares every output with
assert_array_equal: host and device logits, log-probabilities, greedy and sampled tokens, the rng state, the engine
buffers read_state exposes and every cache slot the scenario wrote.  All of it must be finite as well, so a NaN on both
sides cannot pass.  A difference is a read of memory the call did not write, or a nondeterminism.

Each model opened asserts its plan lines, so it is known which kernels served the case."""
import os
import sys
from collections import namedtuple
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from test_stages_gpu import REG, V4K  # noqa: E402
from test_variants_gpu import RING, plan_of  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY  # noqa: E402

pytestmark = pytest.mark.gpu

# spec, seq_len, the attention and matvec kernels prepare_cuda must plan, whether the tensor-core prompt pass serves it.
# Two layers where the width allows, so the activation buffers are reused across layers under programmatic dependent launch.
Shape = namedtuple("Shape", "spec seq_len attn stages batched")
_HD64 = replace(mg.SPECS["pf-tiny-hd128"], name="hd64", dim=2048, hidden_dim=4096, n_heads=32, n_kv_heads=4, head_dim=64, n_layers=2,
                vocab_size=V4K, rope_theta=1e4, qkv_bias=False)
SHAPES = {
    # k_qkv, k_attn2<4, 128>, the ring-fed matvecs, the wgmma pass and its classifier
    "llama": Shape(replace(mg.SPECS["llama3-8b-fp8"], n_layers=2, vocab_size=V4K), 4096, "k_attn2", RING, True),
    "llama-128256": Shape(replace(mg.SPECS["llama3-8b-fp8"], n_layers=1), 4096, "k_attn2", RING, True),  # k_output's candidates, the sampler's chunks, 1002 vocabulary tiles
    "mistral-gf4": Shape(replace(mg.SPECS["mistral-7b-gf4"], n_layers=2, vocab_size=V4K), 4009, "k_attn2", RING, True),  # gf4 staging with its group sums; a partial last block
    "hd64": Shape(_HD64, 512, "k_attn2", RING, True),  # k_attn2<8, 64>
    "qwen-small": Shape(replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=2, vocab_size=V4K), 512, "k_attn", REG, True),  # k_attn, register-fed matvecs, qkv bias
    "tiny-llama": Shape(mg.SPECS["tiny-llama"], 128, "k_attn2", REG, True),  # k_attn2<4, 128> after register-fed matvecs, three layers
    "tiny-hd256": Shape(replace(mg.SPECS["tiny-hd256"], vocab_size=V4K), 4096, "k_attn", RING, False),
    "mixtral-1": Shape(replace(mg.SPECS["mixtral-8x7b-fp8"], n_layers=1, vocab_size=V4K), 4096, "k_attn2", REG, False),  # router, expert rows of hb
    "tiny-moe": Shape(mg.SPECS["tiny-moe"], 64, "k_attn", REG, False),
    "pf-tiny-v1000": Shape(replace(mg.SPECS["pf-tiny"], vocab_size=1000), 512, "k_attn2", REG, True),  # a partial vocabulary tile
}


@pytest.fixture(scope="module")
def weights():
    """Each shape's tensors, generated on the device once and kept while DeviceModels come and go."""
    made = {}

    def get(shape):
        if shape not in made:
            made[shape] = mg.generate(SHAPES[shape].spec, 31, device="cuda")
            torch.cuda.synchronize()
        return made[shape]

    yield get
    made.clear()


@pytest.fixture(autouse=True)
def plan_lines(monkeypatch):
    monkeypatch.delenv("CALM_B200_QUIET", raising=False)


class Opener:
    """open(shape, kvbits) -> DeviceModel, after asserting the kernels prepare_cuda planned; .slices = the attention's slices."""

    def __init__(self, weights, capfd):
        self.weights, self.capfd = weights, capfd

    def __call__(self, shape, kvbits):
        s = SHAPES[shape]
        dm = lib.DeviceModel(s.spec, self.weights(shape), seq_len=s.seq_len, kvbits=kvbits)
        kernel, dm.slices, stages = plan_of(self.capfd)
        assert (kernel, stages) == (s.attn, s.stages), (shape, kernel, stages)
        return dm


@pytest.fixture
def open_model(weights, capfd):
    return Opener(weights, capfd)


# ---- what is recorded and how it is compared

def toks_of(dm, n, start=0):
    return mg.teacher_tokens(dm.vocab, n, start=start)


def cache_slots(dm, slots):
    """KEYS / VALUES of every layer at `slots` (every kv head)."""
    s, slots = dm.spec, sorted(set(slots))
    shape = (s.n_kv_heads, dm.seq_len, s.head_dim)
    return {f"{w}[layer {l}]": dm.read_state(w, l).reshape(shape)[:, slots].copy() for l in range(s.n_layers) for w in ("keys", "values")}


def decode_state(dm):
    return {k: dm.read_state(k) for k in ("x", "q", "att", "hb")}


def pass_matrices(dm):
    """The prompt pass's residual stream, queries, attention output and hidden matrix, every row of the buffers."""
    s = dm.spec
    width = {"pf_x": s.dim, "pf_q": s.q_dim, "pf_att": s.q_dim, "pf_hb": s.hidden_dim}
    return {k: dm.read_state(k).reshape(-1, w) for k, w in width.items()}


def pass_rows(dm, n):
    return {k: m[:n].copy() for k, m in pass_matrices(dm).items()}


def outside(dm, n):
    """What a prompt pass of n tokens at pos 0 must leave as it found it: rows >= n of its matrices, cache slots >= n."""
    s = dm.spec
    out = {k: m[n:].copy() for k, m in pass_matrices(dm).items()}
    out.update({f"{w}[layer {l}]": dm.read_state(w, l).reshape(s.n_kv_heads, dm.seq_len, s.head_dim)[:, n:].copy()
                for l in range(s.n_layers) for w in ("keys", "values")})
    return out


def written_slots(positions, seq_len):
    """Cache slots that steps at `positions` write: their own, and the re-rotated sinks once the cache has rolled over."""
    out = set()
    for p in positions:
        slot, _, sinks = sr.kv_slot(p, seq_len)
        out |= {slot} | set(range(sinks))
    return sorted(out)


def put(rec, prefix, items):
    rec.update({f"{prefix}: {k}": v for k, v in items.items()})


def assert_identical(fresh, dirty, label):
    assert list(fresh) == list(dirty), (label, sorted(set(fresh) ^ set(dirty)))
    for k in fresh:
        a, b = np.asarray(fresh[k]), np.asarray(dirty[k])
        assert a.shape == b.shape, (label, k, a.shape, b.shape)
        assert np.isfinite(a).all(), f"{label}: {k} is not finite on the fresh engine ({int((~np.isfinite(a)).sum())} of {a.size} values)"
        assert np.isfinite(b).all(), f"{label}: {k} is not finite on the dirty engine ({int((~np.isfinite(b)).sum())} of {b.size} values)"
        np.testing.assert_array_equal(b, a, err_msg=f"{label}: {k} depends on the engine's history")


# ---- 1. poisoned decode at the attention's edges

def edge_positions(seq_len, slices):
    """kv_len 1, a full block, one past it, two past it; a context that ends inside a block; a block the attention's last slice
    owns (block b belongs to slice b % slices); the last slot; and a rolled-over cache."""
    nblk = -(-seq_len // 16)
    partial = (seq_len * 5 // 8) // 16 * 16 + 8
    last_slice = 16 * min(nblk - 1, slices - 1) + 7
    return sorted({p for p in (0, 15, 16, 17, partial, last_slice, seq_len - 1) if p < seq_len}) + [seq_len + 5]


def run_edges(dm, poisoned):
    rec = {}
    for pos in edge_positions(dm.seq_len, dm.slices):
        n = min(pos, dm.seq_len)
        dm.fill_kv(n, seed=5)
        if poisoned:
            dm.poison(n)  # the slots the step must not read, and every scratch buffer (past seq_len: scratch only)
        put(rec, f"pos {pos}", {"logits": dm.forward(17, pos), **decode_state(dm), **cache_slots(dm, written_slots([pos], dm.seq_len))})
    return rec


EDGE_CASES = [("llama", 16), ("llama", 8), ("llama-128256", 16), ("mistral-gf4", 8), ("hd64", 16), ("hd64", 8), ("qwen-small", 16),
              ("tiny-llama", 16), ("tiny-hd256", 8), ("mixtral-1", 16), ("tiny-moe", 16)]


@pytest.mark.parametrize("shape,kvbits", EDGE_CASES)
def test_poisoned_decode_at_the_attention_edges(open_model, shape, kvbits):
    """fill_kv(p), one forward at p: with NaN in every slot >= p and in all scratch, against the same calls without."""
    out = []
    for poisoned in (False, True):
        with open_model(shape, kvbits) as dm:
            out.append(run_edges(dm, poisoned))
    assert_identical(out[0], out[1], f"{shape} kv{kvbits}")


# ---- 2. a new conversation over an old one

def conversation_one(dm):
    n1 = min(600, dm.seq_len * 3 // 4)
    toks = toks_of(dm, n1 + 5, start=7)
    dm.prefill(toks[:n1], 0)
    for i in range(5):
        dm.forward(toks[n1 + i], n1 + i)
    if dm.seq_len >= 4096:  # a long context last: the token parameters the next call's early KV request sees say 4001 positions
        dm.fill_kv(4000, seed=3)
        dm.forward(5, 4000), dm.forward(6, 4001)


def conversation_two(dm, shape):
    rec = {}
    n2 = min(130, dm.seq_len // 4)
    toks = toks_of(dm, n2 + 3, start=100)
    assert dm.prefill(toks[:n2], 0) == int(SHAPES[shape].batched)
    if SHAPES[shape].batched:
        put(rec, "prompt pass", pass_rows(dm, n2))
    for i in range(3):
        logits = dm.forward(toks[n2 + i], n2 + i)
        put(rec, f"step {n2 + i}", {"logits": logits})
    put(rec, "greedy", {"tokens": dm.decode_greedy(int(logits.argmax()), n2 + 3, 8), "device logits": dm.device_logits(), **decode_state(dm)})
    put(rec, "cache", cache_slots(dm, range(n2 + 11)))
    return rec


CONVERSATION_CASES = [("llama", 16, False), ("llama", 16, True), ("llama", 8, True), ("mistral-gf4", 8, False), ("mistral-gf4", 8, True),
                      ("hd64", 16, False), ("qwen-small", 16, True), ("tiny-llama", 16, True), ("tiny-hd256", 16, False),
                      ("mixtral-1", 16, True), ("tiny-moe", 16, False)]


@pytest.mark.parametrize("shape,kvbits,poisoned", CONVERSATION_CASES)
def test_new_conversation_over_an_old_one(open_model, shape, kvbits, poisoned):
    """A prompt pass, decode steps and a greedy loop from pos 0 give the same bits on an engine whose cache, prompt-pass
    matrices and token parameters still hold a longer conversation (and, poisoned, NaN wherever data may be)."""
    with open_model(shape, kvbits) as dm:
        fresh = conversation_two(dm, shape)
    with open_model(shape, kvbits) as dm:
        conversation_one(dm)
        if poisoned:
            dm.poison(0)
        dirty = conversation_two(dm, shape)
    assert_identical(fresh, dirty, f"{shape} kv{kvbits}")


# ---- 3. backward and forward jumps of pos

def jump_steps(seq_len):
    """(token, pos, refill): refill = fill_kv(seq_len) first, so the step's cache does not depend on the steps before it;
    without, the step regenerates the position of the step before (the slot is rewritten).  The last four run on a
    rolled-over cache, where the re-rotated sinks share a block with the patched slot."""
    a = seq_len * 3 // 4 - (72 if seq_len >= 4096 else 0)
    return [(11, a, True), (12, 2, True), (13, a + 1, True), (14, 17, True), (15, 16, True), (16, 16, False),
            (17, seq_len + 5, True), (18, seq_len + a, True), (19, seq_len + 5, True), (20, seq_len + 5, False)]


def record_step(dm, rec, i, token, pos):
    put(rec, f"step {i} pos {pos}", {"logits": dm.forward(token, pos), **decode_state(dm), **cache_slots(dm, written_slots([pos], dm.seq_len))})


@pytest.mark.parametrize("shape,kvbits", [("llama", 16), ("llama", 8), ("hd64", 16), ("tiny-hd256", 16), ("qwen-small", 8)])
def test_jumps_of_pos(open_model, shape, kvbits):
    """One engine stepping 3000 -> 2 -> 3001 -> 17 -> 16 -> 16 again and on past seq_len, against a fresh engine per step."""
    steps = jump_steps(SHAPES[shape].seq_len)
    fresh, dirty = {}, {}
    with open_model(shape, kvbits) as dm:
        for i, (token, pos, refill) in enumerate(steps):
            if refill:
                dm.fill_kv(dm.seq_len, seed=8)
            record_step(dm, dirty, i, token, pos)
    for i, (token, pos, refill) in enumerate(steps):
        with open_model(shape, kvbits) as dm:
            dm.fill_kv(dm.seq_len, seed=8)
            if not refill:
                dm.forward(steps[i - 1][0], steps[i - 1][1], FF_UPDATE_KV_ONLY)
            record_step(dm, fresh, i, token, pos)
    assert_identical(fresh, dirty, f"{shape} kv{kvbits}")


# ---- 4. a shorter prompt pass after a longer one

def short_pass(dm, n, after_longer=False):
    rec = {}
    toks = toks_of(dm, n + 1, start=200)
    before = outside(dm, n) if after_longer else None
    assert dm.prefill(toks[:n], 0) == 1
    if after_longer:  # the longer pass's values (NaN is equal to NaN here) are still there, bit for bit
        for k, v in outside(dm, n).items():
            assert len(v) and v.size, k
            np.testing.assert_array_equal(v, before[k], err_msg=f"n {n}: {k}: the pass wrote past its own rows / slots")
    put(rec, f"n {n}", pass_rows(dm, n))
    put(rec, f"n {n}", {"next logits": dm.forward(toks[n], n), **cache_slots(dm, range(n + 1))})
    return rec


@pytest.mark.parametrize("poisoned", [False, True])
@pytest.mark.parametrize("shape,kvbits", [("llama", 16), ("mistral-gf4", 8), ("hd64", 16), ("qwen-small", 8)])
def test_shorter_prompt_pass_after_a_longer_one(open_model, shape, kvbits, poisoned):
    """prefill(300), then prefill(n) at pos 0 inside the same buffers: the padding rows of the last token tile hold the longer
    pass's values (or NaN), and rows < n, the cache and the next token must not notice.  Nor may the short pass write
    anything of its own there: rows >= n and slots >= n keep the longer pass's bits."""
    fresh, dirty = {}, {}
    with open_model(shape, kvbits) as dm:
        for n in (1, 127, 128, 130):
            assert dm.prefill(toks_of(dm, 300, start=50), 0) == 1
            if poisoned:
                dm.poison(0)
            dirty.update(short_pass(dm, n, after_longer=True))
    for n in (1, 127, 128, 130):
        with open_model(shape, kvbits) as dm:
            fresh.update(short_pass(dm, n))
    assert_identical(fresh, dirty, f"{shape} kv{kvbits}")


# ---- 5. scoring on dirty buffers

# shape, kvbits, the call that came before ("score" / "prefill" of up to 300 other tokens), poison, position of the scored block
# (None: 0; "end": 100 before seq_len, so the block would roll the cache over and goes through the decode path instead)
SCORE_CASES = {
    "after a longer score": ("llama", 16, "score", False, None),
    "after a prompt pass alone": ("llama", 16, "prefill", False, None),  # the scoring buffers are allocated after the pass's
    "poisoned, e5m2 cache": ("llama", 8, "score", True, None),
    "partial vocabulary tile": ("pf-tiny-v1000", 16, "score", True, None),
    "vocabulary 128256": ("llama-128256", 16, "score", True, None),
    "mistral-gf4": ("mistral-gf4", 8, "score", True, None),
    "tiny-moe through the decode path": ("tiny-moe", 16, "score", True, None),
    "a block past seq_len through the decode path": ("pf-tiny-v1000", 16, "score", True, "end"),
}


def score_then_prefill(dm, shape, where):
    """score of up to 130 tokens, then a 100-token prompt pass over it."""
    rec = {}
    m = min(130, dm.seq_len // 2)
    pos0 = 0 if where is None else dm.seq_len - 100
    toks = toks_of(dm, m, start=300)
    if where == "end":  # a rolled-over block attends to every slot: both engines start from the same full cache
        dm.fill_kv(dm.seq_len, seed=9)
    lp, served = dm.score(toks, pos0)
    assert served == int(SHAPES[shape].batched and where is None)
    put(rec, "score", {"log-probabilities": lp, **cache_slots(dm, written_slots(range(pos0, pos0 + m - 1), dm.seq_len))})
    if served:
        put(rec, "score", pass_rows(dm, m - 1))
    put(rec, "prefill after score", prefill_only(dm, shape))
    return rec


def prefill_only(dm, shape):
    n = min(100, dm.seq_len // 2)
    assert dm.prefill(toks_of(dm, n, start=400), 0) == int(SHAPES[shape].batched)
    return cache_slots(dm, range(n))


@pytest.mark.parametrize("case", sorted(SCORE_CASES))
def test_scoring_on_dirty_buffers(open_model, case):
    shape, kvbits, before, poisoned, where = SCORE_CASES[case]
    with open_model(shape, kvbits) as dm:
        fresh = score_then_prefill(dm, shape, where)
    with open_model(shape, kvbits) as dm:
        hist = toks_of(dm, min(300, dm.seq_len - 4), start=33)
        dm.score(hist, 0) if before == "score" else dm.prefill(hist, 0)
        if poisoned:
            dm.poison(0)
        dirty = score_then_prefill(dm, shape, where)
    assert_identical(fresh, dirty, case)
    with open_model(shape, kvbits) as dm:  # and the prompt pass after a score leaves what it leaves on an engine that never scored
        alone = prefill_only(dm, shape)
    assert_identical(alone, {k[len("prefill after score: "):]: v for k, v in dirty.items() if k.startswith("prefill after score: ")}, case + ", prefill alone")


# ---- 6. one token stream through every call mode

N_STREAM, N_PERF = 24, 4
MODES = ("kv-only", "forward", "argmax", "greedy-1", "sample-t0", "sample")


def mode_of(i):
    """The call that feeds position i on the dirty side: the six modes in rotation, the last four positions under set_perf(1)."""
    return "perf" if i >= N_STREAM - N_PERF else MODES[i % len(MODES)]


def stream_mixed(dm, toks, want):
    """Teacher-forced `toks` through the rotating call modes; the logits each mode exposes, keyed like stream_plain's.
    `want` = the plain side's logits, for the tokens the sampling modes return."""
    rec, rng = {}, 99
    for i, t in enumerate(toks):
        mode, key = mode_of(i), f"pos {i}: logits"
        if mode == "kv-only":
            assert dm.forward(t, i, FF_UPDATE_KV_ONLY) is None
        elif mode == "forward":
            rec[key] = dm.forward(t, i)
        elif mode == "argmax":
            tok = dm.forward_argmax(t, i)
            rec[key] = dm.logits_view().copy()
            assert tok == int(want[i].argmax()), (i, mode)
        elif mode == "greedy-1":
            tok = int(dm.decode_greedy(t, i, 1)[0])
            rec[key] = dm.device_logits()
            assert tok == int(want[i].argmax()), (i, mode)
        elif mode == "sample-t0":
            tok, rng2 = dm.forward_sample(t, i, 0.0, 0.1, rng)
            rec[key] = dm.device_logits()
            assert (tok, rng2) == (int(want[i].argmax()), rng), (i, mode)
        elif mode == "sample":
            tok, rng2 = dm.forward_sample(t, i, 1.0, 0.1, rng)
            rec[key] = dm.device_logits()
            assert (tok, rng2) == lib.sample_logits(want[i], 1.0, 0.1, rng), (i, mode)
            rng = rng2
        else:
            dm.lib.calm_b200_set_perf(1)
            rec[key] = dm.forward(t, i)  # the stamped graph: the same kernels with a stamp slot each
            dm.lib.calm_b200_set_perf(0)
    return rec


def stream_tail(dm, token):
    """After either history: the cache of the stream, then a sampling loop from its end."""
    rec = cache_slots(dm, range(N_STREAM))
    out, rng = dm.decode_sample(token, N_STREAM, 6, 1.0, 0.1, 321)
    rec.update({"sampled tokens": out, "rng state": np.uint64(rng), "device logits after the loop": dm.device_logits()})
    put(rec, "after the loop", cache_slots(dm, range(N_STREAM, N_STREAM + 6)))
    return rec


@pytest.mark.parametrize("shape,kvbits", [("llama", 16), ("llama-128256", 16), ("mistral-gf4", 8), ("hd64", 16), ("qwen-small", 16), ("mixtral-1", 16), ("tiny-moe", 8)])
def test_one_stream_through_every_call_mode(open_model, shape, kvbits):
    """KV-only, logits, logits + argmax, the greedy loop, the sampling loop (greedy and not) and the stamped graphs share the
    activation buffers, the candidate and sampler scratch and the token parameters: a position computes the same bits
    whichever of them served the positions before it, and whichever serves it."""
    with open_model(shape, kvbits) as dm:
        toks = toks_of(dm, N_STREAM + 1, start=40)
        plain = {f"pos {i}: logits": dm.forward(t, i) for i, t in enumerate(toks[:N_STREAM])}
        tail_plain = stream_tail(dm, toks[N_STREAM])
    with open_model(shape, kvbits) as dm:
        mixed = stream_mixed(dm, toks[:N_STREAM], [plain[f"pos {i}: logits"] for i in range(N_STREAM)])
        tail_mixed = stream_tail(dm, toks[N_STREAM])
    assert len(mixed) == N_STREAM - len([i for i in range(N_STREAM) if mode_of(i) == "kv-only"])
    assert_identical({k: plain[k] for k in mixed}, mixed, f"{shape} kv{kvbits}")
    assert_identical(tail_plain, tail_mixed, f"{shape} kv{kvbits}, after the stream")


# ---- 7. another model in between

def llama_session(dm):
    rec = {}
    toks = toks_of(dm, 131, start=500)
    for i in range(4):
        put(rec, f"decode {i}", {"logits": dm.forward(toks[i], i)})
    put(rec, "decode", {**decode_state(dm), **cache_slots(dm, range(4))})
    assert dm.prefill(toks[:130], 0) == 1
    put(rec, "prompt pass", {**pass_rows(dm, 130), **cache_slots(dm, range(130))})
    lp, served = dm.score(toks, 0)
    assert served == 1
    put(rec, "score", {"log-probabilities": lp, "next logits": dm.forward(toks[130], 130)})
    return rec


def test_another_model_in_between(open_model):
    """release, two other models (k_attn at head_dim 256; a Mixtral-width MoE) and llama again from the same tensors: the
    kernels' shared-memory opt-ins have only grown and the prompt pass's buffers were freed and rebuilt in between."""
    with open_model("llama", 16) as dm:
        first = llama_session(dm)
    for other, kvbits in (("tiny-hd256", 8), ("mixtral-1", 16)):
        with open_model(other, kvbits) as dm:
            toks = toks_of(dm, 40, start=3)
            dm.prefill(toks[:32], 0)
            logits = [dm.forward(t, 32 + i) for i, t in enumerate(toks[32:])]
            assert np.isfinite(logits).all()
            dm.decode_sample(5, 40, 4, 1.0, 0.1, 7)
    with open_model("llama", 16) as dm:
        again = llama_session(dm)
    assert_identical(first, again, "llama, before and after two other models")
