"""calm_b200_score_batch: many independent sequences, each scored from position 0, packed into shared prompt-pass blocks.

Every stage of the pass works per row except attention and RoPE, which the packed block runs per sequence (k_pf_attn<..,
SEG> starts each sequence's key tiles at its own first row, k_pf_rope_rows takes per-row positions).  So the claim is
exact: each sequence's log-probabilities equal, bit for bit, what calm_b200_score gives for that sequence alone.

- Packed equals alone in every weight format, both caches, both head sizes, across block boundaries, with sequences that
  fill a block exactly, sequences too long for a block, a short seq_len and Llama-3-8B widths at vocabulary 128256.
- Packing order does not matter; slots no sequence writes are left alone.
- The decode-path fallback (MoE, head_dim 32, a sequence longer than seq_len) returns 0 with the lone call's values.
- No result depends on what earlier calls left behind, and nothing after a batch depends on it either.

The call is calm_b200_score_context with every context empty; the helpers are test_score_context_gpu.py's, and a case
here is its layout with ctx_off = ctx_len = 0."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_score_context_gpu import (SENTINEL, assert_independent_of_history, assert_nothing_after_depends_on_it,  # noqa: E402
                                    assert_order_does_not_matter, check, fresh_results)

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu


def pack(vocab, lens, seed):
    """Random sequences of the given lengths, concatenated, with empty contexts: (tokens, ctx_off, ctx_len, off, len)."""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
    zero = np.zeros(len(lens), np.int32)
    return rng.integers(0, vocab, int(sum(lens))).astype(np.int32), zero, zero, off, np.asarray(lens, np.int32)


def study_chunks(n_tokens, steps):
    """study()'s chunks of a text: chunk c scores positions c * steps .. and shares its last token with chunk c + 1."""
    off = np.arange(0, n_tokens - 1, steps, dtype=np.int32)
    return off, np.minimum(steps + 1, n_tokens - off).astype(np.int32)


# pf-tiny at seq_len 512: capacity 512 rows.  Rows rounded up to 8: 8, 8, 16, 40, 136, 264 (one block of 472), then 512 (a
# block of exactly capacity rows), then 0, 264, 136, 40 (a third block); len 1 and len 0 contribute nothing.
LENS = [2, 3, 9, 40, 129, 257, 513, 1, 257, 129, 40, 0]


@pytest.mark.parametrize("name,dtype,kvbits", [("pf-tiny", "fp8", 16), ("pf-tiny", "fp8", 8), ("pf-tiny", "fp16", 16), ("pf-tiny", "fp16", 8),
                                               ("pf-tiny", "gf4", 16), ("pf-tiny", "gf4", 8), ("pf-tiny-hd128", "fp8", 16), ("pf-tiny-hd128", "gf4", 8)])
def test_packed_equals_alone(name, dtype, kvbits):
    spec = replace(mg.SPECS[name], dtype=dtype)
    tensors = mg.generate(spec, 11)
    check(spec, tensors, pack(spec.vocab_size, LENS, 1), f"{name}/{dtype}/kv{kvbits}", seq_len=512, kvbits=kvbits, batch=True)


def test_study_chunks_equal_the_per_chunk_loop():
    """A 3000-token text in study() chunks of 256: one batch call against the INTEGRATION.md loop of calm_b200_score
    calls, position by position over the whole output."""
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 12)
    n = 3000
    tokens = np.asarray(mg.teacher_tokens(spec.vocab_size, n), np.int32)
    off, lens = study_chunks(n, 256)
    zero = np.zeros(len(off), np.int32)
    got = check(spec, tensors, (tokens, zero, zero, off, lens), "study chunks", seq_len=4096, batch=True)
    with lib.DeviceModel(spec, tensors, seq_len=4096) as dm:
        loop = np.full(n, SENTINEL, np.float32)
        for c in range(0, n - 1, 256):
            m = min(n - 1 - c, 256)
            loop[c:c + m], served = dm.score(tokens[c:c + m + 1], 0)
            assert served == 1
    assert np.array_equal(got[:n - 1], loop[:n - 1]) and got[n - 1] == SENTINEL


@pytest.mark.parametrize("seq_len,lens", [
    (4096, [50, 2100, 300, 9]),  # 2099 rows: longer than a block, scored alone in two blocks of calm_b200_score
    (300, [300, 297, 100, 50, 33]),  # capacity 296: 299 rows (304 rounded) go alone, 296 rows fill a block exactly
])
def test_sequences_longer_than_a_block(seq_len, lens):
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 13)
    check(spec, tensors, pack(spec.vocab_size, lens, 2), f"seq_len {seq_len}", seq_len=seq_len, batch=True)


def test_llama3_8b_widths():
    """Sixteen 129-token sequences: one block of 2048 rows, k_pf_attn<., 128, 4>, 1002 vocabulary tiles, the last partial."""
    spec = replace(mg.SPECS["llama3-8b-fp8"], n_layers=2)
    tensors = mg.generate(spec, 14, device="cuda")
    torch.cuda.synchronize()
    check(spec, tensors, pack(spec.vocab_size, [129] * 16, 3), "llama3-8b widths", seq_len=4096, batch=True)


def test_packing_order_does_not_matter():
    spec = mg.SPECS["pf-tiny"]
    tensors = mg.generate(spec, 15)
    assert_order_does_not_matter(spec, tensors, pack(spec.vocab_size, [7, 300, 2, 65, 129, 33, 400, 17, 256, 90], 4), batch=True)


@pytest.mark.parametrize("name,seq_len,lens", [("tiny-moe", None, [20, 2, 33, 9]), ("tiny-fp8", None, [20, 2, 33, 9]),
                                               ("pf-tiny", 64, [20, 80, 9])])
def test_falls_back_to_the_decode_path(name, seq_len, lens):
    """MoE and head_dim 32 score every sequence on the decode path; on pf-tiny, only the sequence longer than seq_len goes
    there.  Either way the call returns 0 and the lone calls' values."""
    spec = mg.SPECS[name]
    tensors = mg.generate(spec, 16)
    check(spec, tensors, pack(spec.vocab_size, lens, 6), name, seq_len=seq_len, served=0, batch=True)


# ---- history independence
HIST_LENS = [40, 129, 2, 257, 9, 63]


@pytest.fixture(scope="module")
def hist():
    return fresh_results(17, lambda vocab: pack(vocab, HIST_LENS, 7), batch=True)


@pytest.mark.parametrize("before", ["poison", "score", "prefill", "score+poison"])
def test_batch_does_not_depend_on_history(hist, before):
    assert_independent_of_history(hist, before, batch=True)


def test_nothing_after_a_batch_depends_on_it(hist):
    assert_nothing_after_depends_on_it(hist, batch=True)
