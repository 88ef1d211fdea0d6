"""ctypes binding of libcalm_b200.so -- the host-side mirror of the reference's backend interface.

The function names, argument meaning and error behaviour are the reference's
(run.c:22-25): upload_cuda / prepare_cuda / forward_cuda / perf_cuda.  There is
no CPU path behind these calls: loading fails loudly when the library has not
been built, and prepare_cuda aborts the process when no sm_90 device exists.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np

from .cstructs import FF_UPDATE_KV_ONLY, Transformer
from . import modelgen as mg

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcalm_b200.so")
_fptr = C.POINTER(C.c_float)

# every symbol include/calm_b200.h declares
SYMBOLS = [
    "upload_cuda", "prepare_cuda", "forward_cuda", "perf_cuda", "forward_prefill_cuda", "calm_b200_score", "calm_b200_score_batch", "calm_b200_score_context",
    "calm_b200_score_greedy", "calm_b200_score_batch_greedy", "calm_b200_score_context_greedy",
    "calm_b200_score_topk", "calm_b200_score_batch_topk", "calm_b200_score_context_topk",
    "calm_b200_abi_version", "calm_b200_set_device", "calm_b200_free", "calm_b200_release",
    "calm_b200_forward_argmax", "calm_b200_decode_greedy", "calm_b200_verify_greedy", "calm_b200_decode_lookup", "calm_b200_verify_sample", "calm_b200_decode_lookup_sample",
    "calm_b200_decode_sample_n", "calm_b200_decode_sample_batch", "calm_b200_decode_beam", "calm_b200_decode_sample_queue",
    "calm_b200_decode_sample_queue_context", "calm_b200_decode_sample_queue_logprobs", "calm_b200_decode_sample_queue_penalties",
    "calm_b200_decode_sample_queue_constrained", "calm_b200_decode_sample_queue_truncated", "calm_b200_decode_sample_queue_lookup",
    "calm_b200_timer_start", "calm_b200_timer_stop",
    "calm_b200_stream", "calm_b200_launch_count", "calm_b200_read_kv", "calm_b200_read_state", "calm_b200_poison_state", "calm_b200_fill_kv", "calm_b200_matvec",
    "calm_b200_set_perf", "calm_b200_stage_stats", "calm_b200_perf_token_ms", "calm_b200_debug_stamps",
    "calm_b200_tp_unique_id", "calm_b200_tp_init", "calm_b200_tp_world", "calm_b200_tp_mode",
    "calm_b200_decode_sample", "calm_b200_forward_sample", "calm_b200_read_device_logits", "calm_b200_sample_logits",
    "calm_b200_sample_logits_truncated",
]

# the largest k calm_b200_score_topk and its siblings accept (CALM_B200_TOPK_MAX)
TOPK_MAX = 20

# the largest vocabulary calm_b200_decode_sample_queue_truncated and calm_b200_sample_logits_truncated truncate
TRUNC_VOCAB_MAX = 262144

# the largest block calm_b200_verify_greedy takes (CALM_B200_VERIFY_MAX); decode_lookup drafts at most one fewer
VERIFY_MAX = 16

# the most sequences calm_b200_decode_sample_n and calm_b200_decode_sample_batch sample together, and the most rows
# calm_b200_decode_sample_queue keeps in flight (CALM_B200_SAMPLE_N_MAX)
SAMPLE_N_MAX = 16

# the most beams calm_b200_decode_beam takes (CALM_B200_BEAM_MAX)
BEAM_MAX = 10

# calm_b200_read_state selectors (include/calm_b200.h)
STATE = {"x": 0, "xb": 1, "q": 2, "att": 3, "hb": 4, "moe_sel": 5, "keys": 6, "values": 7, "pf_x": 8, "pf_q": 9, "pf_att": 10, "pf_hb": 11, "pf_logits": 12,
         "beam_ids": 13, "beam_logprobs": 14, "beam_anc": 15}

_lib = None


def load() -> C.CDLL:
    """Load the product library.  Raises if it has not been built -- there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not built: run `python -m calm_b200.build` (CUDA extension is mandatory, no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    T = C.POINTER(Transformer)
    L.upload_cuda.argtypes, L.upload_cuda.restype = [C.c_void_p, C.c_size_t], C.c_void_p
    L.prepare_cuda.argtypes, L.prepare_cuda.restype = [T], None
    L.forward_cuda.argtypes, L.forward_cuda.restype = [T, C.c_int, C.c_int, C.c_uint], _fptr
    L.perf_cuda.argtypes, L.perf_cuda.restype = [], None
    L.forward_prefill_cuda.argtypes, L.forward_prefill_cuda.restype = [T, C.POINTER(C.c_int), C.c_int, C.c_int], C.c_int
    L.calm_b200_score.argtypes, L.calm_b200_score.restype = [T, C.POINTER(C.c_int), C.c_int, C.c_int, _fptr], C.c_int
    _iptr = C.POINTER(C.c_int)
    L.calm_b200_score_batch.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, C.c_int, _fptr]
    L.calm_b200_score_batch.restype = C.c_int
    L.calm_b200_score_context.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, _iptr, _iptr, C.c_int, _fptr]
    L.calm_b200_score_context.restype = C.c_int
    L.calm_b200_score_greedy.argtypes = [T, _iptr, C.c_int, C.c_int, _fptr, _iptr]
    L.calm_b200_score_greedy.restype = C.c_int
    L.calm_b200_score_batch_greedy.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, C.c_int, _fptr, _iptr]
    L.calm_b200_score_batch_greedy.restype = C.c_int
    L.calm_b200_score_context_greedy.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, _iptr, _iptr, C.c_int, _fptr, _iptr]
    L.calm_b200_score_context_greedy.restype = C.c_int
    L.calm_b200_score_topk.argtypes = [T, _iptr, C.c_int, C.c_int, C.c_int, _fptr, _iptr, _fptr]
    L.calm_b200_score_topk.restype = C.c_int
    L.calm_b200_score_batch_topk.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, C.c_int, C.c_int, _fptr, _iptr, _fptr]
    L.calm_b200_score_batch_topk.restype = C.c_int
    L.calm_b200_score_context_topk.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, _iptr, _iptr, C.c_int, C.c_int, _fptr, _iptr, _fptr]
    L.calm_b200_score_context_topk.restype = C.c_int
    L.calm_b200_abi_version.argtypes, L.calm_b200_abi_version.restype = [], C.c_int
    L.calm_b200_set_device.argtypes, L.calm_b200_set_device.restype = [C.c_int], None
    L.calm_b200_free.argtypes, L.calm_b200_free.restype = [C.c_void_p], None
    L.calm_b200_release.argtypes, L.calm_b200_release.restype = [T], None
    L.calm_b200_forward_argmax.argtypes, L.calm_b200_forward_argmax.restype = [T, C.c_int, C.c_int], C.c_int
    L.calm_b200_decode_greedy.argtypes, L.calm_b200_decode_greedy.restype = [T, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)], None
    L.calm_b200_verify_greedy.argtypes, L.calm_b200_verify_greedy.restype = [T, _iptr, C.c_int, C.c_int, _iptr], C.c_int
    L.calm_b200_decode_lookup.argtypes = [T, _iptr, C.c_int, C.c_int, _iptr, C.c_int, C.c_int, _iptr]
    L.calm_b200_decode_lookup.restype = C.c_int
    _u64p = C.POINTER(C.c_ulonglong)
    L.calm_b200_verify_sample.argtypes = [T, _iptr, C.c_int, C.c_int, C.c_float, C.c_float, _u64p, _iptr]
    L.calm_b200_verify_sample.restype = C.c_int
    L.calm_b200_decode_lookup_sample.argtypes = [T, _iptr, C.c_int, C.c_int, _iptr, C.c_int, C.c_int, C.c_float, C.c_float, _u64p, _iptr]
    L.calm_b200_decode_lookup_sample.restype = C.c_int
    L.calm_b200_decode_sample_n.argtypes = [T, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, _u64p, _iptr]
    L.calm_b200_decode_sample_n.restype = C.c_int
    L.calm_b200_decode_sample_batch.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, C.c_int, C.c_int, C.c_float, C.c_float, _u64p, _iptr]
    L.calm_b200_decode_sample_batch.restype = C.c_int
    L.calm_b200_decode_sample_queue.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, C.c_int, _iptr, _fptr, _fptr, _iptr, C.c_int, C.c_int, _u64p, _iptr,
                                                _iptr, _iptr]
    L.calm_b200_decode_sample_queue.restype = C.c_int
    L.calm_b200_decode_sample_queue_context.argtypes = [T, _iptr, C.c_int, _iptr, _iptr, _iptr, _iptr, C.c_int, _iptr, _fptr, _fptr, _iptr, C.c_int, C.c_int,
                                                        _u64p, _iptr, _iptr, _iptr, _iptr]
    L.calm_b200_decode_sample_queue_context.restype = C.c_int
    L.calm_b200_decode_sample_queue_logprobs.argtypes = L.calm_b200_decode_sample_queue_context.argtypes + [C.c_int, _fptr, _iptr, _fptr]
    L.calm_b200_decode_sample_queue_logprobs.restype = C.c_int
    ctx_args = L.calm_b200_decode_sample_queue_context.argtypes
    L.calm_b200_decode_sample_queue_penalties.argtypes = (ctx_args[:11] + [_fptr, _fptr, _fptr, _iptr, _iptr, _iptr, _fptr, C.c_int] + ctx_args[11:]
                                                          + [C.c_int, _fptr, _iptr, _fptr])
    L.calm_b200_decode_sample_queue_penalties.restype = C.c_int
    L.calm_b200_decode_sample_queue_constrained.argtypes = (L.calm_b200_decode_sample_queue_penalties.argtypes
                                                            + [C.c_int, C.POINTER(C.c_uint32), _iptr, _iptr, _iptr, _iptr, _iptr, _iptr])
    L.calm_b200_decode_sample_queue_constrained.restype = C.c_int
    L.calm_b200_decode_sample_queue_truncated.argtypes = L.calm_b200_decode_sample_queue_constrained.argtypes + [_iptr, _fptr]
    L.calm_b200_decode_sample_queue_truncated.restype = C.c_int
    L.calm_b200_decode_sample_queue_lookup.argtypes = L.calm_b200_decode_sample_queue_truncated.argtypes + [C.c_int, _iptr, _iptr]
    L.calm_b200_decode_sample_queue_lookup.restype = C.c_int
    L.calm_b200_decode_beam.argtypes = [T, C.c_int, C.c_int, C.c_int, C.c_int, _iptr, C.c_int, C.c_float, C.c_int, C.c_int, _iptr, _iptr, _fptr, _fptr, _iptr]
    L.calm_b200_decode_beam.restype = C.c_int
    L.calm_b200_timer_start.argtypes, L.calm_b200_timer_start.restype = [], None
    L.calm_b200_timer_stop.argtypes, L.calm_b200_timer_stop.restype = [], C.c_float
    L.calm_b200_stream.argtypes, L.calm_b200_stream.restype = [], C.c_void_p
    L.calm_b200_launch_count.argtypes, L.calm_b200_launch_count.restype = [], C.c_uint64
    L.calm_b200_read_kv.argtypes, L.calm_b200_read_kv.restype = [T, C.c_int, C.c_int, _fptr, _fptr], None
    L.calm_b200_read_state.argtypes, L.calm_b200_read_state.restype = [C.c_int, C.c_int, _fptr, C.c_int], C.c_int
    L.calm_b200_poison_state.argtypes, L.calm_b200_poison_state.restype = [T, C.c_int], None
    L.calm_b200_fill_kv.argtypes, L.calm_b200_fill_kv.restype = [T, C.c_int, C.c_uint64], None
    L.calm_b200_matvec.argtypes = [C.c_int, C.c_void_p, _fptr, _fptr, C.c_int, C.c_int, C.c_int, C.c_int]
    L.calm_b200_matvec.restype = C.c_float
    L.calm_b200_set_perf.argtypes, L.calm_b200_set_perf.restype = [C.c_int], None
    L.calm_b200_stage_stats.argtypes = [C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_long)]
    L.calm_b200_stage_stats.restype = C.c_int
    L.calm_b200_perf_token_ms.argtypes, L.calm_b200_perf_token_ms.restype = [], C.c_double
    L.calm_b200_debug_stamps.argtypes, L.calm_b200_debug_stamps.restype = [C.POINTER(C.c_ulonglong)], None
    L.calm_b200_tp_unique_id.argtypes, L.calm_b200_tp_unique_id.restype = [C.c_void_p], None
    L.calm_b200_tp_init.argtypes, L.calm_b200_tp_init.restype = [C.c_int, C.c_int, C.c_void_p], None
    L.calm_b200_tp_world.argtypes, L.calm_b200_tp_world.restype = [], C.c_int
    L.calm_b200_tp_mode.argtypes, L.calm_b200_tp_mode.restype = [], C.c_int
    L.calm_b200_decode_sample.argtypes = [T, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_ulonglong), C.POINTER(C.c_int)]
    L.calm_b200_decode_sample.restype = None
    L.calm_b200_forward_sample.argtypes = [T, C.c_int, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_ulonglong)]
    L.calm_b200_forward_sample.restype = C.c_int
    L.calm_b200_read_device_logits.argtypes, L.calm_b200_read_device_logits.restype = [_fptr], None
    L.calm_b200_sample_logits.argtypes = [_fptr, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_ulonglong), _fptr]
    L.calm_b200_sample_logits.restype = C.c_int
    L.calm_b200_sample_logits_truncated.argtypes = [_fptr, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, C.POINTER(C.c_ulonglong), _fptr, _fptr]
    L.calm_b200_sample_logits_truncated.restype = C.c_int
    _lib = L
    return L


def tp_unique_id() -> bytes:
    """128-byte NCCL id for calm_b200_tp_init; rank 0 makes it, every rank of the group receives it."""
    buf = C.create_string_buffer(128)
    load().calm_b200_tp_unique_id(buf)
    return buf.raw


def _check_rng(rng_state):
    """A generator state the C calls can take (a NULL state would abort the process)."""
    if not isinstance(rng_state, (int, np.integer)) or not 0 <= rng_state < 1 << 64:
        raise ValueError(f"rng_state must be an unsigned 64-bit integer, got {rng_state!r}")


class TokenAutomaton:
    """A finite token automaton for DeviceModel.decode_sample_queue_constrained, checked as the C call checks it.

    States are 0 .. n_states-1.  `allow` says which tokens each state allows: a bool array [n_states, vocab], or the C
    call's own bitmask, uint32 [n_states, ceil(vocab / 32)] with bit v % 32 of word v / 32 for token v.  After an
    allowed token v, state s moves to exceptions[s][v] when v is a key of that dict (exceptions may be None, and any
    entry None: no exceptions), otherwise to next_default[s]; -1 there means every allowed token is an exception.  A
    state that allows no token is final.  Raises ValueError for an automaton the C call would abort on."""

    def __init__(self, vocab: int, allow, next_default, exceptions=None):
        if not isinstance(vocab, (int, np.integer)) or isinstance(vocab, bool) or vocab < 1:
            raise ValueError(f"vocab must be a positive integer, got {vocab!r}")
        self.vocab, self.words = int(vocab), (int(vocab) + 31) // 32
        a = np.asarray(allow)
        if a.ndim != 2:
            raise ValueError("allow must be a 2-D array, one row per state")
        if a.dtype == np.bool_:
            if a.shape[1] != self.vocab:
                raise ValueError(f"a bool allow has one column per token: {a.shape[1]} columns, {self.vocab} tokens")
            bits = np.zeros((a.shape[0], self.words * 32), np.uint8)
            bits[:, :self.vocab] = a
            a = np.packbits(bits.reshape(a.shape[0], self.words, 4, 8), axis=-1, bitorder="little").reshape(a.shape[0], -1).view("<u4")
        elif a.dtype != np.uint32 or a.shape[1] != self.words:
            raise ValueError(f"allow must be bool [n_states, {self.vocab}] or uint32 [n_states, {self.words}], got {a.dtype} {a.shape}")
        self.allow = np.ascontiguousarray(a, np.uint32)
        self.n_states = n = self.allow.shape[0]
        if self.vocab % 32 and (self.allow[:, -1] >> np.uint32(self.vocab % 32)).any():
            raise ValueError(f"allow has a bit set past the {self.vocab}-token vocabulary")
        nd = np.asarray(next_default)
        if nd.shape != (n,) or (n and nd.dtype.kind not in "iu"):
            raise ValueError(f"next_default must hold one integer per state ({n})")
        if ((nd < -1) | (nd >= n)).any():
            raise ValueError(f"a default next state is outside [-1, {n})")
        self.next_default = np.ascontiguousarray(nd, np.int32)
        exceptions = [None] * n if exceptions is None else list(exceptions)
        if len(exceptions) != n:
            raise ValueError(f"exceptions must hold one dict (or None) per state ({n}), got {len(exceptions)}")
        off, tok, nxt = [0], [], []
        self.allowed_count = np.array([int(np.unpackbits(r.view(np.uint8)).sum()) for r in self.allow], np.int64)
        for s, d in enumerate(exceptions):
            d = {} if d is None else d
            if not isinstance(d, dict):
                raise ValueError(f"exceptions[{s}] must be a dict of token: next state, or None")
            for v in sorted(d):
                t = d[v]
                if not isinstance(v, (int, np.integer)) or isinstance(v, bool) or not 0 <= v < self.vocab or not self._bit(s, v):
                    raise ValueError(f"state {s}'s exception token {v!r} is not a token it allows")
                if not isinstance(t, (int, np.integer)) or isinstance(t, bool) or not 0 <= t < n:
                    raise ValueError(f"state {s}'s exception for token {v} goes to {t!r}, outside [0, {n})")
                tok.append(int(v)), nxt.append(int(t))
            off.append(len(tok))
            if self.next_default[s] == -1 and self.allowed_count[s] > len(d):
                raise ValueError(f"state {s} allows a token outside its exceptions and has no default next state")
        self.exc_off, self.exc_tok, self.exc_next = (np.asarray(x, np.int32) for x in (off, tok, nxt))
        self.final = self.allowed_count == 0

    def _bit(self, s, v):
        return bool((int(self.allow[s, v >> 5]) >> (v & 31)) & 1)

    def allowed(self, s: int) -> np.ndarray:
        """The ids state s allows, ascending."""
        bits = np.unpackbits(self.allow[s].view(np.uint8), bitorder="little")[:self.vocab]
        return np.flatnonzero(bits)

    def next(self, s: int, token: int) -> int:
        """The state after `token` in state s, or ValueError if s does not allow it."""
        if not 0 <= s < self.n_states or not 0 <= token < self.vocab or not self._bit(s, token):
            raise ValueError(f"state {s} does not allow token {token}")
        lo, hi = self.exc_off[s], self.exc_off[s + 1]
        j = lo + int(np.searchsorted(self.exc_tok[lo:hi], token))
        return int(self.exc_next[j]) if j < hi and self.exc_tok[j] == token else int(self.next_default[s])

    @classmethod
    def choices(cls, seqs, vocab: int) -> "TokenAutomaton":
        """guided_choice: a trie over the token sequences `seqs`, from state 0, whose every leaf is the one final state,
        so that a constrained request emits exactly one of them.  ValueError for an empty list, an empty sequence, an id
        outside [0, vocab) or a sequence that is a proper prefix of another (it could not both end and go on)."""
        seqs = [[int(t) for t in q] for q in seqs]
        if not seqs or any(len(q) == 0 for q in seqs):
            raise ValueError("choices takes at least one sequence, none of them empty")
        if any(not 0 <= t < vocab for q in seqs for t in q):
            raise ValueError(f"a choice has a token outside [0, {vocab})")
        END = -1
        nodes = [{}]  # node -> {token: child node, or END}
        for q in seqs:
            u = 0
            for j, t in enumerate(q):
                last = j == len(q) - 1
                c = nodes[u].get(t)
                if (c == END) != last and c is not None:
                    raise ValueError(f"choice {q} and another: one is a proper prefix of the other")
                if last:
                    nodes[u][t] = END
                else:
                    if c is None:
                        c = nodes[u][t] = len(nodes)
                        nodes.append({})
                    u = c
        fin = len(nodes)
        allow = np.zeros((fin + 1, vocab), bool)
        exc = [None] * (fin + 1)
        for u, ch in enumerate(nodes):
            allow[u, list(ch)] = True
            exc[u] = {t: (fin if c == END else c) for t, c in ch.items()}
        return cls(vocab, allow, np.full(fin + 1, -1, np.int32), exc)


class DeviceModel:
    """A model on the GPU behind the reference boundary.

    Mirrors what the reference driver does around the backend (run.c:552-582):
    upload every model.* tensor with upload_cuda, bind the returned device pointers
    in struct Weights, call prepare_cuda, then forward_cuda once per token.
    `tensors` may hold host tensors (uploaded through upload_cuda) or tensors that
    already live on the device (their data_ptr is used directly, which is what
    struct Weights carries after upload anyway).
    """

    def __init__(self, spec: mg.ModelSpec, tensors: Dict[str, "object"], seq_len: Optional[int] = None, kvbits: int = 16,
                 device: Optional[int] = None, tp=None):
        """tp = (rank, world, id128) turns on tensor parallelism (include/calm_b200.h); tensors stay the FULL model."""
        self.lib = load()
        self.spec = spec
        if device is not None:
            self.lib.calm_b200_set_device(device)
        if tp is not None:
            self.lib.calm_b200_tp_init(int(tp[0]), int(tp[1]), C.c_char_p(tp[2]) if tp[2] else None)
        self._uploaded = []
        self._keep = tensors
        ptrs = {}
        for name, t in tensors.items():
            if getattr(t, "is_cuda", False):
                ptrs[name] = t.data_ptr()
            else:
                t = t.contiguous()
                nbytes = t.numel() * t.element_size()
                p = self.lib.upload_cuda(t.data_ptr(), nbytes)
                self._uploaded.append(p)
                ptrs[name] = p
        self.transformer = mg.fill_transformer(spec, lambda n: ptrs.get(n, 0), seq_len, kvbits)
        self.lib.prepare_cuda(C.byref(self.transformer))
        self.vocab = spec.vocab_size

    @property
    def seq_len(self) -> int:
        return self.transformer.config.seq_len

    def forward(self, token: int, pos: int, flags: int = 0):
        """forward_cuda; returns a COPY of the host logits, or None for FF_UPDATE_KV_ONLY."""
        p = self.lib.forward_cuda(C.byref(self.transformer), token, pos, flags)
        if not p:
            return None
        return np.ctypeslib.as_array(p, shape=(self.vocab,)).copy()

    def prefill(self, tokens, pos0: int = 0) -> int:
        """forward_prefill_cuda: the batched prompt pass; returns 1 (tensor-core pass) or 0 (fed token by token)."""
        arr = np.ascontiguousarray(tokens, np.int32)
        return self.lib.forward_prefill_cuda(C.byref(self.transformer), arr.ctypes.data_as(C.POINTER(C.c_int)), len(arr), pos0)

    def score(self, tokens, pos0: int = 0):
        """calm_b200_score: (log-probabilities of tokens[1:] after what precedes each, as float32[n - 1], 1 when the
        tensor-core pass served it or 0 when the decode path did)."""
        arr = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros(max(len(arr) - 1, 0), np.float32)
        served = self.lib.calm_b200_score(C.byref(self.transformer), arr.ctypes.data_as(C.POINTER(C.c_int)), len(arr), pos0, out.ctypes.data_as(_fptr))
        return out, served

    def _check_k(self, k):
        """The binding's copy of the library's check on k, raised before the library would abort the process."""
        kmax = min(TOPK_MAX, self.vocab)
        if not isinstance(k, (int, np.integer)) or not 1 <= k <= kmax:
            raise ValueError(f"k must be an integer in [1, {kmax}], got {k!r}")
        return int(k)

    def _score_packed(self, fn, tokens, index, out, greedy=None, with_greedy=False, k=None, top=None):
        """Call the packed scoring symbol `fn` over `tokens`.  `index` holds its per-sequence arrays in the C argument order
        ((off, len) or (ctx_off, ctx_len, off, len)).  `out` defaults to NaN, and for a greedy symbol (`with_greedy`)
        `greedy` to -1.  Returns (out, served), or (out, greedy, served) with `with_greedy`.  With `k`, a top-k symbol:
        `top` = (top_ids int32[n, k], top_logprobs float32[n, k]) defaults to -1 / NaN, and the result is
        (out, top_ids, top_logprobs, served)."""
        ip = C.POINTER(C.c_int)
        arr = np.ascontiguousarray(tokens, np.int32)
        index = [np.ascontiguousarray(a, np.int32) for a in index]
        assert index[0].ndim == 1 and all(a.shape == index[0].shape for a in index)
        n = len(arr)
        if out is None:
            out = np.full(n, np.nan, np.float32)
        assert out.dtype == np.float32 and out.flags.c_contiguous and len(out) >= n
        outs = [out.ctypes.data_as(_fptr)]
        if with_greedy:
            if greedy is None:
                greedy = np.full(n, -1, np.int32)
            assert greedy.dtype == np.int32 and greedy.flags.c_contiguous and len(greedy) >= n
            outs.append(greedy.ctypes.data_as(ip))
        if k is not None:
            k = self._check_k(k)
            ids, tlp = top if top is not None else (np.full((n, k), -1, np.int32), np.full((n, k), np.nan, np.float32))
            assert ids.dtype == np.int32 and tlp.dtype == np.float32 and ids.flags.c_contiguous and tlp.flags.c_contiguous
            assert ids.shape[1:] == (k,) == tlp.shape[1:] and len(ids) >= n and len(tlp) >= n
            served = fn(C.byref(self.transformer), arr.ctypes.data_as(ip), n, *[a.ctypes.data_as(ip) for a in index], len(index[0]), k, *outs,
                        ids.ctypes.data_as(ip), tlp.ctypes.data_as(_fptr))
            return out, ids, tlp, served
        served = fn(C.byref(self.transformer), arr.ctypes.data_as(ip), n, *[a.ctypes.data_as(ip) for a in index], len(index[0]), *outs)
        return (out, greedy, served) if with_greedy else (out, served)

    def score_batch(self, tokens, off, len_, out=None):
        """calm_b200_score_batch: independent sequences tokens[off[i] : off[i] + len_[i]], each scored from position 0 and
        packed into shared prompt-pass blocks.  Returns (float32[len(tokens)] with sequence i's log-probabilities at
        off[i] .. off[i] + len_[i] - 2, 1 when the tensor-core pass served every sequence or 0).  Slots no sequence writes
        keep what `out` held (NaN when no `out` is given)."""
        return self._score_packed(self.lib.calm_b200_score_batch, tokens, (off, len_), out)

    def score_context(self, tokens, ctx_off, ctx_len, off, len_, out=None):
        """calm_b200_score_context: sequences tokens[off[i] : off[i] + len_[i]], each continuing the context
        tokens[ctx_off[i] : ctx_off[i] + ctx_len[i]], packed into shared prompt-pass blocks with each context computed once
        per block.  Returns (float32[len(tokens)] with sequence i's log-probabilities at off[i] .. off[i] + len_[i] - 2, 1
        when the tensor-core pass served every sequence or 0).  Slots no sequence writes keep what `out` held (NaN when no
        `out` is given)."""
        return self._score_packed(self.lib.calm_b200_score_context, tokens, (ctx_off, ctx_len, off, len_), out)

    def score_greedy(self, tokens, pos0: int = 0):
        """calm_b200_score_greedy: score()'s log-probabilities, bit for bit, and the argmax of the logits at each scored
        position (lowest index on ties).  Returns (float32[n - 1], int32[n - 1], served)."""
        arr = np.ascontiguousarray(tokens, np.int32)
        out = np.full(max(len(arr) - 1, 0), np.nan, np.float32)
        greedy = np.full(len(out), -1, np.int32)
        ip = C.POINTER(C.c_int)
        served = self.lib.calm_b200_score_greedy(C.byref(self.transformer), arr.ctypes.data_as(ip), len(arr), pos0, out.ctypes.data_as(_fptr),
                                                 greedy.ctypes.data_as(ip))
        return out, greedy, served

    def score_batch_greedy(self, tokens, off, len_, out=None, greedy=None):
        """calm_b200_score_batch_greedy: score_batch()'s log-probabilities, bit for bit, and the greedy token at the same
        slots.  Returns (float32[len(tokens)], int32[len(tokens)], served); unwritten slots keep what `out` / `greedy` held
        (NaN / -1 when not given)."""
        return self._score_packed(self.lib.calm_b200_score_batch_greedy, tokens, (off, len_), out, greedy, with_greedy=True)

    def score_context_greedy(self, tokens, ctx_off, ctx_len, off, len_, out=None, greedy=None):
        """calm_b200_score_context_greedy: score_context()'s log-probabilities, bit for bit, and the greedy token at the
        same slots.  Returns (float32[len(tokens)], int32[len(tokens)], served); unwritten slots keep what `out` / `greedy`
        held (NaN / -1 when not given)."""
        return self._score_packed(self.lib.calm_b200_score_context_greedy, tokens, (ctx_off, ctx_len, off, len_), out, greedy, with_greedy=True)

    def score_topk(self, tokens, k: int, pos0: int = 0):
        """calm_b200_score_topk: score()'s log-probabilities, bit for bit, and at each scored position the k most likely
        tokens (logit descending, lowest index on ties) with their log-probabilities.  Returns (float32[n - 1],
        int32[n - 1, k], float32[n - 1, k], served).  Raises ValueError unless 1 <= k <= min(TOPK_MAX, vocab)."""
        k = self._check_k(k)
        arr = np.ascontiguousarray(tokens, np.int32)
        out = np.full(max(len(arr) - 1, 0), np.nan, np.float32)
        ids = np.full((len(out), k), -1, np.int32)
        tlp = np.full((len(out), k), np.nan, np.float32)
        ip = C.POINTER(C.c_int)
        served = self.lib.calm_b200_score_topk(C.byref(self.transformer), arr.ctypes.data_as(ip), len(arr), pos0, k, out.ctypes.data_as(_fptr),
                                               ids.ctypes.data_as(ip), tlp.ctypes.data_as(_fptr))
        return out, ids, tlp, served

    def score_batch_topk(self, tokens, off, len_, k: int, out=None, top=None):
        """calm_b200_score_batch_topk: score_batch()'s log-probabilities, bit for bit, and the top-k ids and
        log-probabilities at the same slots.  Returns (float32[len(tokens)], int32[len(tokens), k], float32[len(tokens), k],
        served); unwritten slots keep what `out` / `top` = (ids, logprobs) held (NaN / -1 / NaN when not given)."""
        return self._score_packed(self.lib.calm_b200_score_batch_topk, tokens, (off, len_), out, k=k, top=top)

    def score_context_topk(self, tokens, ctx_off, ctx_len, off, len_, k: int, out=None, top=None):
        """calm_b200_score_context_topk: score_context()'s log-probabilities, bit for bit, and the top-k ids and
        log-probabilities at the same slots.  Returns (float32[len(tokens)], int32[len(tokens), k], float32[len(tokens), k],
        served); unwritten slots keep what `out` / `top` = (ids, logprobs) held (NaN / -1 / NaN when not given)."""
        return self._score_packed(self.lib.calm_b200_score_context_topk, tokens, (ctx_off, ctx_len, off, len_), out, k=k, top=top)

    def forward_raw(self, token: int, pos: int, flags: int = 0):
        return self.lib.forward_cuda(C.byref(self.transformer), token, pos, flags)

    def forward_argmax(self, token: int, pos: int) -> int:
        return self.lib.calm_b200_forward_argmax(C.byref(self.transformer), token, pos)

    def decode_greedy(self, token0: int, pos0: int, n: int) -> np.ndarray:
        out = np.zeros(n, np.int32)
        self.lib.calm_b200_decode_greedy(C.byref(self.transformer), token0, pos0, n, out.ctypes.data_as(C.POINTER(C.c_int)))
        return out

    @staticmethod
    def _verify_block(tokens, who):
        """The verify calls' tokens as int32, or ValueError for a bad length."""
        arr = np.ascontiguousarray(tokens, np.int32)
        if arr.ndim != 1 or not 1 <= len(arr) <= VERIFY_MAX:
            raise ValueError(f"{who} takes 1 to {VERIFY_MAX} tokens, got {arr.shape}")
        return arr

    def verify_greedy(self, tokens, pos0: int):
        """calm_b200_verify_greedy: feed tokens (1 .. VERIFY_MAX of them) at pos0 .. and return (greedy int32[n], served):
        greedy[i] is the argmax of the logits after tokens[i], served is 1 on the short-block path or 0 when n
        forward_argmax calls gave them.  Raises ValueError for a bad length."""
        arr = self._verify_block(tokens, "verify_greedy")
        greedy = np.full(len(arr), -1, np.int32)
        ip = C.POINTER(C.c_int)
        served = self.lib.calm_b200_verify_greedy(C.byref(self.transformer), arr.ctypes.data_as(ip), len(arr), pos0, greedy.ctypes.data_as(ip))
        return greedy, served

    def verify_sample(self, tokens, pos0: int, temperature: float, minp: float, rng_state: int):
        """calm_b200_verify_sample: feed tokens (1 .. VERIFY_MAX of them) at pos0 .. and return (sampled int32[n], new rng
        state, served): sampled[i] is the reference sampler's draw on the logits after tokens[i] with the (i + 1)-th coin of
        rng_state, and the new state is rng_state advanced by the draws the caller emits (the accepted drafts plus one).
        served is 1 on the short-block path or 0 when forward_sample calls gave them.  Raises ValueError for a bad length or
        rng_state."""
        if tokens is None:
            raise ValueError("verify_sample needs tokens")
        arr = self._verify_block(tokens, "verify_sample")
        _check_rng(rng_state)
        sampled = np.full(len(arr), -1, np.int32)
        ip = C.POINTER(C.c_int)
        rng = C.c_ulonglong(rng_state)
        served = self.lib.calm_b200_verify_sample(C.byref(self.transformer), arr.ctypes.data_as(ip), len(arr), pos0, temperature, minp, C.byref(rng),
                                                  sampled.ctypes.data_as(ip))
        return sampled, int(rng.value), served

    @staticmethod
    def _lookup_args(tokens, n_tokens, source, max_draft, who):
        """The lookup calls' (tokens, out, source) arrays, or ValueError for an empty `tokens`, a negative n_tokens or
        max_draft outside [1, VERIFY_MAX - 1]."""
        arr = np.ascontiguousarray(tokens, np.int32)
        if arr.ndim != 1 or len(arr) < 1:
            raise ValueError(f"{who} needs at least one token")
        if not isinstance(n_tokens, (int, np.integer)) or n_tokens < 0:
            raise ValueError(f"n_tokens must be a non-negative integer, got {n_tokens!r}")
        if not isinstance(max_draft, (int, np.integer)) or not 1 <= max_draft < VERIFY_MAX:
            raise ValueError(f"max_draft must be an integer in [1, {VERIFY_MAX - 1}], got {max_draft!r}")
        src = None if source is None else np.ascontiguousarray(source, np.int32)
        return arr, np.full(int(n_tokens), -1, np.int32), src

    def decode_lookup(self, tokens, n_tokens: int, source=None, max_draft: int = 7):
        """calm_b200_decode_lookup: greedy decoding with prompt-lookup drafts after `tokens` (the cache holds all but the
        last).  The drafts come from `source`, or from tokens ++ emitted when it is None.  Returns (int32[n_tokens],
        model steps run).  Raises ValueError for an empty `tokens`, a negative n_tokens or max_draft outside
        [1, VERIFY_MAX - 1]."""
        arr, out, src = self._lookup_args(tokens, n_tokens, source, max_draft, "decode_lookup")
        ip = C.POINTER(C.c_int)
        steps = self.lib.calm_b200_decode_lookup(C.byref(self.transformer), arr.ctypes.data_as(ip), len(arr), int(n_tokens),
                                                 None if src is None else src.ctypes.data_as(ip), 0 if src is None else len(src), int(max_draft),
                                                 out.ctypes.data_as(ip))
        return out, steps

    def decode_lookup_sample(self, tokens, n_tokens: int, temperature: float, minp: float, rng_state: int, source=None, max_draft: int = 7):
        """calm_b200_decode_lookup_sample: decode_lookup's loop with temperature / min-p sampling, each draft accepted
        exactly when the sampled token equals it.  Returns (int32[n_tokens], model steps run, new rng state); the state is
        where decode_sample of the same tokens leaves it.  Raises ValueError where decode_lookup does, and for a bad
        rng_state."""
        if tokens is None:
            raise ValueError("decode_lookup_sample needs at least one token")
        arr, out, src = self._lookup_args(tokens, n_tokens, source, max_draft, "decode_lookup_sample")
        _check_rng(rng_state)
        ip = C.POINTER(C.c_int)
        rng = C.c_ulonglong(rng_state)
        steps = self.lib.calm_b200_decode_lookup_sample(C.byref(self.transformer), arr.ctypes.data_as(ip), len(arr), int(n_tokens),
                                                        None if src is None else src.ctypes.data_as(ip), 0 if src is None else len(src), int(max_draft),
                                                        temperature, minp, C.byref(rng), out.ctypes.data_as(ip))
        return out, steps, int(rng.value)

    def decode_sample(self, token0: int, pos0: int, n: int, temperature: float, minp: float, rng_state: int):
        """Device-resident temperature / min-p sampling; returns (tokens, new rng state)."""
        out = np.zeros(n, np.int32)
        rng = C.c_ulonglong(rng_state)
        self.lib.calm_b200_decode_sample(C.byref(self.transformer), token0, pos0, n, temperature, minp, C.byref(rng), out.ctypes.data_as(C.POINTER(C.c_int)))
        return out, int(rng.value)

    def decode_sample_n(self, token0: int, pos0: int, n_tokens: int, temperature: float, minp: float, rng_states):
        """calm_b200_decode_sample_n: len(rng_states) = nseq continuations of the prompt in cache slots [0, pos0), each
        feeding token0 at pos0 and then its own samples, as decode_sample(token0, pos0, n_tokens, ..., rng_states[b])
        would.  Returns (tokens int32[nseq, n_tokens], the nseq new generator states, served): served is 1 on the
        shared-prompt path, 0 when nseq decode_sample runs gave them (shapes the prompt pass does not serve, or
        pos0 + nseq * n_tokens > seq_len).  Raises ValueError for 0 or more than SAMPLE_N_MAX states, a bad state, a
        negative n_tokens or pos0, or token0 outside the vocabulary."""
        if rng_states is None or isinstance(rng_states, (int, np.integer)):
            raise ValueError("decode_sample_n takes a sequence of generator states, one per sequence")
        states = list(rng_states)
        if not 1 <= len(states) <= SAMPLE_N_MAX:
            raise ValueError(f"decode_sample_n samples 1 to {SAMPLE_N_MAX} sequences, got {len(states)} states")
        for s in states:
            _check_rng(s)
        if not isinstance(n_tokens, (int, np.integer)) or n_tokens < 0:
            raise ValueError(f"n_tokens must be a non-negative integer, got {n_tokens!r}")
        if not isinstance(token0, (int, np.integer)) or not 0 <= token0 < self.vocab:
            raise ValueError(f"token0 must be in [0, {self.vocab}), got {token0!r}")
        if not isinstance(pos0, (int, np.integer)) or pos0 < 0:
            raise ValueError(f"pos0 must be a non-negative integer, got {pos0!r}")
        nseq = len(states)
        rng = (C.c_ulonglong * nseq)(*[int(s) for s in states])
        out = np.full((nseq, int(n_tokens)), -1, np.int32)
        served = self.lib.calm_b200_decode_sample_n(C.byref(self.transformer), int(token0), int(pos0), int(n_tokens), nseq, temperature, minp, rng,
                                                    out.ctypes.data_as(C.POINTER(C.c_int)))
        return out, [int(s) for s in rng], served

    def decode_beam(self, token0: int, pos0: int, max_new: int, num_beams: int, stop=(), length_penalty: float = 1.0, early_stopping: bool = False,
                    num_return: Optional[int] = None):
        """calm_b200_decode_beam: beam search over the prompt in cache slots [0, pos0), feeding token0 at pos0, with
        include/calm_b200.h's rules (Hugging Face's num_beams, length_penalty, early_stopping, num_return_sequences and
        eos_token_id = stop).  Returns (hypotheses, served, steps): hypotheses is a list of num_return (default num_beams)
        tuples (tokens int32[len], logprobs float32[len], score), best first, or [] when served is 0 (MoE, tensor-parallel
        or unserved shapes, or pos0 + num_beams * max_new > seq_len).  Raises ValueError wherever the C call would abort."""
        def whole(name, x, lo, hi):
            if isinstance(x, bool) or not isinstance(x, (int, np.integer)) or not lo <= x <= hi:
                raise ValueError(f"decode_beam: {name} must be an integer in [{lo}, {hi}], got {x!r}")
            return int(x)

        B = whole("num_beams", num_beams, 1, BEAM_MAX)
        max_new = whole("max_new", max_new, 0, 1 << 31)
        pos0 = whole("pos0", pos0, 0, 1 << 31)
        token0 = whole("token0", token0, 0, self.vocab - 1)
        R = B if num_return is None else whole("num_return", num_return, 1, B)
        if early_stopping not in (0, 1):  # (True and False included)
            raise ValueError(f"decode_beam: early_stopping must be 0 or 1, got {early_stopping!r}")
        try:
            stop = np.ascontiguousarray(np.asarray(list(stop), np.int64).reshape(-1))
        except (TypeError, ValueError) as e:
            raise ValueError(f"decode_beam: bad stop list: {e}") from None
        if ((stop < 0) | (stop >= self.vocab)).any():
            raise ValueError(f"decode_beam: stop ids must be in [0, {self.vocab})")
        K = max(2, 1 + len(stop)) * B
        if K > TOPK_MAX:
            raise ValueError(f"decode_beam: max(2, 1 + len(stop)) * num_beams = {K} candidates per beam exceed {TOPK_MAX}")
        if not np.isfinite(np.float32(length_penalty)):
            raise ValueError(f"decode_beam: length_penalty must be finite, got {length_penalty!r}")
        stop = stop.astype(np.int32)
        ip = C.POINTER(C.c_int)
        toks = np.full((R, max(max_new, 1)), -1, np.int32)
        lps = np.zeros((R, max(max_new, 1)), np.float32)
        lens, scores, steps = np.zeros(R, np.int32), np.zeros(R, np.float32), C.c_int(0)
        served = self.lib.calm_b200_decode_beam(C.byref(self.transformer), token0, pos0, max_new, B, stop.ctypes.data_as(ip), len(stop),
                                                float(length_penalty), int(early_stopping), R, toks.ctypes.data_as(ip), lens.ctypes.data_as(ip),
                                                lps.ctypes.data_as(_fptr), scores.ctypes.data_as(_fptr), C.byref(steps))
        if not served or max_new == 0:
            return [], served, 0
        return [(toks[r, :lens[r]].copy(), lps[r, :lens[r]].copy(), float(scores[r])) for r in range(R)], served, steps.value

    def decode_sample_batch(self, prompts, n_tokens: int, temperature: float, minp: float, rng_states):
        """calm_b200_decode_sample_batch: len(prompts) = nseq sequences, sequence b continuing prompts[b] (a sequence of at
        least one token id) as forward_prefill_cuda(prompts[b][:-1], 0) and then decode_sample(prompts[b][-1], len - 1,
        n_tokens, ..., rng_states[b]) would.  Returns (tokens int32[nseq, n_tokens], the nseq new generator states,
        served): served is 1 on the packed path, 0 when those per-sequence pairs gave them (shapes the prompt pass does
        not serve, or a layout past seq_len).  Raises ValueError for 0 or more than SAMPLE_N_MAX prompts, as many states
        as prompts not given, a bad state, a negative n_tokens, an empty prompt or a token outside the vocabulary."""
        if prompts is None or rng_states is None or isinstance(rng_states, (int, np.integer)):
            raise ValueError("decode_sample_batch takes a list of prompts and a sequence of generator states, one per prompt")
        prompts = [np.asarray(p) for p in prompts]
        states = list(rng_states)
        if not 1 <= len(prompts) <= SAMPLE_N_MAX:
            raise ValueError(f"decode_sample_batch samples 1 to {SAMPLE_N_MAX} sequences, got {len(prompts)} prompts")
        if len(states) != len(prompts):
            raise ValueError(f"decode_sample_batch takes one generator state per prompt: {len(prompts)} prompts, {len(states)} states")
        for s in states:
            _check_rng(s)
        if not isinstance(n_tokens, (int, np.integer)) or n_tokens < 0:
            raise ValueError(f"n_tokens must be a non-negative integer, got {n_tokens!r}")
        for b, p in enumerate(prompts):
            if p.ndim != 1 or len(p) < 1 or p.dtype.kind not in "iu":
                raise ValueError(f"prompt {b} must be a non-empty sequence of token ids")
            if not ((p >= 0) & (p < self.vocab)).all():
                raise ValueError(f"prompt {b} has a token outside [0, {self.vocab})")
        nseq = len(prompts)
        tokens = np.ascontiguousarray(np.concatenate(prompts), np.int32)
        len_ = np.asarray([len(p) for p in prompts], np.int32)
        off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(len_)[:-1]]), np.int32)
        rng = (C.c_ulonglong * nseq)(*[int(s) for s in states])
        out = np.full((nseq, int(n_tokens)), -1, np.int32)
        ip = C.POINTER(C.c_int)
        served = self.lib.calm_b200_decode_sample_batch(C.byref(self.transformer), tokens.ctypes.data_as(ip), len(tokens), off.ctypes.data_as(ip),
                                                        len_.ctypes.data_as(ip), nseq, int(n_tokens), temperature, minp, rng,
                                                        out.ctypes.data_as(ip))
        return out, [int(s) for s in rng], served

    def _queue_args(self, who, prompts, max_new, temperature, minp, stop, max_rows, rng_states):
        """The queue calls' checked per-request arrays (prompts, max_new, temperature, minp, stop, states), or ValueError
        wherever the C call would abort, and for per-request lists whose lengths differ."""
        if prompts is None or rng_states is None or isinstance(rng_states, (int, np.integer)):
            raise ValueError(f"{who} takes a list of prompts and a sequence of generator states, one per prompt")
        prompts = [np.asarray(p) for p in prompts]
        nreq = len(prompts)
        states = list(rng_states)
        try:
            max_new = [m for m in max_new]
            temperature = np.ascontiguousarray(temperature, np.float32).reshape(-1)
            minp = np.ascontiguousarray(minp, np.float32).reshape(-1)
            stop = np.asarray([] if stop is None else stop)
        except (TypeError, ValueError) as e:
            raise ValueError(f"{who}: bad per-request list: {e}") from None
        for name, xs in (("max_new", max_new), ("temperature", temperature), ("minp", minp), ("rng_states", states)):
            if len(xs) != nreq:
                raise ValueError(f"{who} takes one {name} per prompt: {nreq} prompts, {len(xs)} values")
        if not isinstance(max_rows, (int, np.integer)) or not 1 <= max_rows <= SAMPLE_N_MAX:
            raise ValueError(f"max_rows must be an integer in [1, {SAMPLE_N_MAX}], got {max_rows!r}")
        for s in states:
            _check_rng(s)
        for i, m in enumerate(max_new):
            if not isinstance(m, (int, np.integer)) or m < 0:
                raise ValueError(f"max_new[{i}] must be a non-negative integer, got {m!r}")
        for i, p in enumerate(prompts):
            if p.ndim != 1 or len(p) < 1 or p.dtype.kind not in "iu":
                raise ValueError(f"prompt {i} must be a non-empty sequence of token ids")
            if not ((p >= 0) & (p < self.vocab)).all():
                raise ValueError(f"prompt {i} has a token outside [0, {self.vocab})")
        if stop.ndim != 1 or (len(stop) and stop.dtype.kind not in "iu"):
            raise ValueError("stop must be a sequence of token ids")
        if not ((stop >= 0) & (stop < self.vocab)).all():
            raise ValueError(f"a stop id is outside [0, {self.vocab})")
        if sum(int(m) for m in max_new) >= 1 << 31:
            raise ValueError(f"{who}: the sum of max_new does not fit an int")
        return prompts, max_new, temperature, minp, stop, states

    def _queue_call(self, fn, tokens, ctx, off, len_, max_new, temperature, minp, stop, max_rows, states, k=None, pen=None, aut=None, trunc=None,
                    max_draft=None):
        """Run a queue call over the laid-out tokens; ctx is (ctx_off, ctx_len), either of them None for a NULL array, or
        None for a call without those arguments.  Returns (tokens, states, served, steps, prompt_rows), and with `k` (the
        log-probability call) also each request's float32[out_len] log-probabilities and, for k > 0, its top ids and
        log-probabilities [out_len, k] (None for k == 0).  `pen` (the penalty call) is the list of its arguments after
        minp; without `k` that call gets k 0 and NULL outputs.  `aut` (the constrained call) is the list of its automaton
        arguments before out_state; the return value then ends with each request's final state.  `trunc` (the truncated
        call) is its (top_k, top_p) pointers, after out_state.  `max_draft` (the lookup call) follows them; the return value
        then ends with (drafted, accepted)."""
        nreq = len(len_)
        mn = np.ascontiguousarray(max_new, np.int32)
        st = np.ascontiguousarray(stop, np.int32)
        rng = (C.c_ulonglong * max(nreq, 1))(*[int(s) for s in states])
        total = max(int(mn.sum()), 1)
        out = np.full(total, -1, np.int32)
        out_len = np.zeros(max(nreq, 1), np.int32)
        steps, rows = C.c_int(-1), C.c_int(-1)
        ip, fp = C.POINTER(C.c_int), C.POINTER(C.c_float)
        args = [C.byref(self.transformer), tokens.ctypes.data_as(ip), len(tokens)]
        if ctx is not None:
            args += [None if c is None else c.ctypes.data_as(ip) for c in ctx]
        args += [off.ctypes.data_as(ip), len_.ctypes.data_as(ip), nreq, mn.ctypes.data_as(ip), temperature.ctypes.data_as(fp), minp.ctypes.data_as(fp)]
        args += pen or []
        args += [st.ctypes.data_as(ip) if len(st) else None, len(st), int(max_rows), rng, out.ctypes.data_as(ip), out_len.ctypes.data_as(ip), C.byref(steps)]
        if ctx is not None:
            args.append(C.byref(rows))
        if k is not None:
            lp = np.full(total, np.nan, np.float32)
            ids = np.full((total, k), -1, np.int32) if k else None
            tlp = np.full((total, k), np.nan, np.float32) if k else None
            args += [k, lp.ctypes.data_as(fp), ids.ctypes.data_as(ip) if k else None, tlp.ctypes.data_as(fp) if k else None]
        elif pen is not None:
            args += [0, None, None, None]
        out_state = np.full(max(nreq, 1), -2, np.int32)
        if aut is not None:
            args += aut + [out_state.ctypes.data_as(ip)]
        if trunc is not None:
            args += trunc
        drafted, accepted = C.c_int(-1), C.c_int(-1)
        if max_draft is not None:
            args += [int(max_draft), C.byref(drafted), C.byref(accepted)]
        served = fn(*args)
        o = np.concatenate([[0], np.cumsum(mn)]).astype(np.int64)
        toks = [out[o[i]:o[i] + out_len[i]].copy() for i in range(nreq)]
        res = (toks, [int(rng[i]) for i in range(nreq)], served, int(steps.value), int(rows.value))
        if k is not None:
            cut = lambda a: [a[o[i]:o[i] + out_len[i]].copy() for i in range(nreq)] if a is not None else None  # noqa: E731
            res += (cut(lp), cut(ids), cut(tlp))
        if aut is not None:
            res += ([int(x) for x in out_state[:nreq]],)
        if max_draft is not None:
            res += (int(drafted.value), int(accepted.value))
        return res

    def _context_layout(self, who, contexts, ctx_of, prompts):
        """The context calls' laid-out tokens and (ctx_off, ctx_len, off, len) for contexts / ctx_of / prompts (each
        context once), or ValueError for an index outside contexts or a bad context."""
        if contexts is None or ctx_of is None:
            raise ValueError(f"{who} takes a list of contexts and one context index per prompt")
        contexts = [np.asarray(c) for c in contexts]
        try:
            ctx_of = [c for c in ctx_of]
        except TypeError as e:
            raise ValueError(f"{who}: bad ctx_of: {e}") from None
        nreq = len(prompts)
        if len(ctx_of) != nreq:
            raise ValueError(f"{who} takes one ctx_of per prompt: {nreq} prompts, {len(ctx_of)} values")
        for i, c in enumerate(ctx_of):
            if not isinstance(c, (int, np.integer)) or not -1 <= c < len(contexts):
                raise ValueError(f"ctx_of[{i}] must be -1 or an index into the {len(contexts)} contexts, got {c!r}")
        for k, c in enumerate(contexts):
            if c.ndim != 1 or (len(c) and c.dtype.kind not in "iu"):
                raise ValueError(f"context {k} must be a sequence of token ids")
            if not ((c >= 0) & (c < self.vocab)).all():
                raise ValueError(f"context {k} has a token outside [0, {self.vocab})")
        pieces = contexts + prompts
        starts = np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(np.int64)
        if starts[-1] >= 1 << 31:
            raise ValueError(f"{who}: the tokens do not fit an int index")
        tokens = np.ascontiguousarray(np.concatenate(pieces) if len(pieces) else np.zeros(0), np.int32)
        ctx_off = np.asarray([starts[c] if c >= 0 else 0 for c in ctx_of], np.int32)
        ctx_len = np.asarray([len(contexts[c]) if c >= 0 else 0 for c in ctx_of], np.int32)
        off = np.asarray(starts[len(contexts):len(contexts) + nreq], np.int32)
        len_ = np.asarray([len(p) for p in prompts], np.int32)
        return tokens, ctx_off, ctx_len, off, len_

    def _optional_context_layout(self, who, contexts, ctx_of, prompts):
        """_context_layout, or with contexts and ctx_of both None the prompts alone: (tokens, (ctx_off, ctx_len), off, len)
        with (None, None) for NULL context arrays."""
        if contexts is None and ctx_of is None:
            nreq = len(prompts)
            tokens = np.ascontiguousarray(np.concatenate(prompts) if nreq else np.zeros(0), np.int32)
            len_ = np.asarray([len(p) for p in prompts], np.int32)
            off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(len_)[:-1]]) if nreq else np.zeros(0), np.int32)
            return tokens, (None, None), off, len_
        tokens, ctx_off, ctx_len, off, len_ = self._context_layout(who, contexts, ctx_of, prompts)
        return tokens, (ctx_off, ctx_len), off, len_

    def _check_queue_k(self, k):
        """The queue calls' check on k (0 allowed), raised before the library would abort the process."""
        kmax = min(TOPK_MAX, self.vocab)
        if not isinstance(k, (int, np.integer)) or isinstance(k, bool) or not 0 <= k <= kmax:
            raise ValueError(f"k must be an integer in [0, {kmax}], got {k!r}")

    def decode_sample_queue(self, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states):
        """calm_b200_decode_sample_queue: request i continues prompts[i] (a sequence of at least one token id) for at most
        max_new[i] tokens at temperature[i] / minp[i] from rng_states[i], stopping after a token in `stop` (a sequence of
        ids shared by all requests, possibly empty), with at most max_rows requests in flight.  Returns (tokens, states,
        served, steps): tokens[i] is request i's int32 tokens (its out_len[i] of them), states the nreq generator states
        after the call, served 1 on the new path and 0 when the per-request fallback gave them, steps the number of steps
        run.  Raises ValueError where the C call would abort, and for per-request lists whose lengths differ."""
        prompts, max_new, temperature, minp, stop, states = self._queue_args("decode_sample_queue", prompts, max_new, temperature, minp, stop, max_rows,
                                                                             rng_states)
        nreq = len(prompts)
        tokens = np.ascontiguousarray(np.concatenate(prompts) if nreq else np.zeros(0), np.int32)
        len_ = np.asarray([len(p) for p in prompts], np.int32)
        off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(len_)[:-1]]) if nreq else np.zeros(0), np.int32)
        return self._queue_call(self.lib.calm_b200_decode_sample_queue, tokens, None, off, len_, max_new, temperature, minp, stop, max_rows, states)[:4]

    def decode_sample_queue_context(self, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states):
        """calm_b200_decode_sample_queue_context: decode_sample_queue where request i's prompt is contexts[ctx_of[i]] ++
        prompts[i] (ctx_of[i] == -1: prompts[i] alone).  Each context (a sequence of token ids, possibly empty) is laid
        out once, so the requests that name it share it.  Returns (tokens, states, served, steps, prompt_rows), prompt_rows
        being the rows the call's prompt passes computed.  Raises ValueError where the C call would abort, for an index
        outside contexts and for per-request lists whose lengths differ."""
        prompts, max_new, temperature, minp, stop, states = self._queue_args("decode_sample_queue_context", prompts, max_new, temperature, minp, stop,
                                                                             max_rows, rng_states)
        tokens, ctx_off, ctx_len, off, len_ = self._context_layout("decode_sample_queue_context", contexts, ctx_of, prompts)
        return self._queue_call(self.lib.calm_b200_decode_sample_queue_context, tokens, (ctx_off, ctx_len), off, len_, max_new, temperature, minp, stop,
                                max_rows, states)

    def decode_sample_queue_logprobs(self, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states, k: int = 0):
        """calm_b200_decode_sample_queue_logprobs: decode_sample_queue_context (contexts and ctx_of both None: no
        contexts, decode_sample_queue), returning its tuple and each request's log-probabilities of its tokens and the k
        most likely tokens at each step: (tokens, states, served, steps, prompt_rows, logprobs, top_ids, top_logprobs)
        with logprobs[i] float32[out_len[i]] and, for k > 0, top_ids[i] int32 / top_logprobs[i] float32 [out_len[i], k]
        (None for k == 0).  The numbers are the log-softmax of the step's logits at temperature 1 without the min-p cut.
        Raises ValueError where the C call would abort (k outside [0, min(TOPK_MAX, vocab)] included)."""
        who = "decode_sample_queue_logprobs"
        self._check_queue_k(k)
        prompts, max_new, temperature, minp, stop, states = self._queue_args(who, prompts, max_new, temperature, minp, stop, max_rows, rng_states)
        tokens, ctx, off, len_ = self._optional_context_layout(who, contexts, ctx_of, prompts)
        return self._queue_call(self.lib.calm_b200_decode_sample_queue_logprobs, tokens, ctx, off, len_, max_new, temperature, minp, stop, max_rows, states,
                                k=int(k))

    def decode_sample_queue_penalties(self, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states, presence=None,
                                      frequency=None, repetition=None, logit_bias=None, k=None):
        """calm_b200_decode_sample_queue_penalties: decode_sample_queue_logprobs (contexts and ctx_of both None: no
        contexts) where request i's logits go through its presence[i], frequency[i] and repetition[i] penalties and its
        logit_bias[i] ({token id: value}, or None) before its token is chosen, as include/calm_b200.h states.  presence /
        frequency / repetition None mean 0 / 0 / 1 for every request, logit_bias None no bias.  k None: no
        log-probabilities, and the return value is decode_sample_queue_context's (tokens, states, served, steps,
        prompt_rows); otherwise decode_sample_queue_logprobs' tuple, of the processed logits.  Raises ValueError where
        the C call would abort."""
        who = "decode_sample_queue_penalties"
        if k is not None:
            self._check_queue_k(k)
        prompts, max_new, temperature, minp, stop, states = self._queue_args(who, prompts, max_new, temperature, minp, stop, max_rows, rng_states)
        keep = []  # the arrays the C call reads
        pen = self._penalty_args(who, len(prompts), presence, frequency, repetition, logit_bias, keep)
        tokens, ctx, off, len_ = self._optional_context_layout(who, contexts, ctx_of, prompts)
        return self._queue_call(self.lib.calm_b200_decode_sample_queue_penalties, tokens, ctx, off, len_, max_new, temperature, minp, stop, max_rows,
                                states, k=None if k is None else int(k), pen=pen)

    def _penalty_args(self, who, nreq, presence, frequency, repetition, logit_bias, keep):
        """The penalty calls' arguments after minp (presence .. n_bias), or ValueError wherever the C call would abort;
        the arrays they point to go to `keep`."""
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)

        def per_request(name, xs, lo, hi):
            if xs is None:
                return None
            try:
                a = np.ascontiguousarray(xs, np.float32).reshape(-1)
            except (TypeError, ValueError) as e:
                raise ValueError(f"{who}: bad {name}: {e}") from None
            if len(a) != nreq:
                raise ValueError(f"{who} takes one {name} per prompt: {nreq} prompts, {len(a)} values")
            if not (np.isfinite(a) & (a >= lo) & (a <= hi)).all():
                raise ValueError(f"{who}: every {name} must be finite and in [{lo:g}, {hi:g}]")
            keep.append(a)
            return a.ctypes.data_as(fp)

        pen = [per_request("presence", presence, -1e6, 1e6), per_request("frequency", frequency, -1e6, 1e6),
               per_request("repetition", repetition, np.float32(1e-6), 1e6)]
        if logit_bias is None:
            pen += [None, None, None, None, 0]
        else:
            logit_bias = list(logit_bias)
            if len(logit_bias) != nreq:
                raise ValueError(f"{who} takes one logit_bias per prompt: {nreq} prompts, {len(logit_bias)} values")
            ids, vals, blen = [], [], []
            for i, d in enumerate(logit_bias):
                d = {} if d is None else d
                if not isinstance(d, dict):
                    raise ValueError(f"logit_bias[{i}] must be a dict of token id: value, or None")
                for t, b in d.items():
                    if not isinstance(t, (int, np.integer)) or isinstance(t, bool) or not 0 <= t < self.vocab:
                        raise ValueError(f"logit_bias[{i}] has an id outside [0, {self.vocab}): {t!r}")
                    b32 = np.float32(b)
                    if not np.isfinite(b32) or abs(b32) > 1e6:
                        raise ValueError(f"logit_bias[{i}][{t}] must be finite and in [-1e6, 1e6], got {b!r}")
                    ids.append(int(t)), vals.append(b32)
                blen.append(len(d))
            b_len = np.asarray(blen, np.int32)
            b_off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(b_len)[:-1]]) if nreq else np.zeros(0), np.int32)
            b_ids, b_val = np.asarray(ids, np.int32), np.asarray(vals, np.float32)
            keep += [b_len, b_off, b_ids, b_val]
            pen += [b_off.ctypes.data_as(ip), b_len.ctypes.data_as(ip), b_ids.ctypes.data_as(ip) if len(ids) else None,
                    b_val.ctypes.data_as(fp) if len(ids) else None, len(ids)]
        return pen

    def decode_sample_queue_constrained(self, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states,
                                        automaton=None, start=None, presence=None, frequency=None, repetition=None, logit_bias=None, k=None):
        """calm_b200_decode_sample_queue_constrained: decode_sample_queue_penalties where request i with start[i] >= 0 is
        constrained to `automaton` (a TokenAutomaton over this model's vocabulary) from state start[i]: at each step only
        the tokens its state allows can be chosen, and it retires after a token that leads to a final state.  start None
        (or every entry -1) constrains no request.  Returns decode_sample_queue_penalties' tuple followed by each request's
        state after its last token (-1 for an unconstrained request).  Raises ValueError where the C call would abort."""
        return self._constrained_call("decode_sample_queue_constrained", contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows,
                                      rng_states, automaton, start, presence, frequency, repetition, logit_bias, k)

    def decode_sample_queue_truncated(self, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states, top_k=None,
                                      top_p=None, automaton=None, start=None, presence=None, frequency=None, repetition=None, logit_bias=None, k=None):
        """calm_b200_decode_sample_queue_truncated: decode_sample_queue_constrained where sampled request i keeps only its
        top_k[i] most likely tokens (0: off) and the shortest prefix of those whose probability reaches top_p[i] (1: off)
        before the draw, by include/calm_b200.h's rule.  top_k / top_p None mean off for every request.  Returns
        decode_sample_queue_constrained's tuple; log-probabilities stay those before truncation.  Raises ValueError where
        the C call would abort."""
        return self._truncated_call("decode_sample_queue_truncated", contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows, rng_states,
                                    top_k, top_p, automaton, start, presence, frequency, repetition, logit_bias, k)

    def decode_sample_queue_lookup(self, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows: int, rng_states, max_draft: int = 7,
                                   top_k=None, top_p=None, automaton=None, start=None, presence=None, frequency=None, repetition=None, logit_bias=None,
                                   k=None):
        """calm_b200_decode_sample_queue_lookup: decode_sample_queue_truncated, with the rows its steps leave free holding
        prompt-lookup drafts of each request's own tokens (up to max_draft per request and step, in [0, 15]) that the same
        step verifies.  Returns decode_sample_queue_truncated's tuple, bit for bit except that steps may be fewer, followed
        by (drafted, accepted): the draft rows the call ran and the drafts it accepted.  Raises ValueError where the C call
        would abort."""
        if not isinstance(max_draft, (int, np.integer)) or isinstance(max_draft, bool) or not 0 <= max_draft <= VERIFY_MAX - 1:
            raise ValueError(f"max_draft must be an integer in [0, {VERIFY_MAX - 1}], got {max_draft!r}")
        return self._truncated_call("decode_sample_queue_lookup", contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows, rng_states,
                                    top_k, top_p, automaton, start, presence, frequency, repetition, logit_bias, k, max_draft=int(max_draft))

    def _truncated_call(self, who, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows, rng_states, top_k, top_p, automaton, start,
                        presence, frequency, repetition, logit_bias, k, max_draft=None):
        """decode_sample_queue_truncated (max_draft None) or _lookup: the top_k / top_p checks, then _constrained_call."""
        nreq = len(prompts)
        keep = []
        trunc = []
        for name, xs, dt in (("top_k", top_k, np.int32), ("top_p", top_p, np.float32)):
            if xs is None:
                trunc.append(None)
                continue
            try:
                a = np.asarray(xs)
                if name == "top_k" and (a.dtype.kind not in "iu" or a.ndim != 1):
                    raise TypeError("not a sequence of integers")
                a = np.ascontiguousarray(a, dt).reshape(-1)
            except (TypeError, ValueError) as e:
                raise ValueError(f"{who}: bad {name}: {e}") from None
            if len(a) != nreq:
                raise ValueError(f"{who} takes one {name} per prompt: {nreq} prompts, {len(a)} values")
            if name == "top_k" and not (a >= 0).all():
                raise ValueError(f"{who}: every top_k must be >= 0")
            if name == "top_p" and not (np.isfinite(a) & (a > 0) & (a <= 1)).all():
                raise ValueError(f"{who}: every top_p must be finite and in (0, 1]")
            keep.append(a)
            trunc.append(a.ctypes.data_as(C.POINTER(C.c_int) if name == "top_k" else _fptr))
        if self.vocab > TRUNC_VOCAB_MAX and nreq:
            t = np.ascontiguousarray(temperature, np.float32).reshape(-1)
            m = np.ascontiguousarray(minp, np.float32).reshape(-1)
            for i in range(min(nreq, len(t), len(m), len(max_new))):
                on = (top_k is not None and keep[0][i] > 0) or (top_p is not None and keep[-1][i] < 1)
                if on and max_new[i] > 0 and t[i] != 0 and m[i] < 1:
                    raise ValueError(f"{who}: truncation serves vocabularies up to {TRUNC_VOCAB_MAX} tokens, not {self.vocab}")
        return self._constrained_call(who, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows, rng_states, automaton, start,
                                      presence, frequency, repetition, logit_bias, k, trunc=trunc, keep=keep, max_draft=max_draft)

    def _constrained_call(self, who, contexts, ctx_of, prompts, max_new, temperature, minp, stop, max_rows, rng_states, automaton, start, presence,
                          frequency, repetition, logit_bias, k, trunc=None, keep=None, max_draft=None):
        """decode_sample_queue_constrained (trunc None), _truncated (trunc: its top_k / top_p pointers, their arrays in
        keep) or, with max_draft, _lookup."""
        if k is not None:
            self._check_queue_k(k)
        prompts, max_new, temperature, minp, stop, states = self._queue_args(who, prompts, max_new, temperature, minp, stop, max_rows, rng_states)
        nreq = len(prompts)
        if automaton is not None:
            if not isinstance(automaton, TokenAutomaton):
                raise ValueError(f"{who}: automaton must be a TokenAutomaton or None")
            if automaton.vocab != self.vocab:
                raise ValueError(f"{who}: the automaton's vocabulary has {automaton.vocab} tokens, the model's {self.vocab}")
        st = None
        if start is not None:
            st = list(start)
            if len(st) != nreq:
                raise ValueError(f"{who} takes one start state per prompt: {nreq} prompts, {len(st)} values")
            n_states = automaton.n_states if automaton is not None else 0
            for i, s0 in enumerate(st):
                if not isinstance(s0, (int, np.integer)) or isinstance(s0, bool) or not -1 <= s0 < n_states:
                    raise ValueError(f"start[{i}] must be -1 or a state in [0, {n_states}), got {s0!r}")
                if s0 >= 0 and max_new[i] > 0 and automaton.final[s0]:
                    raise ValueError(f"request {i} starts in final state {s0}")
            st = np.ascontiguousarray(st, np.int32)
        keep = (keep or []) + [st]
        pen = self._penalty_args(who, nreq, presence, frequency, repetition, logit_bias, keep)
        ip = C.POINTER(C.c_int)
        if automaton is None:
            aut = [0, None, None, None, None, None]
        else:
            a = automaton
            aut = [a.n_states, a.allow.ctypes.data_as(C.POINTER(C.c_uint32)), a.next_default.ctypes.data_as(ip), a.exc_off.ctypes.data_as(ip),
                   a.exc_tok.ctypes.data_as(ip), a.exc_next.ctypes.data_as(ip)]
        aut.append(None if st is None else st.ctypes.data_as(ip))
        tokens, ctx, off, len_ = self._optional_context_layout(who, contexts, ctx_of, prompts)
        fn = self.lib.calm_b200_decode_sample_queue_constrained if trunc is None else self.lib.calm_b200_decode_sample_queue_truncated
        if max_draft is not None:
            fn = self.lib.calm_b200_decode_sample_queue_lookup
        return self._queue_call(fn, tokens, ctx, off, len_, max_new, temperature, minp, stop, max_rows, states, k=None if k is None else int(k), pen=pen,
                                aut=aut, trunc=trunc, max_draft=max_draft)

    def forward_sample(self, token: int, pos: int, temperature: float, minp: float, rng_state: int):
        """calm_b200_forward_sample: one token, sampled on the device; returns (token, new rng state)."""
        rng = C.c_ulonglong(rng_state)
        tok = self.lib.calm_b200_forward_sample(C.byref(self.transformer), token, pos, temperature, minp, C.byref(rng))
        return int(tok), int(rng.value)

    def device_logits(self) -> np.ndarray:
        out = np.zeros(self.vocab, np.float32)
        self.lib.calm_b200_read_device_logits(out.ctypes.data_as(_fptr))
        return out

    def logits_view(self) -> np.ndarray:
        return np.ctypeslib.as_array(self.transformer.state.logits, shape=(self.vocab,))

    def read_kv(self, layer: int, kv_pos: int):
        k = np.zeros(self.spec.kv_dim, np.float32)
        v = np.zeros(self.spec.kv_dim, np.float32)
        self.lib.calm_b200_read_kv(C.byref(self.transformer), layer, kv_pos, k.ctypes.data_as(_fptr), v.ctypes.data_as(_fptr))
        return k, v

    def read_state(self, which: str, layer: int = 0) -> np.ndarray:
        """calm_b200_read_state: one engine buffer (a key of STATE) as a flat float32 array, for stage-level tests."""
        n = self.lib.calm_b200_read_state(STATE[which], layer, None, 0)
        out = np.zeros(n, np.float32)
        assert self.lib.calm_b200_read_state(STATE[which], layer, out.ctypes.data_as(_fptr), n) == n
        return out

    def poison(self, kv_from_pos: int) -> None:
        """calm_b200_poison_state: NaN bytes into every scratch buffer and the cache slots [kv_from_pos, seq_len)."""
        self.lib.calm_b200_poison_state(C.byref(self.transformer), kv_from_pos)

    def fill_kv(self, n_pos: int, seed: int = 1) -> None:
        self.lib.calm_b200_fill_kv(C.byref(self.transformer), n_pos, seed)

    def profile(self, token: int, pos0: int, n: int):
        """Run n greedy tokens of the production graph with in-kernel stage stamps; returns
        ({stage: (ms_total, bytes_total, launches)}, mean token span in ms)."""
        self.lib.calm_b200_set_perf(1)
        tok = token
        for i in range(n):
            tok = self.forward_argmax(tok, pos0 + i)
        out = {}
        i = 0
        name = C.create_string_buffer(64)
        ms, by, nl = C.c_double(), C.c_double(), C.c_long()
        while self.lib.calm_b200_stage_stats(i, name, 64, C.byref(ms), C.byref(by), C.byref(nl)):
            out[name.value.decode()] = (ms.value, by.value, nl.value)
            i += 1
        span = self.lib.calm_b200_perf_token_ms()
        self.lib.calm_b200_set_perf(0)
        return out, span

    def close(self) -> None:
        if self.transformer is not None:
            self.lib.calm_b200_release(C.byref(self.transformer))
            for p in self._uploaded:
                self.lib.calm_b200_free(p)
            self._uploaded = []
            self._keep = None  # the caller's tensors (device weights of a large model) can be freed now
            self.transformer = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def matvec(dbits: int, w_dev_ptr: int, x: np.ndarray, n: int, d: int, warmup: int = 0, iters: int = 1):
    """Run the production matvec kernel once (y = W.x); returns (y, ms per launch)."""
    L = load()
    x = np.ascontiguousarray(x, np.float32)
    y = np.zeros(d, np.float32)
    ms = L.calm_b200_matvec(dbits, w_dev_ptr, x.ctypes.data_as(_fptr), y.ctypes.data_as(_fptr), n, d, warmup, iters)
    return y, ms


def sample_logits(logits: np.ndarray, temperature: float, minp: float, rng_state: int, timed: bool = False):
    """The device sampler on host logits; returns (token, new rng state[, microseconds of the sampler kernels])."""
    L = load()
    buf = np.ascontiguousarray(logits, np.float32)
    rng = C.c_ulonglong(rng_state)
    us = C.c_float(0)
    tok = L.calm_b200_sample_logits(buf.ctypes.data_as(_fptr), len(buf), temperature, minp, C.byref(rng), C.byref(us) if timed else None)
    return (tok, int(rng.value), us.value) if timed else (tok, int(rng.value))


def sample_logits_truncated(logits: np.ndarray, temperature: float, minp: float, top_k: int, top_p: float, rng_state: int, timed: bool = False):
    """calm_b200_sample_logits_truncated: the device sampler on host logits after top_k (0: off) / top_p (1: off)
    truncation by include/calm_b200.h's rule; returns (token, new rng state, the row after truncation with -inf at the
    dropped ids[, microseconds of the kernels]).  Raises ValueError where the C call would abort."""
    buf = np.ascontiguousarray(logits, np.float32).reshape(-1)
    if not len(buf):
        raise ValueError("sample_logits_truncated: empty vocabulary")
    if not isinstance(top_k, (int, np.integer)) or isinstance(top_k, bool) or top_k < 0:
        raise ValueError(f"top_k must be a non-negative integer, got {top_k!r}")
    p32 = np.float32(top_p)
    if not (np.isfinite(p32) and 0 < p32 <= 1):
        raise ValueError(f"top_p must be finite and in (0, 1], got {top_p!r}")
    _check_rng(rng_state)
    if (top_k > 0 or p32 < 1) and np.float32(temperature) != 0 and np.float32(minp) < 1 and len(buf) > TRUNC_VOCAB_MAX:
        raise ValueError(f"sample_logits_truncated: truncation serves vocabularies up to {TRUNC_VOCAB_MAX} tokens, not {len(buf)}")
    L = load()
    rng = C.c_ulonglong(rng_state)
    us = C.c_float(0)
    row = np.empty_like(buf)
    tok = L.calm_b200_sample_logits_truncated(buf.ctypes.data_as(_fptr), len(buf), temperature, minp, int(top_k), float(p32), C.byref(rng),
                                              row.ctypes.data_as(_fptr), C.byref(us) if timed else None)
    return (tok, int(rng.value), row, us.value) if timed else (tok, int(rng.value), row)
