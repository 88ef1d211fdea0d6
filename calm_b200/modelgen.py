"""Seeded synthetic models in calm's formats.

There is no network in the build or on the GPU box, so every model in the
tests and in bench.py is random-initialised here with the SHAPES the reference
expects (reference run.c:71-117 lists every tensor name, dtype and shape) and,
when written to disk, in the reference's `.calm` container (a safetensors-like
file: u64 header length, JSON header padded so data starts 256-byte aligned,
raw tensor bytes; reference tools/convert.py:502-536, parser tensors.c:216-270).

Weight formats (reference infer.c:28-40, convert.py:247-268, 311):
  fp16  IEEE half
  fp8   e5m2, round-to-nearest-even from fp32 (torch.float8_e5m2)
  gf4   groups of 8 weights in one uint32: low byte = e5m2 scale (the signed
        max-magnitude element of the group), then eight 3-bit codes q_k,
        w_k = (q_k - 4) * scale / -4.
"""
from __future__ import annotations

import ctypes as C
import json
import math
from dataclasses import dataclass, field, replace
from typing import Dict, Optional

import numpy as np
import torch

from .cstructs import MAX_LAYERS, Transformer

FLT_MAX = 3.4028234663852886e38


@dataclass(frozen=True)
class ModelSpec:
    name: str
    dim: int
    hidden_dim: int
    n_layers: int
    n_heads: int
    n_kv_heads: int
    head_dim: int
    vocab_size: int
    dtype: str = "fp8"  # fp16 | fp8 | gf4
    rope_theta: float = 10000.0
    rotary_dim: Optional[int] = None  # default head_dim
    n_experts: int = 0
    n_experts_active: int = 0
    norm_eps: float = 1e-5
    act_type: str = "silu"  # silu | gelu
    norm_type: str = "rmsnorm"  # rmsnorm | layernorm | layernorm_par
    qkv_clip: Optional[float] = None
    qkv_bias: bool = False
    tied: bool = False  # no model.output.weight: classifier = embedding
    max_seq_len: int = 4096
    init_std: float = 0.02
    gate_std: float = 0.2  # wider router init keeps top-k margins healthy (SURVEY.md s.9)
    bos_id: int = 0
    eos_id: int = 1

    @property
    def dbits(self) -> int:
        return {"fp16": 16, "fp8": 8, "gf4": 4}[self.dtype]

    @property
    def q_dim(self) -> int:
        return self.n_heads * self.head_dim

    @property
    def kv_dim(self) -> int:
        return self.n_kv_heads * self.head_dim


# The five BASELINE.json configurations (shapes from SURVEY.md s.8) ...
SPECS: Dict[str, ModelSpec] = {
    "qwen2-0.5b-fp16": ModelSpec("qwen2-0.5b-fp16", 896, 4864, 24, 14, 2, 64, 151936, "fp16", rope_theta=1e6,
                                 norm_eps=1e-6, qkv_bias=True, tied=True, bos_id=2, eos_id=1),
    "llama3-8b-fp8": ModelSpec("llama3-8b-fp8", 4096, 14336, 32, 32, 8, 128, 128256, "fp8", rope_theta=5e5),
    "mistral-7b-gf4": ModelSpec("mistral-7b-gf4", 4096, 14336, 32, 32, 8, 128, 32000, "gf4", rope_theta=1e6),
    "mixtral-8x7b-fp8": ModelSpec("mixtral-8x7b-fp8", 4096, 14336, 32, 32, 8, 128, 32000, "fp8", rope_theta=1e6,
                                  n_experts=8, n_experts_active=2),
    "llama3-70b-fp8": ModelSpec("llama3-70b-fp8", 8192, 28672, 80, 64, 8, 128, 128256, "fp8", rope_theta=5e5),
}
SPECS["llama3-8b-fp16"] = replace(SPECS["llama3-8b-fp8"], name="llama3-8b-fp16", dtype="fp16")
SPECS["llama3-8b-gf4"] = replace(SPECS["llama3-8b-fp8"], name="llama3-8b-gf4", dtype="gf4")

# ... and small shapes for parity tests (the oracle finishes these in well under a second).
_T = ModelSpec("tiny", 256, 704, 3, 8, 4, 32, 512, "fp8", max_seq_len=64)
SPECS.update({
    "tiny-fp8": replace(_T, name="tiny-fp8"),
    "tiny-fp16": replace(_T, name="tiny-fp16", dtype="fp16"),
    "tiny-gf4": replace(_T, name="tiny-gf4", dtype="gf4"),
    # Qwen2 flavour: QKV bias, tied classifier, kv_mul 7, head_dim 64
    "tiny-qwen": replace(_T, name="tiny-qwen", dtype="fp16", dim=448, n_heads=7, n_kv_heads=1, head_dim=64,
                         hidden_dim=1216, qkv_bias=True, tied=True, rope_theta=1e6, norm_eps=1e-6),
    # Llama-3 flavour: head_dim 128, kv_mul 4, long rows in w2
    "tiny-llama": replace(_T, name="tiny-llama", dim=512, n_heads=4, n_kv_heads=1, head_dim=128, hidden_dim=1792,
                          vocab_size=1024, rope_theta=5e5, max_seq_len=128),
    # Mixtral flavour: 8 experts, top-2
    "tiny-moe": replace(_T, name="tiny-moe", n_experts=8, n_experts_active=2, hidden_dim=512),
    "tiny-moe-gf4": replace(_T, name="tiny-moe-gf4", dtype="gf4", n_experts=8, n_experts_active=2, hidden_dim=512),
    # model switches of the reference that the five configs do not exercise (SURVEY.md s.8f row 4)
    "tiny-gelu-clip": replace(_T, name="tiny-gelu-clip", act_type="gelu", qkv_clip=1.0, rotary_dim=16),
    "tiny-ln": replace(_T, name="tiny-ln", norm_type="layernorm", dtype="fp16"),
    "tiny-lnpar": replace(_T, name="tiny-lnpar", norm_type="layernorm_par", dtype="fp16"),
    "tiny-mha": replace(_T, name="tiny-mha", n_heads=8, n_kv_heads=8),
    # QKV bias + tied classifier on a shape two tensor-parallel ranks can split (tiny-qwen has a single kv head)
    "tiny-bias2": replace(_T, name="tiny-bias2", dtype="fp16", n_heads=4, n_kv_heads=2, head_dim=64, qkv_bias=True, tied=True),
    # a shape that 2, 4 and 8 tensor-parallel ranks can split (8 kv heads, hidden = 4 * 32 * 8), and its MoE twin
    "tiny-tp8": replace(_T, name="tiny-tp8", n_heads=8, n_kv_heads=8, head_dim=32, hidden_dim=1024),
    "tiny-tp8-moe": replace(_T, name="tiny-tp8-moe", n_heads=8, n_kv_heads=8, head_dim=32, hidden_dim=1024, n_experts=4, n_experts_active=2),
    # the smallest shapes the batched prompt pass serves (every dim a multiple of 128, head_dim 64 / 128)
    "pf-tiny": ModelSpec("pf-tiny", 256, 512, 2, 4, 2, 64, 512, "fp8", rope_theta=1e4, max_seq_len=512),
    "pf-tiny-hd128": ModelSpec("pf-tiny-hd128", 512, 1024, 2, 4, 1, 128, 512, "fp8", rope_theta=5e5, max_seq_len=512, qkv_bias=True),
    # wide enough for the ring-fed kernels (rows of whole 1 KB chunks) and splittable over 2 / 4 tensor-parallel ranks
    "ring-tp": ModelSpec("ring-tp", 2048, 4096, 2, 8, 4, 128, 512, "fp8", rope_theta=5e5, max_seq_len=64),
    # Gemma-style multi-query attention: 8 query heads on ONE kv head of 256 dims (the attention kernel's merge
    # records exceed the default 48 KB of dynamic shared memory)
    # (hidden >= dim >= q_dim: the reference CPU backend reuses xb2[dim] and hb[hidden] as scratch, infer.c:152-153, 404, 409)
    "tiny-hd256": replace(_T, name="tiny-hd256", dim=2048, n_layers=2, n_heads=8, n_kv_heads=1, head_dim=256, hidden_dim=2048),
    # Llama-3-8B's attention geometry (32 query / 8 kv heads of 128, so 8 units x 16 slices on 132 SMs) at the full
    # 4096-token context, on widths the CPU oracle finishes in milliseconds per token
    "attn-l8": ModelSpec("attn-l8", 256, 512, 2, 32, 8, 128, 512, "fp8", rope_theta=5e5, max_seq_len=4096),
})


# --------------------------------------------------------------------------- quantisers

def to_fp8_bytes(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> e5m2 bytes, round-to-nearest-even (convert.py:311 uses the same cast)."""
    return t.to(torch.float8_e5m2).view(torch.uint8)


def to_gf4_words(t: torch.Tensor) -> torch.Tensor:
    """fp32 (..., n) with n % 8 == 0 -> int32 (..., n/8) gf4 words.

    Restates the reference quantiser (convert.py:247-268): per group of 8 take
    the element of largest magnitude WITH its sign as the scale, round it to
    e5m2, express every element as a fraction of it, map [-1, 1] onto the codes
    0..7 through code = round(frac * -4 + 4) clamped to 7 (so the scale element
    itself gets code 0, i.e. (0 - 4) * s / -4 = s).
    """
    g = t.reshape(*t.shape[:-1], t.shape[-1] // 8, 8).to(torch.float32)
    idx = g.abs().argmax(dim=-1, keepdim=True)
    scale = g.gather(-1, idx)
    scale8 = scale.to(torch.float8_e5m2)
    scale = scale8.to(torch.float32)
    frac = g / scale
    frac = torch.nan_to_num(frac, nan=0.0, posinf=0.0, neginf=0.0)
    code = (frac.to(torch.float16) * -4 + 4).clamp(0, 7).round().to(torch.int64)
    shifts = torch.arange(8, device=t.device, dtype=torch.int64) * 3 + 8
    word = (code << shifts).sum(-1) + scale8.view(torch.uint8).squeeze(-1).to(torch.int64)
    word = torch.where(word >= 2 ** 31, word - 2 ** 32, word)
    return word.to(torch.int32)


def gf4_words_to_float(words: np.ndarray) -> np.ndarray:
    """Decode gf4 words (uint32/int32 array) to float32, 8 values per word (infer.c:37-40)."""
    w = words.astype(np.uint32)
    scale = ((w & 0xFF).astype(np.uint16) << 8).view(np.float16).astype(np.float32) / np.float32(-4.0)
    out = np.empty(w.shape + (8,), np.float32)
    for k in range(8):
        out[..., k] = (((w >> np.uint32(8 + 3 * k)) & 7).astype(np.int32) - 4).astype(np.float32) * scale
    return out.reshape(*w.shape[:-1], w.shape[-1] * 8)


def fp8_bytes_to_float(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint16) << 8).view(np.float16).astype(np.float32)


def quantize(t: torch.Tensor, dtype: str) -> torch.Tensor:
    if dtype == "fp16":
        return t.to(torch.float16)
    if dtype == "fp8":
        return to_fp8_bytes(t)
    if dtype == "gf4":
        return to_gf4_words(t)
    raise ValueError(dtype)


_ST_DTYPE = {torch.float32: "F32", torch.float16: "F16", torch.uint8: "U8", torch.int32: "I32"}


# --------------------------------------------------------------------------- generation

def tensor_plan(spec: ModelSpec):
    """(name, shape, kind) for every model.* tensor in the order the reference
    binds them (run.c:79-115).  kind: w = quantised weight, g = router weight,
    n = norm weight (f32), b = bias (f32)."""
    s = spec
    plan = [("model.embed.weight", (s.vocab_size, s.dim), "w")]
    e = (s.n_experts,) if s.n_experts else ()
    for l in range(s.n_layers):
        p = f"model.layers.{l}."
        plan.append((p + "attn.norm.weight", (s.dim,), "n"))
        if s.norm_type != "layernorm_par":
            plan.append((p + "mlp.norm.weight", (s.dim,), "n"))
        plan.append((p + "attn.wq.weight", (s.q_dim, s.dim), "w"))
        plan.append((p + "attn.wk.weight", (s.kv_dim, s.dim), "w"))
        plan.append((p + "attn.wv.weight", (s.kv_dim, s.dim), "w"))
        plan.append((p + "attn.wo.weight", (s.dim, s.q_dim), "w"))
        if s.qkv_bias:
            plan.append((p + "attn.wqkv.bias", (s.q_dim + 2 * s.kv_dim,), "b"))
        if s.n_experts:
            plan.append((p + "moegate.weight", (s.n_experts, s.dim), "g"))
        plan.append((p + "mlp.w1.weight", e + (s.hidden_dim, s.dim), "w"))
        plan.append((p + "mlp.w2.weight", e + (s.dim, s.hidden_dim), "w"))
        plan.append((p + "mlp.w3.weight", e + (s.hidden_dim, s.dim), "w"))
    plan.append(("model.norm.weight", (s.dim,), "n"))
    if not s.tied:
        plan.append(("model.output.weight", (s.vocab_size, s.dim), "w"))
    return plan


def generate(spec: ModelSpec, seed: int = 0, device: str = "cpu", chunk_rows: int = 1 << 14) -> Dict[str, torch.Tensor]:
    """Random-init every model.* tensor: weights ~ N(0, init_std) then quantised,
    norm weights 1 + N(0, 0.05), biases N(0, init_std), router N(0, gate_std).
    The classifier rows of the BOS/EOS tokens are zeroed so that greedy decoding
    of random weights does not stop early (run.c:225)."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    out: Dict[str, torch.Tensor] = {}
    for name, shape, kind in tensor_plan(spec):
        if kind == "n":
            t = 1.0 + 0.05 * torch.randn(shape, generator=gen, device=device, dtype=torch.float32)
        elif kind == "b":
            t = spec.init_std * torch.randn(shape, generator=gen, device=device, dtype=torch.float32)
        else:
            std = spec.gate_std if kind == "g" else spec.init_std
            rows = int(np.prod(shape[:-1]))
            flat_shape = (rows, shape[-1])
            qshape = (rows, shape[-1] // 8) if spec.dtype == "gf4" else flat_shape
            qdtype = {"fp16": torch.float16, "fp8": torch.uint8, "gf4": torch.int32}[spec.dtype]
            q = torch.empty(qshape, dtype=qdtype, device=device)
            for r0 in range(0, rows, chunk_rows):  # bounded fp32 staging for the 70B shapes
                r1 = min(rows, r0 + chunk_rows)
                blk = std * torch.randn((r1 - r0, shape[-1]), generator=gen, device=device, dtype=torch.float32)
                q[r0:r1] = quantize(blk, spec.dtype)
            t = q.reshape(shape[:-1] + (qshape[-1],))
        out[name] = t
    cls = out["model.embed.weight" if spec.tied else "model.output.weight"]
    if not spec.tied:
        for tok in (spec.bos_id, spec.eos_id):
            if 0 <= tok < spec.vocab_size:
                cls[tok].zero_()
    return out


def metadata(spec: ModelSpec) -> Dict[str, str]:
    """The `__metadata__` strings the reference reads (run.c:33-68, 72, 125-126)."""
    m = {
        "dim": spec.dim, "hidden_dim": spec.hidden_dim, "n_layers": spec.n_layers, "n_heads": spec.n_heads,
        "n_kv_heads": spec.n_kv_heads, "vocab_size": spec.vocab_size, "head_dim": spec.head_dim,
        "max_seq_len": spec.max_seq_len, "rope_theta": repr(float(spec.rope_theta)),
        "rotary_dim": spec.rotary_dim if spec.rotary_dim is not None else spec.head_dim,
        "dtype": spec.dtype, "bos_token_id": spec.bos_id, "eos_token_id": spec.eos_id,
        "norm_eps": repr(float(spec.norm_eps)), "act_type": spec.act_type, "norm_type": spec.norm_type,
    }
    if spec.n_experts:
        m["n_experts"] = spec.n_experts
        m["n_experts_active"] = spec.n_experts_active
    if spec.qkv_clip is not None:
        m["qkv_clip"] = repr(float(spec.qkv_clip))
    return {k: str(v) for k, v in m.items()}


def synthetic_tokenizer(spec: ModelSpec):
    """tokenizer.tokens / tokenizer.scores tensors: pieces "<|t%d|>" so that every id
    decodes to something printable and `<|t5|>` round-trips through the reference's
    special-token path (tokenizer.c:219-240)."""
    pieces = b"".join(b"<|t%d|>\0" % i for i in range(spec.vocab_size))
    return {
        "tokenizer.tokens": torch.frombuffer(bytearray(pieces), dtype=torch.uint8),
        "tokenizer.scores": torch.zeros(spec.vocab_size, dtype=torch.float32),
    }


def write_calm(path: str, spec: ModelSpec, tensors: Dict[str, torch.Tensor]) -> None:
    """Write a .calm file the reference loader accepts (layout: convert.py:502-536)."""
    allt = dict(tensors)
    allt.update(synthetic_tokenizer(spec))
    header = {"__metadata__": metadata(spec)}
    off = 0
    for k, v in allt.items():
        size = v.numel() * v.element_size()
        st = "F8_E5M2" if (v.dtype == torch.uint8 and k.startswith("model.")) else _ST_DTYPE[v.dtype]
        header[k] = {"dtype": st, "shape": list(v.shape), "data_offsets": [off, off + size]}
        off += size
    hj = json.dumps(header).encode()
    hj += b" " * (-(len(hj) + 8) % 256)
    with open(path, "wb") as f:
        f.write(len(hj).to_bytes(8, "little"))
        f.write(hj)
        for v in allt.values():
            f.write(v.contiguous().cpu().view(torch.uint8).numpy().tobytes())


# --------------------------------------------------------------------------- struct Transformer

def algorithmic_bytes(spec: ModelSpec, tensors: Optional[Dict[str, torch.Tensor]] = None) -> int:
    """n_bandwidth of reference run.c:523-532: bytes of all model.* tensors, minus
    the embedding table (plus it back when tied), minus the inactive experts."""
    total = 0
    embed = 0
    mlp = 0
    for name, shape, kind in tensor_plan(spec):
        n = int(np.prod(shape))
        b = n * 4 if kind in "nb" else n * spec.dbits // 8
        total += b
        if name.startswith("model.embed."):
            embed += b
        if ".mlp.w" in name:
            mlp += b
    bw = total - embed + (embed if spec.tied else 0)
    if spec.n_experts:
        bw = bw - mlp + mlp // spec.n_experts * spec.n_experts_active
    return bw


def kv_bytes(spec: ModelSpec, pos: int, seq_len: int, kvbits: int = 16) -> int:
    """kvcache_bandwidth of reference run.c:161-165."""
    kv_len = seq_len if pos >= seq_len else pos + 1
    return 2 * (kvbits // 8) * spec.n_layers * spec.kv_dim * kv_len


def fill_transformer(spec: ModelSpec, ptr_of, seq_len: Optional[int] = None, kvbits: int = 16) -> Transformer:
    """Build struct Transformer the way the reference driver does (get_config
    run.c:32-69, get_weights run.c:71-117).  `ptr_of(name)` returns the address
    (host or device) of a tensor, or 0 when absent."""
    t = Transformer()
    c = t.config
    c.dim, c.hidden_dim, c.head_dim = spec.dim, spec.hidden_dim, spec.head_dim
    c.n_layers, c.n_heads, c.n_kv_heads = spec.n_layers, spec.n_heads, spec.n_kv_heads
    c.vocab_size = spec.vocab_size
    c.seq_len = seq_len if seq_len else min(spec.max_seq_len, 4096)
    c.rope_theta = spec.rope_theta
    c.rotary_dim = spec.rotary_dim if spec.rotary_dim is not None else spec.head_dim
    c.n_experts, c.n_experts_ac = spec.n_experts, spec.n_experts_active
    c.norm_eps = spec.norm_eps
    c.act_gelu = spec.act_type == "gelu"
    c.norm_ln = spec.norm_type.startswith("layernorm")
    c.norm_par = spec.norm_type == "layernorm_par"
    c.qkv_clip = spec.qkv_clip if spec.qkv_clip is not None else FLT_MAX

    w = t.weights
    w.dbits = spec.dbits
    assert spec.n_layers <= MAX_LAYERS
    w.token_embedding_table = ptr_of("model.embed.weight")
    for l in range(spec.n_layers):
        p = f"model.layers.{l}."
        w.rms_att_weight[l] = ptr_of(p + "attn.norm.weight")
        w.rms_ffn_weight[l] = ptr_of(p + "mlp.norm.weight")
        w.wq[l] = ptr_of(p + "attn.wq.weight")
        w.wk[l] = ptr_of(p + "attn.wk.weight")
        w.wv[l] = ptr_of(p + "attn.wv.weight")
        w.wo[l] = ptr_of(p + "attn.wo.weight")
        w.bqkv[l] = ptr_of(p + "attn.wqkv.bias")
        w.moegate[l] = ptr_of(p + "moegate.weight")
        w.w1[l] = ptr_of(p + "mlp.w1.weight")
        w.w2[l] = ptr_of(p + "mlp.w2.weight")
        w.w3[l] = ptr_of(p + "mlp.w3.weight")
    w.rms_final_weight = ptr_of("model.norm.weight")
    w.wcls = ptr_of("model.embed.weight") if spec.tied else ptr_of("model.output.weight")

    t.state.kvbits = kvbits
    t.n_bandwidth = algorithmic_bytes(spec)
    return t


class HostModel:
    """A generated model held in host memory + the struct Transformer pointing at it
    (what the CPU reference / oracle consume)."""

    def __init__(self, spec: ModelSpec, seed: int = 0, seq_len: Optional[int] = None, tensors=None, kvbits: int = 16):
        self.spec = spec
        self.tensors = tensors if tensors is not None else generate(spec, seed)
        self.tensors = {k: v.contiguous().cpu() for k, v in self.tensors.items()}
        self._seq_len, self._kvbits = seq_len, kvbits
        self.rebind()

    def rebind(self) -> None:
        """(Re)build struct Transformer over self.tensors (call after replacing tensors with copies elsewhere in memory)."""

        def ptr_of(name):
            v = self.tensors.get(name)
            return v.data_ptr() if v is not None else 0

        self.transformer = fill_transformer(self.spec, ptr_of, self._seq_len, self._kvbits)

    @property
    def seq_len(self) -> int:
        return self.transformer.config.seq_len


def teacher_tokens(vocab_size: int, n: int, start: int = 0) -> list:
    """Fixed token list for teacher-forced parity runs: tok_i = (7919 i + 13) mod vocab (SURVEY.md s.8d)."""
    return [((7919 * (i + start)) + 13) % vocab_size for i in range(n)]


def kv_fill_pattern(n_layers_heads: int, n_pos: int, head_dim: int, seed: int):
    """The deterministic pseudo-random cache fill of calm_b200_fill_kv (csrc/stages.cuh k_fill_kv), restated in numpy
    so a CPU checker can be given the SAME cache: returns (k, v) float32 [n_layers_heads, n_pos, head_dim] BEFORE the
    rounding to the cache element type (fp16 RN, or e5m2 RN)."""
    i = np.arange(n_layers_heads * n_pos * head_dim, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (i + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    a = ((z & np.uint64(0xFFFFFF)).astype(np.float64) / 16777216.0 - 0.5) * 2.0
    b = (((z >> np.uint64(24)) & np.uint64(0xFFFFFF)).astype(np.float64) / 16777216.0 - 0.5) * 2.0
    shape = (n_layers_heads, n_pos, head_dim)
    return a.astype(np.float32).reshape(shape), b.astype(np.float32).reshape(shape)
