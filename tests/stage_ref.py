"""Float64 references of the engine's stages, one small function per stage, in plain numpy.

Each function states one operation of the per-token path (oracle/calm_oracle.c gives the order and the rules) on inputs
the caller hands it, so a test can feed a stage the DEVICE's own output of the previous stage and be left with the
arithmetic of the stage under test alone.  `forward` composes them into whole tokens; tests/test_stage_ref.py checks that
composition against the double-precision build of the oracle before any GPU test relies on it.

Weights are decoded once per model to float32 (every fp16 / e5m2 / gf4 weight is a float32 exactly) and multiplied in row
blocks promoted to float64, so no large matrix ever exists in double."""
import ctypes
import ctypes.util

import numpy as np

from calm_b200 import modelgen as mg

KV_SINKS = 2  # include/calm_model.h
_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.powf.argtypes, _libm.powf.restype = [ctypes.c_float, ctypes.c_float], ctypes.c_float


# ---- weights

def decode(t, dtype):
    """A model tensor in its stored format (torch tensor on the host) -> float32 array of the same logical shape."""
    a = t.numpy()
    if dtype == "fp16":
        return a.astype(np.float32)
    if dtype == "fp8":
        return mg.fp8_bytes_to_float(a)
    return mg.gf4_words_to_float(a.view(np.uint32))


class Weights:
    """Decoded weights of a model held on the host (mg.HostModel.tensors); matrices are decoded on first use and kept."""

    def __init__(self, spec, tensors):
        self.spec, self.tensors, self._mat = spec, tensors, {}

    def mat(self, name, expert=None):
        key = (name, expert)
        if key not in self._mat:
            t = self.tensors[name]
            self._mat[key] = decode(t if expert is None else t[expert], self.spec.dtype)
        return self._mat[key]

    def vec(self, name):
        t = self.tensors.get(name)
        return None if t is None else t.numpy().astype(np.float64)

    def layer(self, l, name, expert=None):
        return self.mat(f"model.layers.{l}.{name}.weight", expert)

    def classifier(self):
        return self.mat("model.embed.weight" if self.spec.tied else "model.output.weight")


def matvec(W, x, block=2048):
    """W[d, n] . x[n] (or x[n, m]) in float64, W promoted block by block."""
    x = np.asarray(x, np.float64)
    out = np.empty((W.shape[0],) + x.shape[1:], np.float64)
    for r in range(0, W.shape[0], block):
        out[r:r + block] = W[r:r + block].astype(np.float64) @ x
    return out


# ---- element-wise pieces

def norm(x, weight, eps, ln):
    """RMSNorm, or the mean-subtracting LayerNorm without bias; x[..., dim]."""
    x = np.asarray(x, np.float64)
    if ln:
        x = x - x.mean(-1, keepdims=True)
    return x / np.sqrt((x * x).mean(-1, keepdims=True) + eps) * weight


def rope_angles(spec, pos):
    """fp32 angles pos * theta^(-j / rotary_dim) for j = 0, 2, ...: the frequency from the C library's powf and the product
    in fp32, as the engine forms them on the host, so both sides rotate by the same angle.  pos: int or int array."""
    rd = spec.rotary_dim if spec.rotary_dim is not None else spec.head_dim
    freq = np.array([0.0 if j >= rd else np.float32(1.0) / np.float32(_libm.powf(spec.rope_theta, float(np.float32(j) / np.float32(rd))))
                     for j in range(0, spec.head_dim, 2)], np.float32)
    return np.multiply.outer(np.asarray(pos).astype(np.float32), freq).astype(np.float32)


def rope(v, angles, head_dim):
    """Rotate adjacent pairs of v[..., heads * head_dim] by angles[..., head_dim / 2] (cos / sin in float64)."""
    p = np.asarray(v, np.float64).reshape(v.shape[:-1] + (-1, head_dim // 2, 2))
    c, s = np.cos(angles.astype(np.float64))[..., None, :], np.sin(angles.astype(np.float64))[..., None, :]
    out = np.stack([p[..., 0] * c - p[..., 1] * s, p[..., 0] * s + p[..., 1] * c], -1)
    return out.reshape(v.shape)


def ulp(v, kvbits):
    """Spacing of the cache format (fp16, or e5m2 when kvbits == 8) around |v|."""
    a = np.abs(np.asarray(v, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - (10 if kvbits == 16 else 2))


def round_kv(v, kvbits):
    """Round to nearest even into the cache format; e5m2 saturates at 57344."""
    v = np.asarray(v, np.float64)
    q = ulp(v, kvbits)
    r = np.rint(v / q) * q  # power-of-two scaling is exact; rint rounds ties to even
    return np.clip(r, -57344.0, 57344.0) if kvbits == 8 else r


def kv_slot(pos, seq_len):
    """(slot written, slots attended, sinks re-rotated) of the rolling cache at `pos`."""
    sink = KV_SINKS if pos >= seq_len else 0
    return sink + (pos - sink) % (seq_len - sink), min(pos + 1, seq_len), sink


def act(spec, u):
    if spec.act_type == "gelu":
        return 0.5 * u * (1.0 + np.tanh(0.797885 * (u + 0.044715 * u * u * u)))
    return u / (1.0 + np.exp(-u))


# ---- stages

def embed(w, token):
    return w.mat("model.embed.weight")[token].astype(np.float64)


def qkv(w, l, x, pos):
    """The attention norm, q / k / v with bias and clip, RoPE on q and k.  x[dim] at `pos`, or x[n, dim] at pos[n].
    Returns (q, k, v, xn): q and k rotated, k and v before their rounding into the cache."""
    s = w.spec
    p = f"model.layers.{l}."
    xn = norm(x, w.vec(p + "attn.norm.weight"), s.norm_eps, s.norm_type != "rmsnorm")
    out = []
    bias = w.vec(p + "attn.wqkv.bias")
    for name, off, n in (("wq", 0, s.q_dim), ("wk", s.q_dim, s.kv_dim), ("wv", s.q_dim + s.kv_dim, s.kv_dim)):
        y = matvec(w.layer(l, "attn." + name), xn.T).T
        if bias is not None:
            y = y + bias[off:off + n]
        if s.qkv_clip is not None:
            y = np.clip(y, -s.qkv_clip, s.qkv_clip)
        out.append(y)
    ang = rope_angles(s, pos)
    return rope(out[0], ang, s.head_dim), rope(out[1], ang, s.head_dim), out[2], xn


def rotate_sinks(spec, keys):
    """keys[n_kv_heads, KV_SINKS, head_dim] moved on by one position, before rounding."""
    return rope(keys, rope_angles(spec, 1), spec.head_dim)


def attention(spec, q, keys, values, kv_len):
    """Softmax attention of q[q_dim] over slots [0, kv_len) of keys / values[n_kv_heads, seq_len, head_dim]."""
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    out = np.empty((spec.n_heads, hd), np.float64)
    qh = np.asarray(q, np.float64).reshape(spec.n_heads, hd)
    for g in range(spec.n_kv_heads):
        K, V = np.asarray(keys[g, :kv_len], np.float64), np.asarray(values[g, :kv_len], np.float64)
        sc = qh[g * kv_mul:(g + 1) * kv_mul] @ K.T / np.sqrt(hd)
        p = np.exp(sc - sc.max(-1, keepdims=True))
        out[g * kv_mul:(g + 1) * kv_mul] = (p / p.sum(-1, keepdims=True)) @ V
    return out.reshape(-1)


def wo(w, l, x, att):
    """x + Wo . att: the residual stream the FFN reads."""
    return np.asarray(x, np.float64) + matvec(w.layer(l, "attn.wo"), np.asarray(att, np.float64).T).T


def router(w, l, xn):
    """(experts, weights, logits): repeated arg-max, lowest index on ties; exp(l - max) normalised over the chosen."""
    s = w.spec
    logits = matvec(w.layer(l, "moegate"), xn)
    left, experts = logits.copy(), []
    for _ in range(s.n_experts_active):
        experts.append(int(np.argmax(left)))  # first maximum
        left[experts[-1]] = -np.inf
    e = np.exp(logits[experts] - logits.max())
    return experts, e / e.sum(), logits


def ffn_input(w, l, x1, xn_attn):
    s = w.spec
    if s.norm_type == "layernorm_par":
        return xn_attn
    return norm(x1, w.vec(f"model.layers.{l}.mlp.norm.weight"), s.norm_eps, s.norm_type != "rmsnorm")


def ffn_up(w, l, xn, expert=None):
    """act(w1 . xn) * (w3 . xn); xn[dim] or xn[n, dim]."""
    u1 = matvec(w.layer(l, "mlp.w1", expert), xn.T).T
    u3 = matvec(w.layer(l, "mlp.w3", expert), xn.T).T
    return act(w.spec, u1) * u3


def ffn_down(w, l, x1, hb, experts=(None,), weights=(1.0,)):
    """x1 + sum_e weight_e W2_e . hb_e; hb[len(experts), hidden] (dense: hb[hidden] or hb[n, hidden])."""
    x = np.asarray(x1, np.float64).copy()
    hb = np.asarray(hb, np.float64)
    for i, (e, g) in enumerate(zip(experts, weights)):
        x += g * matvec(w.layer(l, "mlp.w2", e), (hb if e is None else hb[i]).T).T
    return x


def classifier(w, x):
    s = w.spec
    return matvec(w.classifier(), norm(x, w.vec("model.norm.weight"), s.norm_eps, s.norm_type != "rmsnorm"))


# ---- the composition: whole tokens on a float64 model of the cache

class Cache:
    def __init__(self, spec, seq_len, kvbits):
        self.seq_len, self.kvbits = seq_len, kvbits
        self.k = np.zeros((spec.n_layers, spec.n_kv_heads, seq_len, spec.head_dim))
        self.v = np.zeros_like(self.k)


def forward(w, cache, token, pos, after_store=None):
    """One token through every layer.  Returns (logits, q, att, x) with q / att / x stacked per layer.  after_store(l) runs
    once layer l's cache entries are written, before its attention reads them."""
    s = w.spec
    slot, kv_len, sinks = kv_slot(pos, cache.seq_len)
    x = embed(w, token)
    taps = [], [], []
    for l in range(s.n_layers):
        q, k, v, xn = qkv(w, l, x, pos)
        cache.k[l, :, slot] = round_kv(k, cache.kvbits).reshape(s.n_kv_heads, s.head_dim)
        cache.v[l, :, slot] = round_kv(v, cache.kvbits).reshape(s.n_kv_heads, s.head_dim)
        if sinks:
            cache.k[l, :, :sinks] = round_kv(rotate_sinks(s, cache.k[l, :, :sinks]), cache.kvbits)
        if after_store:
            after_store(l)
        att = attention(s, q, cache.k[l], cache.v[l], kv_len)
        x1 = wo(w, l, x, att)
        xn2 = ffn_input(w, l, x1, xn)
        if s.n_experts:
            experts, weights, _ = router(w, l, xn2)
            x = ffn_down(w, l, x1, np.stack([ffn_up(w, l, xn2, e) for e in experts]), experts, weights)
        else:
            x = ffn_down(w, l, x1, ffn_up(w, l, xn2))
        for t, a in zip(taps, (q, att, x)):
            t.append(a)
    return (classifier(w, x),) + tuple(np.stack(t) for t in taps)
