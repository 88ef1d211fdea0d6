"""Decode, the prompt pass and the short-block paths against float64 at 32K-128K-token contexts, and the cache's per-layer
offsets past 2^31 bytes and past 2^31 elements.

The method is test_stages_gpu.py's: each stage read back with calm_b200_read_state / calm_b200_read_kv and compared with
tests/stage_ref.py fed the DEVICE's own output of the stage before it, through the sibling files' own checks
(check_decode_step, check_pass, and the last-step checks of decode_sample_n, verify_greedy, decode_sample_batch and
decode_sample_queue_context).  What changes with length:

1. Decode at Llama-3-8B widths on both sides of the k_attn2 -> k_attn switch (make_plan's rule is restated in
   attn2_serves and the plan line must agree with it), at 32768 and 131072 positions with RoPE past 65536 and the rolled
   cache with its re-rotated sinks, at Llama-3-70B and Qwen2-0.5B widths, and on a model whose scores are large enough
   that the softmax over 131072 keys is peaked rather than a near-uniform average.
2. The prompt pass over a warm cache of 126000 (Llama-3-8B) and 30000 (Qwen2) positions.
3. decode_sample_n and verify_greedy at position 100000 (about 780 shared 128-key chunks folded by k_sn_fold), the queue
   over one 32768-token context shared by 16 requests, and decode_sample_batch with a 40000-token prompt.
4. A deep model whose caches lie past 2^31 bytes (9 layers) and past 2^31 elements (17 layers).  Every layer but the
   last has wo and w2 zero, so every layer's input is exactly the embedding row: every layer's written cache entries are
   checked against float64 q / k / v of that layer, and the last layer's stages exactly as layer 0's are elsewhere.  The
   cache is poisoned above the filled slots first; afterwards the first, middle and last two layers are compared whole,
   on the device and bit for bit: the filled slots must still hold calm_b200_fill_kv's pattern and every slot past the
   written ones must still hold the poison.  Coverage: this checks the writes of every layer, but the attention (the
   reads) of the last layer only.

The float64 matrix products and the attention run on the GPU in torch float64 (keys and values of one layer read back
once per call and kept on the device while the checks use them).  Every case prints its wall time; the last test prints
each stage's largest error beside its bound.

Bounds: the suite's own (STAGE_TOL, pf_tol) hold at every length here, so this file adds none.  The attention errors do
not grow with kv_len: on an H100 80GB HBM3 (700 W limit, 132 SMs) the largest were 6.7e-7 of scale for k_attn (the x16
peaked softmax at 131072 keys; near-uniform softmaxes stay below 1e-8), 2.4e-7 for k_pf_attn and 4.5e-8 for k_sn_attn,
against bounds of 2e-6 and 3e-6.  The whole file took 168 s there."""
import os
import sys
import time
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
import test_decode_sample_batch_gpu as batch  # noqa: E402
import test_decode_sample_n_gpu as sample_n  # noqa: E402
import test_decode_sample_queue_context_gpu as queue_context  # noqa: E402
import test_stages_gpu as ts  # noqa: E402
import test_verify_gpu as verify  # noqa: E402
from test_prefill_stages_gpu import check_pass, f64  # noqa: E402,F401  (f64 is a fixture)
from test_stages_gpu import L8B, REG, V4K, check_decode_step, check_entries, make_model, pf_tol, run_decode  # noqa: E402
from test_variants_gpu import RING, plan_of  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

worst = {}  # this file's largest error per stage key, (error, bound, share)
peak = {}  # the largest softmax weight of the last float64 attention


# ---- float64 attention on the device
_on_device = {}


def on_device(a):
    """A float64 device copy of host array `a`, kept while the same array object is handed in again (one layer's keys are
    attended by many rows)."""
    hit = _on_device.get(id(a))
    if hit is None or hit[0] is not a:
        if len(_on_device) >= 4:
            _on_device.clear()
        hit = _on_device[id(a)] = (a, torch.as_tensor(np.ascontiguousarray(a), device="cuda").to(torch.float64))
    return hit[1]


def attention_on_device(spec, q, keys, values, kv_len):
    """stage_ref.attention in float64 on the GPU."""
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    K, V = on_device(keys)[:, :kv_len], on_device(values)[:, :kv_len]
    qh = torch.as_tensor(np.asarray(q, np.float64), device="cuda").reshape(spec.n_kv_heads, kv_mul, hd)
    sc = qh @ K.transpose(1, 2) / np.sqrt(hd)
    p = torch.exp(sc - sc.amax(-1, keepdim=True))
    p /= p.sum(-1, keepdim=True)
    peak["p"] = float(p.max())
    return (p @ V).reshape(-1).cpu().numpy()


@pytest.fixture
def f64_long(f64, monkeypatch):
    """test_prefill_stages_gpu's device products, the attention on the device too, and this file's record of errors."""
    monkeypatch.setattr(sr, "attention", attention_on_device)
    monkeypatch.setattr(ts, "worst_seen", worst)
    monkeypatch.delenv("CALM_B200_QUIET", raising=False)
    t0 = time.perf_counter()
    yield
    _on_device.clear()
    torch.cuda.empty_cache()
    print(f"  wall time {time.perf_counter() - t0:.1f} s")


@pytest.fixture(scope="module")
def l8b():
    """One Llama-3-8B-width layer (fp8 weights, vocabulary 4096), shared by the cases of this file."""
    return make_model(L8B, 1)


# ---- 1. decode
def attn2_serves(spec, seq_len, kvbits):
    """make_plan's choice of k_attn2 (engine.cu), restated for shapes k_attn2 is instantiated for and whose grid is resident:
    query heads per CTA hg = the largest divisor of kv_mul up to 8, units = n_kv_heads * kv_mul / hg, slices = SMs / units
    (at most ceil(seq_len / 64) and ATTN2_MAXB + 4 = 36), nbmax = ceil(ceil(seq_len / 16) / slices) blocks of 16
    positions per CTA; k_attn2 serves while nbmax <= ATTN2_MAXB = 32 and its shared memory (attn2_smem_bytes: K and V
    blocks, fp32 scores, f16 hi / lo probabilities, the CTA's record) stays within 200 KB.  At Llama-3-8B widths on 132 SMs
    (8 units x 16 slices) that is seq_len <= 5888 with an fp16 cache (nbmax 23: 202400 bytes; 24: 211104) and
    seq_len <= 8192 with e5m2 (nbmax 32)."""
    kv_mul, hd = spec.n_heads // spec.n_kv_heads, spec.head_dim
    hg = max(h for h in range(1, 9) if kv_mul % h == 0)
    units = spec.n_kv_heads * (kv_mul // hg)
    slices = max(1, min(torch.cuda.get_device_properties(0).multi_processor_count // units, -(-seq_len // 64), 36))
    nbmax = -(-(-(-seq_len // 16)) // slices)
    npos = 16 * nbmax
    smem = 2 * npos * hd * kvbits // 8 + hg * npos * 4 + 2 * hg * (npos + 8) * 2 + hg * (hd + 2) * 4
    return nbmax <= 32 and smem <= 200 * 1024


def positions(seq_len, *extra):
    """The last slot, a kv_len one past a multiple of 16 slices of 16 positions (a one-position last block), a slot in the
    rolled cache's last slice, and `extra`."""
    return [(17, seq_len - 1), (9, 256 * (seq_len // 512)), (3, ("kv", "last-slice"))] + [(5 + 2 * i, p) for i, p in enumerate(extra)]


@pytest.mark.parametrize("kvbits,last", [(16, 5888), (8, 8192)])
def test_decode_on_both_sides_of_the_attention_switch(kvbits, last, l8b, f64_long, capfd, monkeypatch):
    """The longest cache k_attn2 serves and one position more, at Llama-3-8B widths."""
    for seq_len in (last, last + 1):
        kernel = "k_attn2" if attn2_serves(L8B, seq_len, kvbits) else "k_attn"
        assert kernel == ("k_attn2" if seq_len == last else "k_attn"), f"seq_len {seq_len} kv{kvbits}: the restated rule no longer puts the switch here"
        run_decode(L8B, 1, seq_len, kvbits, positions(seq_len), kernel, RING, capfd, monkeypatch, f"llama3-8b seq_len {seq_len} {kernel}", model=l8b)


LONG = [(17, 0), (9, 65535), (3, 65536)]


@pytest.mark.parametrize("kvbits", [16, 8])
@pytest.mark.parametrize("seq_len", [32768, 131072])
def test_decode_at_long_contexts(seq_len, kvbits, l8b, f64_long, capfd, monkeypatch):
    """Positions 0, 65535, 65536 (RoPE past 2^16; rolled at seq_len 32768), the last slot and seq_len + 1000 (rolled, with
    re-rotated sinks)."""
    steps = LONG + [(5, seq_len - 1), (11, seq_len + 1000)]
    run_decode(L8B, 1, seq_len, kvbits, steps, "k_attn", RING, capfd, monkeypatch, f"llama3-8b seq_len {seq_len}", model=l8b)


WIDTHS = {
    "llama3-70b kv_mul8": (replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K), 16, RING),
    "qwen2-0.5b kv_mul7 hd64": (replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=1, vocab_size=V4K), 8, REG),
}


@pytest.mark.parametrize("case", sorted(WIDTHS))
def test_decode_at_32k_other_widths(case, f64_long, capfd, monkeypatch):
    spec, kvbits, matvec = WIDTHS[case]
    assert not attn2_serves(spec, 32768, kvbits)
    run_decode(spec, 3, 32768, kvbits, LONG + [(5, 32767), (11, 32768 + 1000)], "k_attn", matvec, capfd, monkeypatch, case)


@pytest.mark.parametrize("scale,lo,hi", [(4, 1e-3, 0.5), (16, 0.5, 1.0)])
def test_decode_with_a_peaked_softmax(scale, lo, hi, f64_long, capfd):
    """wq x scale (a power of two: exact in fp16) spreads the scores over the fill's keys (standard deviation about 3 at
    x4, 12 at x16), so the softmax over 131072 keys is not a near-uniform average that would hide an error in the long
    sums and the slice fold: at x4 the largest weight is a few percent and many keys share the rest, at x16 one key
    carries nearly all of it.  The largest weight must lie in [lo, hi]."""
    spec = replace(L8B, dtype="fp16")
    tensors = mg.generate(spec, 11, device="cuda")
    tensors["model.layers.0.attn.wq.weight"] *= scale
    torch.cuda.synchronize()
    w = sr.Weights(spec, {k: v.cpu() for k, v in tensors.items()})
    with lib.DeviceModel(spec, tensors, seq_len=131072, kvbits=16) as dm:
        plan = plan_of(capfd)
        assert plan[0] == "k_attn"
        with capfd.disabled():
            for token, pos in ((17, 131071), (9, 131072 + 1000)):
                check_decode_step(dm, w, token, pos, 16, plan, f"llama3-8b fp16 wq x{scale}")
                print(f"  largest softmax weight {peak['p']:.3g}")
                assert lo <= peak["p"] <= hi, f"largest softmax weight {peak['p']:.3g} outside [{lo}, {hi}]: the case lost its premise"


# ---- 2. the prompt pass over a deep warm cache: (spec, kvbits, seq_len, pos0, n)
PROMPT = {
    "llama3-8b pos0 126000 n 2100": (L8B, 16, 131072, 126000, 2100),  # two blocks, the second 52 rows (a partial tile)
    "qwen2-0.5b pos0 30000 to the last slot": (WIDTHS["qwen2-0.5b kv_mul7 hd64"][0], 16, 32768, 30000, 2768),
}


@pytest.mark.parametrize("case", sorted(PROMPT))
def test_prompt_pass_over_a_deep_cache(case, f64_long):
    spec, kvbits, seq_len, pos0, n = PROMPT[case]
    tensors, w = make_model(spec, 4)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        dm.fill_kv(pos0, seed=6)
        check_pass(dm, w, mg.teacher_tokens(spec.vocab_size, n), pos0, kvbits, case)


# ---- 3. the short-block paths at long prompts
def test_sample_n_at_position_100000(l8b, f64_long):
    """16 sequences over a 100000-token prompt: 782 prompt chunks of 128 keys, folded by k_sn_fold."""
    with lib.DeviceModel(L8B, l8b[0], seq_len=100352, kvbits=16) as dm:
        dm.fill_kv(100000, seed=6)
        sample_n.check_last_step(dm, l8b[1], 16, 16, 2, 100000, "llama3-8b n16 t2 pos 100000")


def test_verify_at_position_100000(l8b, f64_long):
    with lib.DeviceModel(L8B, l8b[0], seq_len=100352, kvbits=16) as dm:
        dm.fill_kv(100000, seed=6)
        verify.check_block(dm, l8b[1], 16, 16, 100000, "llama3-8b n16 pos 100000")


def test_queue_over_one_32k_context(l8b, f64_long):
    """16 requests on one 32768-token context (256 shared chunks), 8 rows at a time, so the last step's rows were admitted
    in different rounds and sit at different own steps.  The call's own prompt pass computes the context."""
    lens = [1 + 5 * b for b in range(16)]
    with lib.DeviceModel(L8B, l8b[0], seq_len=36864, kvbits=16) as dm:
        queue_context.check_last_step(dm, l8b[1], 16, [32768], [0] * 16, lens, [40 - 2 * b for b in range(16)], 8, "llama3-8b 32k context r8")


def test_batch_with_a_40k_prompt(l8b, f64_long):
    with lib.DeviceModel(L8B, l8b[0], seq_len=40960, kvbits=8) as dm:
        batch.check_last_step(dm, l8b[1], 8, [300, 40001, 9, 1, 130], 3, "llama3-8b 40001 beside short prompts")


# ---- 4. cache offsets past 2^31 on a deep model
def pass_through_model(spec, seed):
    """wo and w2 zero in every layer but the last: each layer adds nothing to the residual stream."""
    tensors = mg.generate(spec, seed, device="cuda")
    for l in range(spec.n_layers - 1):
        tensors[f"model.layers.{l}.attn.wo.weight"].zero_()
        tensors[f"model.layers.{l}.mlp.w2.weight"].zero_()
    torch.cuda.synchronize()
    return tensors, sr.Weights(spec, {k: v.cpu() for k, v in tensors.items()})


class _DeviceArray:
    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<i2", "data": (ptr, False), "version": 3}


def raw_cache(dm):
    """The fp16 key and value caches as int16 bit patterns [layer, kv head, slot, dim], viewed in place on the device:
    read_state widens to float and makes every NaN the same, so the poison's bits are only visible here."""
    s, st = dm.spec, dm.transformer.state
    shape = (s.n_layers, s.n_kv_heads, dm.seq_len, s.head_dim)
    torch.cuda.synchronize()
    return [torch.as_tensor(_DeviceArray(p, shape), device="cuda") for p in (st.key_cache, st.value_cache)]


def fill_pattern(lh, n_pos, head_dim, seed):
    """modelgen.kv_fill_pattern's (k, v) of cache row lh = layer * n_kv_heads + head, on the device in int64 (wrapping
    products, shifts masked to be logical) and rounded to fp16 as bit patterns."""
    def srl(z, s):
        return (z >> s) & ((1 << (64 - s)) - 1)

    def i64(c):
        return c - (1 << 64) if c >= 1 << 63 else c

    i = torch.arange(lh * n_pos * head_dim, (lh + 1) * n_pos * head_dim, dtype=torch.int64, device="cuda")
    z = (i + 1) * i64(0x9E3779B97F4A7C15) + seed
    z = (z ^ srl(z, 30)) * i64(0xBF58476D1CE4E5B9)
    z = (z ^ srl(z, 27)) * i64(0x94D049BB133111EB)
    z = z ^ srl(z, 31)
    a = ((z & 0xFFFFFF).to(torch.float64) / 16777216.0 - 0.5) * 2.0
    b = ((srl(z, 24) & 0xFFFFFF).to(torch.float64) / 16777216.0 - 0.5) * 2.0
    return [x.to(torch.float32).to(torch.float16).view(torch.int16).reshape(n_pos, head_dim) for x in (a, b)]


def check_whole_layers(dm, label, fill_n, fill_seed, written_end):
    """Layers 0, L / 2, L - 2 and L - 1 whole: slots [0, fill_n) hold the fill, slots [written_end, seq_len) the poison."""
    s = dm.spec
    K, V = raw_cache(dm)
    for l in sorted({0, s.n_layers // 2, s.n_layers - 2, s.n_layers - 1}):
        for h in range(s.n_kv_heads):
            want = fill_pattern(l * s.n_kv_heads + h, fill_n, s.head_dim, fill_seed)
            for name, got, ref in (("K", K, want[0]), ("V", V, want[1])):
                bad = (got[l, h, :fill_n] != ref).nonzero()
                assert len(bad) == 0, f"{label}: layer {l} kv head {h} {name}: filled slot {int(bad[0, 0])} changed"
                bad = (got[l, h, written_end:] != -1).nonzero()
                assert len(bad) == 0, f"{label}: layer {l} kv head {h} {name}: slot {written_end + int(bad[0, 0])} past the written ones is not the poison"
    print(f"  {label}: layers {sorted({0, s.n_layers // 2, s.n_layers - 2, s.n_layers - 1})}: slots below {fill_n} hold the fill, slots from {written_end} the poison")


def check_every_layer(dm, w, tokens, pos, slots, kernel, key, tol, label):
    """Every layer's cache entries at `slots` (written from tokens at positions pos) against float64 q / k / v of that
    layer applied to the embedding rows."""
    s, slots = w.spec, np.asarray(slots)
    X0 = w.mat("model.embed.weight")[np.asarray(tokens)].astype(np.float64)
    hd = s.head_dim
    for l in range(s.n_layers):
        _, k_ref, v_ref, _ = sr.qkv(w, l, X0, np.asarray(pos))
        kv = [dm.read_kv(l, int(t)) for t in slots]
        for name, i, ref in (("K", 0, k_ref), ("V", 1, v_ref)):
            check_entries(f"{label} layer {l}", name, kernel, np.stack([e[i] for e in kv]), ref, 16,
                          lambda i: f"slot {slots[i[0]]} kv head {i[1] // hd} dim {i[1] % hd}", key, tol)


@pytest.mark.parametrize("n_layers", [9, 17])
def test_deep_cache_every_layer(n_layers, f64_long, capfd):
    """attn-l8's attention shape (32 / 8 heads of 128) with n_layers layers at seq_len 131072 and an fp16 cache: the last
    layer's base is 2^31 bytes (9 layers) or 2^31 elements (17 layers) into the cache.  A prompt pass of 1000 rows at
    130000, a decode step at 131000 and decode_sample_n of 16 x 2 tokens at 131001, each checked at every layer."""
    spec = replace(mg.SPECS["attn-l8"], n_layers=n_layers)
    S, last, label = 131072, n_layers - 1, f"{n_layers} layers"
    base = last * spec.n_kv_heads * S * spec.head_dim
    assert (2 ** 31 <= 2 * base, base >= 2 ** 31) == (True, n_layers == 17)
    tensors, w = pass_through_model(spec, 9)
    with lib.DeviceModel(spec, tensors, seq_len=S, kvbits=16) as dm:
        plan = plan_of(capfd)
        assert plan[0] == "k_attn"
        with capfd.disabled():
            assert np.array_equal(fill_pattern(1, 50, 128, 6)[0].cpu().numpy(),
                                  mg.kv_fill_pattern(2, 50, 128, 6)[0][1].astype(np.float16).view(np.int16)), "fill_pattern is not modelgen's"
            dm.poison(130000)
            dm.fill_kv(130000, seed=6)
            toks = mg.teacher_tokens(spec.vocab_size, 1000)
            check_pass(dm, w, toks, 130000, 16, f"{label} prompt pass", layer=last)
            pos = 130000 + np.arange(1000)
            check_every_layer(dm, w, toks, pos, pos, "k_pf_gemm QKV", "pf_kv", pf_tol(spec.dim), f"{label} prompt pass")
            check_whole_layers(dm, f"{label} prompt pass", 130000, 6, 131000)

            check_decode_step(dm, w, 17, 131000, 16, plan, f"{label} decode", layer=last)  # fills slots below 131000 again
            check_every_layer(dm, w, [17], [131000], [131000], "k_qkv", "kv", None, f"{label} decode")
            check_whole_layers(dm, f"{label} decode", 131000, 5, 131001)

            toks = sample_n.check_last_step(dm, w, 16, 16, 2, 131001, f"{label} pos 131001", layer=last)
            rows = np.arange(16)
            check_every_layer(dm, w, np.concatenate([np.full(16, 3), toks[:, 0]]), np.repeat([131001, 131002], 16),
                              131001 + np.concatenate([rows, 16 + rows]), "k_vf_gemm QKV", "vf_kv", pf_tol(spec.dim), f"{label} sample_n")
            check_whole_layers(dm, f"{label} sample_n", 131000, 5, 131033)


def test_zz_summary_of_largest_errors():
    """Runs last in this file: each stage's largest error in this file's cases, beside its bound."""
    if not worst:
        pytest.skip("the long-context tests did not run in this session")
    print("\n  long contexts, largest error per stage: " + ", ".join(f"{k} {e:.2e} of {tol:.1e}" for k, (e, tol, _) in sorted(worst.items())))
    assert all(e <= tol for e, tol, _ in worst.values())
