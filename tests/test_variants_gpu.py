"""The model switches, query groupings and cache edges on the kernels that serve real widths, against the CPU oracle.

The tiny-* parity shapes run the oldest kernels (k_ffn_up, k_matres, k_attn) and the prompt pass rejects them.  Here:
  * GELU + qkv clip + partial rotary, LayerNorm and parallel LayerNorm on a shape the ring-fed matvecs (k_ffn_up_ring,
    k_matres_ring), k_attn2 and the wgmma prompt pass all serve -- decode teacher-forced, and a prompt of a partial tile;
  * the prompt pass at 1, 7 and 8 query heads per kv head (k_pf_attn's KM = 1 instantiation, and KM = 4 looping twice),
    and the Qwen2-0.5B widths;
  * prompt-pass block edges: one token, two 2048-token chunks, a block that ends at seq_len and is followed by decode steps
    that roll the cache over, a block that would roll over (fed token by token), and a second, longer turn (buffers regrow);
  * the device-resident greedy / sampling loops stepping across pos == seq_len.
Every case asserts the kernel that served it: prepare_cuda's plan lines, forward_prefill_cuda's return value."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import KV_ATOL, KV_RTOL, TOL_SIGMA  # noqa: E402
from test_prefill_gpu import _both, _check  # noqa: E402
from test_scale_gpu import TOL8_SIGMA  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY  # noqa: E402

# the shape of test_scale_gpu.test_ring_fed_kernels_vs_oracle: rows of whole 1 KB chunks (ring kernels), 4 query heads per
# kv head of 128 (k_attn2), every dim a multiple of 128 (prompt pass)
_BASE = replace(mg.SPECS["pf-tiny-hd128"], name="var", dim=2048, hidden_dim=4096, n_heads=8, n_kv_heads=2, n_layers=2)
SEQ_LEN = 512
VARIANTS = {  # switch on, and the settings that turn each of its switches off again
    "gelu-clip-rot64": (replace(_BASE, act_type="gelu", qkv_clip=0.5, rotary_dim=64, rope_theta=1e4),  # Phi-2 style
                        [{"act_type": "silu"}, {"qkv_clip": None}, {"rotary_dim": None}]),
    "layernorm": (replace(_BASE, norm_type="layernorm"), [{"norm_type": "rmsnorm"}]),
    "layernorm-par": (replace(_BASE, norm_type="layernorm_par"), [{"norm_type": "layernorm"}]),
}
RING = {"up": "k_ffn_up_ring", "wo": "k_matres_ring", "down": "k_matres_ring"}


def plan_of(capfd):
    """(attention kernel, slices, {stage: matvec kernel}) from the plan lines prepare_cuda printed."""
    out = capfd.readouterr().out.splitlines()
    att = [l for l in out if l.startswith("# plan: attention ")]
    mv = [l for l in out if l.startswith("# plan: matvec ")]
    assert att and mv, out
    w = att[-1].split()
    stages = dict(s.split() for s in mv[-1][len("# plan: matvec "):].split(", "))
    return w[3].rstrip(","), int(w[-2]), stages


def kv_close(got, want, kvbits, same=0.95):
    """Lists of (k, v) cache entries.  fp16 cache: the rule of test_prefill_gpu._check; e5m2 cache: equal or neighbouring values."""
    assert len(got) == len(want)
    for pa, pb in zip(got, want):
        for a, b in zip(pa, pb):
            if kvbits == 16:
                np.testing.assert_allclose(a, b, rtol=KV_RTOL, atol=max(KV_ATOL, 5e-4 * float(np.abs(b).max())))
            else:
                assert (np.abs(a - b) <= 0.26 * np.maximum(np.abs(a), np.abs(b)) + 2e-5).all() and (a == b).mean() > same


def logits_close(got, want, tol, label):
    sigma = float(want.std())
    err = float(np.abs(got - want).max())
    print(f"{label}: |cuda - oracle| {err:.2e} = {err / sigma:.1e} sigma")
    assert err <= tol * sigma, (label, err, sigma)
    return sigma


def oracle_run(oracle_pkg, host, toks, kind="port", pos0=0, warm=()):
    """Teacher-forced oracle logits of `toks` at pos0.. (after `warm` at 0..), and the checker (its cache still held)."""
    ck = oracle_pkg.Checker(kind)
    ck.prepare(host)
    for i, t in enumerate(warm):
        ck.forward(host, int(t), i, FF_UPDATE_KV_ONLY)
    return np.stack([ck.forward(host, int(t), pos0 + i) for i, t in enumerate(toks)]), ck


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_switch_changes_the_oracle(oracle_pkg, variant):
    """The switch is live on this shape: the oracle's logits with it off (same weights) move by far more than the tolerance."""
    spec, offs = VARIANTS[variant]
    tensors = mg.generate(spec, 21)
    toks = mg.teacher_tokens(spec.vocab_size, 12)
    on, ck = oracle_run(oracle_pkg, mg.HostModel(spec, tensors=tensors, seq_len=SEQ_LEN), toks)
    for off in offs:
        spec_off = replace(spec, **off)
        t = dict(tensors)
        if spec.norm_type == "layernorm_par":  # the sequential norm needs an FFN norm weight: reuse the attention norm's
            t.update({f"model.layers.{l}.mlp.norm.weight": tensors[f"model.layers.{l}.attn.norm.weight"] for l in range(spec.n_layers)})
        host_off = mg.HostModel(spec_off, tensors=t, seq_len=SEQ_LEN)
        got, ck2 = oracle_run(oracle_pkg, host_off, toks)
        ck2.release(host_off)
        d = float(np.abs(on - got).max() / on.std())
        print(f"{variant} vs {off}: |on - off| {d:.2f} sigma")
        assert d >= 20 * TOL_SIGMA, (variant, off, d)


@pytest.mark.gpu
@pytest.mark.parametrize("variant,dtype,kvbits", [("gelu-clip-rot64", "fp8", 16), ("gelu-clip-rot64", "gf4", 8), ("layernorm", "fp8", 16),
                                                  ("layernorm-par", "fp8", 16), ("layernorm-par", "fp16", 16)])
def test_switches_on_ring_attn2_and_prompt_pass_vs_oracle(oracle_pkg, variant, dtype, kvbits, capfd, monkeypatch):
    """Decode teacher-forced over 24 tokens (k_ffn_up_ring, k_matres_ring, k_attn2), then a 200-token prompt pass (a partial
    second token tile) and the next token, each against the oracle: logits, clear-margin argmax, and KV entries."""
    monkeypatch.delenv("CALM_B200_QUIET", raising=False)
    spec = replace(VARIANTS[variant][0], dtype=dtype)
    host = mg.HostModel(spec, seed=21, seq_len=SEQ_LEN, kvbits=kvbits)
    n_dec, n_pf = 24, 200
    toks = mg.teacher_tokens(spec.vocab_size, n_pf + 1)
    ref, ck = oracle_run(oracle_pkg, host, toks)
    tol = TOL_SIGMA if kvbits == 16 else TOL8_SIGMA
    label = f"{variant}/{dtype}/kv{kvbits}"

    with lib.DeviceModel(spec, host.tensors, seq_len=SEQ_LEN, kvbits=kvbits) as dm:
        kernel, _, stages = plan_of(capfd)
        assert kernel == "k_attn2"
        assert stages == (dict(RING, wo="k_matres") if dtype == "gf4" else RING), stages  # gf4 wo rows are 512 bytes
        got = np.stack([dm.forward(t, i) for i, t in enumerate(toks[:n_dec])])
        kv_dev = [dm.read_kv(l, p) for l in range(spec.n_layers) for p in (0, 11, n_dec - 1)]
    want = ref[:n_dec]
    sigma = logits_close(got, want, tol, label + " decode")
    srt = np.sort(want, 1)
    safe = (srt[:, -1] - srt[:, -2]) > 2 * tol * sigma
    assert (got.argmax(1)[safe] == want.argmax(1)[safe]).all()
    kv_ref = [ck.read_kv(host, l, p) for l in range(spec.n_layers) for p in (0, 11, n_dec - 1)]
    kv_close(kv_dev, kv_ref, kvbits, same=0.97)

    serial, batched = _both(spec, host.tensors, toks, 0, SEQ_LEN, kvbits)  # asserts prefill() == 1
    _check(spec, serial, batched, kvbits, label + f" prompt pass n = {n_pf}")
    logits_close(batched[0], ref[-1], tol, label + f" after a {n_pf}-token prompt pass")
    positions = sorted({0, n_pf // 3, n_pf // 2, n_pf - 1})  # the positions _both samples
    kv_ref = [ck.read_kv(host, l, p) for l in range(spec.n_layers) for p in positions]
    kv_close(batched[1], kv_ref, kvbits)
    ck.release(host)


# prompt-pass query groupings: kv_mul 1 (k_pf_attn KM = 1), 7 (KM = 1) and 8 (KM = 4, two passes) at head_dim 64 and 128
_PF = replace(mg.SPECS["pf-tiny"], name="pf-group", dim=512, hidden_dim=1024, max_seq_len=512)
GROUPINGS = {
    "kv1-hd64": replace(_PF, n_heads=2, n_kv_heads=2, head_dim=64),
    "kv7-hd64": replace(_PF, n_heads=14, n_kv_heads=2, head_dim=64),
    "kv8-hd64": replace(_PF, n_heads=16, n_kv_heads=2, head_dim=64),
    "kv1-hd128": replace(_PF, n_heads=2, n_kv_heads=2, head_dim=128, rope_theta=5e5),
    "kv7-hd128": replace(_PF, n_heads=7, n_kv_heads=1, head_dim=128, rope_theta=5e5),
    "kv8-hd128": replace(_PF, n_heads=8, n_kv_heads=1, head_dim=128, rope_theta=5e5),
    # Qwen2-0.5B widths (dim 896, hidden 4864, 14 query / 2 kv heads of 64, QKV bias, tied classifier, fp16) at two layers
    "qwen2-0.5b": replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=2, vocab_size=1024, max_seq_len=512),
}


def _prefill_vs_serial_and_oracle(oracle_pkg, spec, seed, toks, seq_len, pos0=0, warm=(), kvbits=16, label=""):
    host = mg.HostModel(spec, seed=seed, seq_len=seq_len, kvbits=kvbits)
    serial, batched = _both(spec, host.tensors, toks, pos0, seq_len, kvbits, warm=warm)  # asserts prefill() == 1
    _check(spec, serial, batched, kvbits, label)
    ref, ck = oracle_run(oracle_pkg, host, toks[-1:], pos0=pos0 + len(toks) - 1, warm=list(warm) + list(toks[:-1]))
    logits_close(batched[0], ref[0], TOL_SIGMA if kvbits == 16 else TOL8_SIGMA, label)
    n = len(toks) - 1
    positions = sorted({pos0, pos0 + n // 3, pos0 + n // 2, pos0 + n - 1})
    kv_close(batched[1], [ck.read_kv(host, l, p) for l in range(spec.n_layers) for p in positions], kvbits)
    ck.release(host)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(GROUPINGS))
def test_prefill_query_groupings_vs_serial_and_oracle(oracle_pkg, shape):
    spec = GROUPINGS[shape]
    toks = mg.teacher_tokens(spec.vocab_size, 151)
    _prefill_vs_serial_and_oracle(oracle_pkg, spec, 9, toks, SEQ_LEN, label=f"{shape}, n = 150")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2100])
def test_prefill_block_sizes_vs_serial_and_oracle(oracle_pkg, n):
    """One token; 2100 tokens = a 2048-token chunk and a second one starting at pos0 + 2048."""
    spec = mg.SPECS["pf-tiny"]
    toks = mg.teacher_tokens(spec.vocab_size, n + 1)
    _prefill_vs_serial_and_oracle(oracle_pkg, spec, 12, toks, 2304 if n > 512 else SEQ_LEN, label=f"pf-tiny, n = {n}")


@pytest.mark.gpu
def test_prefill_second_turn_regrows_its_buffers(oracle_pkg):
    """A chat's second turn: a 60-token prompt pass, three decode steps, then a 300-token pass at pos0 = 63 (its token tiles
    outgrow the first pass's buffers, which are freed and rebuilt with new tensor maps)."""
    spec = mg.SPECS["pf-tiny"]
    host = mg.HostModel(spec, seed=13, seq_len=SEQ_LEN)
    first = mg.teacher_tokens(spec.vocab_size, 63, start=300)
    toks = mg.teacher_tokens(spec.vocab_size, 301)
    ref, ck = oracle_run(oracle_pkg, host, first + toks)
    out = []
    for batched in (False, True):
        with lib.DeviceModel(spec, host.tensors, seq_len=SEQ_LEN) as dm:
            if batched:
                assert dm.prefill(first[:60], 0) == 1
            else:
                for i, t in enumerate(first[:60]):
                    dm.forward(t, i, FF_UPDATE_KV_ONLY)
            steps = [dm.forward(t, 60 + i) for i, t in enumerate(first[60:])]
            if batched:
                assert dm.prefill(toks[:-1], 63) == 1
            else:
                for i, t in enumerate(toks[:-1]):
                    dm.forward(t, 63 + i, FF_UPDATE_KV_ONLY)
            last = dm.forward(toks[-1], 363)
            kv = [dm.read_kv(l, p) for l in range(spec.n_layers) for p in (0, 59, 62, 63, 200, 362)]
        out.append((np.stack(steps), last, kv))
    (ss, ls, kvs), (sb, lb, kvb) = out
    for i in range(3):
        logits_close(sb[i], ref[60 + i], TOL_SIGMA, f"second turn: decode step {60 + i}")
    _check(spec, (ls, kvs), (lb, kvb), 16, "second turn: pos0 = 63, n = 300")
    logits_close(lb, ref[-1], TOL_SIGMA, "second turn: after the second pass")
    kv_close(kvb, [ck.read_kv(host, l, p) for l in range(spec.n_layers) for p in (0, 59, 62, 63, 200, 362)], 16)
    ck.release(host)


@pytest.mark.gpu
def test_prefill_up_to_seq_len_then_roll_over(oracle_pkg):
    """A block that ends exactly at seq_len (pos0 + n == seq_len) runs batched; the decode steps after it roll the cache
    over with re-rotated sinks.  A block that would cross seq_len is fed token by token: bit-identical to serial."""
    spec = mg.SPECS["pf-tiny"]
    seq_len = 256
    host = mg.HostModel(spec, seed=14, seq_len=seq_len)
    toks = mg.teacher_tokens(spec.vocab_size, seq_len + 6)
    ref, ck = oracle_run(oracle_pkg, host, toks)
    ck.release(host)
    with lib.DeviceModel(spec, host.tensors, seq_len=seq_len) as dm:
        assert dm.prefill(toks[:seq_len], 0) == 1
        got = np.stack([dm.forward(t, seq_len + i) for i, t in enumerate(toks[seq_len:])])
    with lib.DeviceModel(spec, host.tensors, seq_len=seq_len) as dm:
        for i, t in enumerate(toks[:seq_len]):
            dm.forward(t, i, FF_UPDATE_KV_ONLY)
        serial = np.stack([dm.forward(t, seq_len + i) for i, t in enumerate(toks[seq_len:])])
    # a rolled-over cache re-rounds its sinks every step: the rolling-cache rule of test_rolling_cache_with_sinks (4x)
    logits_close(got, ref[seq_len:], 4 * TOL_SIGMA, f"prompt pass to pos {seq_len}, then {len(toks) - seq_len} rolled-over steps")
    logits_close(got, serial, 4 * TOL_SIGMA, "  ... against serial")
    # pos0 + n > seq_len: no batched pass, the tokens go through the decode path one by one
    out = []
    for batched in (False, True):
        with lib.DeviceModel(spec, host.tensors, seq_len=seq_len) as dm:
            for i, t in enumerate(toks[:200]):
                dm.forward(t, i, FF_UPDATE_KV_ONLY)
            if batched:
                assert dm.prefill(toks[200:-1], 200) == 0
            else:
                for i, t in enumerate(toks[200:-1]):
                    dm.forward(t, 200 + i, FF_UPDATE_KV_ONLY)
            out.append((dm.forward(toks[-1], len(toks) - 1), [dm.read_kv(l, p) for l in range(spec.n_layers) for p in (0, 1, 5, 100, 255)]))
    np.testing.assert_array_equal(out[0][0], out[1][0])
    for (ka, va), (kb, vb) in zip(out[0][1], out[1][1]):
        np.testing.assert_array_equal(ka, kb)
        np.testing.assert_array_equal(va, vb)
    logits_close(out[1][0], ref[-1], 4 * TOL_SIGMA, "rolled-over block fed token by token")


# ---- the device-resident loops (k_advance, k_sample_pick) across the rollover
LOOP_SEQ_LEN, LOOP_START, LOOP_N = 32, 27, 12  # steps at pos 27 .. 38: kv_pos goes 27 .. 31, then 2, 3, ...


def _warm(dm, spec):
    for i, t in enumerate(mg.teacher_tokens(spec.vocab_size, LOOP_START)):
        dm.forward(t, i, FF_UPDATE_KV_ONLY)


@pytest.mark.gpu
def test_greedy_loop_across_the_rollover():
    spec = mg.SPECS["tiny-llama"]
    host = mg.HostModel(spec, seed=4)
    with lib.DeviceModel(spec, host.tensors, seq_len=LOOP_SEQ_LEN) as dm:
        _warm(dm, spec)
        tok, seq = 5, []
        for pos in range(LOOP_START, LOOP_START + LOOP_N):
            logits = dm.forward(tok, pos)
            tok = int(np.argmax(logits))
            seq.append(tok)
    with lib.DeviceModel(spec, host.tensors, seq_len=LOOP_SEQ_LEN) as dm:
        _warm(dm, spec)
        loop = list(dm.decode_greedy(5, LOOP_START, LOOP_N))
        dev = dm.device_logits()
    print(f"greedy across pos {LOOP_SEQ_LEN}: {seq}")
    assert loop == seq
    np.testing.assert_allclose(dev, logits, rtol=0, atol=1e-5 * float(logits.std()))


@pytest.mark.gpu
@pytest.mark.parametrize("temperature,minp", [(1.0, 0.1), (1.3, 0.02)])
def test_sampling_loop_across_the_rollover(temperature, minp):
    spec = mg.SPECS["tiny-llama"]
    host = mg.HostModel(spec, seed=6)
    with lib.DeviceModel(spec, host.tensors, seq_len=LOOP_SEQ_LEN) as dm:
        _warm(dm, spec)
        seq, rng, tok = [], 321, 5
        for pos in range(LOOP_START, LOOP_START + LOOP_N):
            o, rng = dm.decode_sample(tok, pos, 1, temperature, minp, rng)
            tok = int(o[0])
            seq.append(tok)
        stepped = dm.device_logits()
    with lib.DeviceModel(spec, host.tensors, seq_len=LOOP_SEQ_LEN) as dm:
        _warm(dm, spec)
        loop, rng_loop = dm.decode_sample(5, LOOP_START, LOOP_N, temperature, minp, 321)
        dev = dm.device_logits()
    print(f"sampling T {temperature} minp {minp} across pos {LOOP_SEQ_LEN}: {seq}")
    assert list(loop) == seq and rng_loop == rng
    np.testing.assert_allclose(dev, stepped, rtol=0, atol=1e-5 * float(stepped.std()))
