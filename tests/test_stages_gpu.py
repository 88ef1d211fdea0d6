"""Every decode and prompt-pass stage, element by element, against a float64 reference computed from that stage's own inputs.

The other GPU tests compare logits at 5e-3 sigma after a whole model has diluted whatever one kernel did.  Here the model
has ONE layer, so after a token (or a prompt pass) every stage's output is still in the engine's buffers;
calm_b200_read_state hands them over, and each stage is checked against tests/stage_ref.py fed with the DEVICE's output of
the stage before it: k_qkv from the exact embedding row, the attention from the device's q and the device's cache, the
FFN from the device's attention output, w2 from the device's hidden vector, the classifier from the device's x.  A cache
entry on the other side of a rounding boundary therefore costs nothing, and what is left is the arithmetic of one kernel.
The production plan and graph run unchanged; every case asserts the kernels prepare_cuda planned for it.

Errors are normalised by the stage's own scale (max |reference| of the vector, per kv head for the attention) and printed
per case and stage.  STAGE_TOL holds the bounds, with the arithmetic behind each and the largest error measured beside it.
A failure names the stage, its kernel and the worst element's coordinates."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402
from test_scale_gpu import ROLLED, rolled_position  # noqa: E402
from test_variants_gpu import GROUPINGS, RING, VARIANTS, plan_of  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

# Bounds on |device - float64| / scale; u = 2^-24 is half an fp32 ulp.  Beside each bound: the largest error over every
# case of this file on an H100 80GB HBM3 (700 W limit, 132 SMs).  No bound is more than 10x its measurement.
STAGE_TOL = {
    # k_qkv: fp32 sums of dim products, split over 32 lanes x 4 vectors and folded as a tree, so the error is a few u of the
    # partial sums' size rather than dim u; an fp32 norm scale; sincosf on the shared fp32 angle.  Measured 8.0e-7.
    "q": 3e-6,
    # K / V entries: half a spacing of the cache format around the float64 value, plus this much of max |row| for the fp32
    # sum that is rounded.  Measured 2.2e-7 beyond half a spacing.
    "kv": 1e-6,
    # re-rotated sinks: an fp32 rotation of two cache values, rounded again.  No entry was ever off by more than half a
    # spacing (measured 0), so the bound is the rotation's few u and cannot be tied to a measurement.
    "sink": 1e-6,
    # k_attn2: q and p as f16 hi + lo pairs (2^-22 each) into fp32 mma accumulators over kv_len positions, expf on fp32
    # scores, a slice fold in fp32.  k_attn: all fp32.  Of max |V| of the kv head over the attended slots.  Measured 4.0e-7.
    "att": 2e-6,
    # k_ffn_up(_ring): two fp32 sums of dim products, expf / tanhf, one product.  Its input is x1 = x0 + Wo att in float64
    # while the device read its own fp32 x1, so wo's fp32 sum of q_dim products (K-sliced in k_matres_ring) is charged here
    # too: a wrong wo row moves every hidden row.  Measured 9.3e-7.
    "hb": 4e-6,
    "moe_w": 4e-6,  # router weights: fp32 sums of dim products, expf, one division; absolute.  Measured 9.8e-7.
    # w2 through k_matres(_ring): fp32 sums of hidden products in up to 32 K-slices folded in shared memory, added to x.
    "x": 2e-6,  # measured 4.8e-7
    "xb": 5e-7,  # parallel norm: the saved attention-norm output (fp32 mean, variance, scale).  Measured 9.4e-8.
    "logits": 2e-6,  # k_output: fp32 norm and sums of dim products.  Measured 5.2e-7.
    "pf_att": 3e-6,  # k_pf_attn: fp32 throughout, online softmax per warp.  Measured 7.1e-7.
}


def pf_tol(K):
    """Bound for an output of the prompt pass's wgmma GEMMs over K products.  The inputs are good to 22 bits (activations as
    f16 hi + lo, weights exact in f16), yet the measured error grows in proportion to K, about 2.5e-9 K of scale (1.2e-6 at
    K = 512, 1.3e-5 at 4096, 3.6e-5 at 14336): the tensor core adds into its fp32 accumulator with truncation, which biases a
    long sum instead of averaging out.  The bound follows that law with a factor of 6 and the floor of the short sums."""
    return 2e-6 + 1.5e-8 * K


REG = {"up": "k_ffn_up", "wo": "k_matres", "down": "k_matres"}
worst_seen = {}


def note(key, e, tol):
    if e / tol >= worst_seen.get(key, (0.0, 1.0, -1.0))[2]:
        worst_seen[key] = (e, tol, e / tol)


def report(label, stage, kernel, got, want, scale, coords, key=None, tol=None):
    """Assert |got - want| / scale <= the stage's bound over the whole array; name the worst element on failure."""
    err = np.abs(np.asarray(got, np.float64) - want) / scale
    i = np.unravel_index(int(np.argmax(err)), err.shape)
    e, tol = float(err[i]), tol or STAGE_TOL[key or stage]
    note(key or stage, e, tol)
    print(f"  {label}: {stage:7s} {kernel:14s} max err {e:.2e} of scale (tol {tol:.0e}) at {coords(i)}")
    assert np.isfinite(err).all() and e <= tol, f"{label}: stage {stage} ({kernel}): device {np.asarray(got)[i]!r} vs float64 {want[i]!r} at {coords(i)}: {e:.2e} of scale > {tol:.0e}"


def check_entries(label, stage, kernel, got, want, kvbits, coords, key="kv", tol=None):
    """Cache entries must be a correct rounding of the float64 value: within half a spacing, plus the fp32 sum's slack."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    excess = (np.abs(got - want) - 0.5 * sr.ulp(want, kvbits)) / np.abs(want).max()
    i = np.unravel_index(int(np.argmax(excess)), excess.shape)
    e, tol = float(excess[i]), tol or STAGE_TOL[key]
    note(key, max(e, 0.0), tol)
    print(f"  {label}: {stage:7s} {kernel:14s} beyond half a spacing by {max(e, 0):.2e} of max |row| (tol {tol:.0e}) at {coords(i)}")
    assert np.isfinite(got).all() and e <= tol, f"{label}: stage {stage} ({kernel}): entry {got[i]!r} is not a rounding of {want[i]!r} at {coords(i)}: off by {e:.2e} of max |row| beyond half a spacing"


def make_model(spec, seed):
    """Weights generated on the device (the 70B-width layer is 0.9 GB), and the float64 reference's view of the same bytes."""
    tensors = mg.generate(spec, seed, device="cuda")
    torch.cuda.synchronize()
    return tensors, sr.Weights(spec, {k: v.cpu() for k, v in tensors.items()})


def layer_cache(dm, spec, layer=0):
    shape = (spec.n_kv_heads, dm.seq_len, spec.head_dim)
    return dm.read_state("keys", layer).reshape(shape), dm.read_state("values", layer).reshape(shape)


def check_decode_step(dm, w, token, pos, kvbits, plan, label, fill_seed=5, layer=0):
    """fill_kv below `pos`, one forward_cuda, then every stage against float64 on the device's own inputs.  The stages are
    those of `layer`, whose input must be the embedding row: layer 0, or a later one behind layers that pass it through."""
    s = w.spec
    attn_kernel, _, mv = plan
    slot, kv_len, sinks = sr.kv_slot(pos, dm.seq_len)
    dm.fill_kv(min(pos, dm.seq_len), seed=fill_seed)
    keys_before = dm.read_state("keys", layer).reshape(s.n_kv_heads, dm.seq_len, s.head_dim)[:, :sr.KV_SINKS].copy() if sinks else None
    logits = dm.forward(token, pos)
    q, att, x = dm.read_state("q"), dm.read_state("att"), dm.read_state("x")
    hb = dm.read_state("hb").reshape(-1, s.hidden_dim)
    keys, values = layer_cache(dm, s, layer)
    hd, kv_mul = s.head_dim, s.n_heads // s.n_kv_heads
    label = f"{label} pos {pos} slot {slot}"

    x0 = sr.embed(w, token)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, layer, x0, pos)
    head_dim_of = lambda i: f"head {i[0] // hd} dim {i[0] % hd}"  # noqa: E731
    report(label, "q", "k_qkv", q, q_ref, np.abs(q_ref).max(), head_dim_of)
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        check_entries(label, name, "k_qkv", dev[:, slot].reshape(-1), ref, kvbits, lambda i: f"kv head {i[0] // hd} dim {i[0] % hd} slot {slot}")
    if sinks:
        check_entries(label, "sinks", "k_embed", keys[:, :sinks], sr.rotate_sinks(s, keys_before), kvbits, lambda i: f"kv head {i[0]} sink {i[1]} dim {i[2]}", "sink")
    if s.norm_type == "layernorm_par":
        report(label, "xb", "k_qkv", dm.read_state("xb"), xn, np.abs(xn).max(), lambda i: f"row {i[0]}")

    att_ref = sr.attention(s, q, keys, values, kv_len)
    vmax = np.repeat(np.abs(values[:, :kv_len]).max((1, 2)), kv_mul * hd)
    report(label, "att", attn_kernel, att, att_ref, vmax, lambda i: f"head {i[0] // hd} dim {i[0] % hd}, kv_len {kv_len}")

    x1 = sr.wo(w, layer, x0, att)
    xn2 = sr.ffn_input(w, layer, x1, xn)
    if s.n_experts:
        experts, weights, glog = sr.router(w, layer, xn2)
        sel = dm.read_state("moe_sel")
        dev_experts, dev_weights = [int(e) for e in sel[:len(experts)]], sel[len(experts):]
        srt = np.sort(glog)[::-1]
        if min(srt[i] - srt[i + 1] for i in range(len(experts))) > 1e-4 * np.abs(glog).max():  # a clear top-k
            assert dev_experts == experts, f"{label}: stage router ({mv['up']}): experts {dev_experts} vs float64 {experts} (logits {glog})"
        experts = dev_experts  # the hidden rows below belong to the device's choice
        e = np.exp(glog[experts] - glog.max())
        weights = e / e.sum()
        report(label, "moe_w", mv["up"], dev_weights, weights, 1.0, lambda i: f"active expert {i[0]} (expert {experts[i[0]]})")
        hb_ref = np.stack([sr.ffn_up(w, layer, xn2, e) for e in experts])
        x_ref = sr.ffn_down(w, layer, x1, hb, experts, dev_weights)
    else:
        hb_ref = sr.ffn_up(w, layer, xn2)[None]
        x_ref = sr.ffn_down(w, layer, x1, hb[0])
    report(label, "hb", mv["up"] + "+wo", hb, hb_ref, np.abs(hb_ref).max(), lambda i: f"expert slot {i[0]} hidden row {i[1]} (wo: {mv['wo']}, weight rows of {s.q_dim * s.dbits // 8} bytes)")
    report(label, "x", mv["down"], x, x_ref, np.abs(x_ref).max(), lambda i: f"row {i[0]} (weight rows of {s.hidden_dim * s.dbits // 8} bytes, sliced by 1 KB / 2 KB chunk)")
    logits_ref = sr.classifier(w, x)
    report(label, "logits", "k_output", logits, logits_ref, np.abs(logits_ref).max(), lambda i: f"vocabulary row {i[0]}")


def run_decode(spec, seed, seq_len, kvbits, steps, attn_kernel, matvec, capfd, monkeypatch, label, model=None):
    monkeypatch.delenv("CALM_B200_QUIET", raising=False)
    tensors, w = model or make_model(spec, seed)
    with lib.DeviceModel(spec, tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        plan = plan_of(capfd)
        assert (plan[0], plan[2]) == (attn_kernel, matvec), (label, plan)
        with capfd.disabled():
            for token, p in steps:
                check_decode_step(dm, w, token, rolled_position(p, seq_len, plan[1]), kvbits, plan, f"{label} kv{kvbits}")
    return tensors, w


# ---- decode cases: (spec, seq_len, [(token, position)], attention kernel, matvec kernels)
V4K = 4096
L8B = replace(mg.SPECS["llama3-8b-fp8"], n_layers=1, vocab_size=V4K)
_RING = replace(mg.SPECS["pf-tiny-hd128"], name="ring", dim=2048, hidden_dim=4096, n_heads=8, n_kv_heads=2, n_layers=1, vocab_size=V4K)
_HD64 = replace(_RING, head_dim=64, n_kv_heads=4, rope_theta=1e4, qkv_bias=False)
DECODE = {
    # 1 KB chunks for w2 (7168-byte rows), the staged group sums of gf4
    "mistral-gf4": (replace(mg.SPECS["mistral-7b-gf4"], n_layers=1, vocab_size=V4K), 4096, [(17, 0), (9, 1000), (3, 4095)], "k_attn2", RING),
    "fp16-2048": (replace(_RING, dtype="fp16"), 512, [(17, 0), (9, 77), (3, 511), (5, ("kv", 16))], "k_attn2", RING),
    # dim 8192, hidden 28672, 64 / 8 heads: w2's 112 KB activation vector takes plan_res to 1 KB chunks; k_attn2<8, 128>
    "llama3-70b": (replace(mg.SPECS["llama3-70b-fp8"], n_layers=1, vocab_size=V4K), 4096, [(17, 0), (9, 2500), (3, 4095)], "k_attn2", RING),
    "hd64-kvmul2": (replace(_HD64, n_heads=8), 512, [(17, 0), (9, 100), (3, 511), (5, ("kv", 2))], "k_attn2", dict(RING, wo="k_matres")),  # wo rows of 512 bytes
    "hd64-kvmul4": (replace(_HD64, n_heads=16), 512, [(17, 0), (9, 100), (3, 511)], "k_attn2", RING),
    "hd64-kvmul8": (replace(_HD64, n_heads=32), 512, [(17, 0), (9, 100), (3, 511)], "k_attn2", RING),
    # k_attn: a 256-wide multi-query head; 7 and 3 query heads per kv head (wo rows of 896 / 768 bytes: k_matres)
    "hd256-mq": (replace(mg.SPECS["tiny-hd256"], n_layers=1, vocab_size=V4K), 4096, [(17, 0), (9, 1001), (3, 4095)], "k_attn", RING),
    "kvmul7": (replace(_RING, n_heads=7, n_kv_heads=1), 512, [(17, 0), (9, 300), (5, ("kv", 15))], "k_attn", dict(RING, wo="k_matres")),
    "kvmul3": (replace(_RING, n_heads=6, n_kv_heads=2), 512, [(17, 0), (9, 300)], "k_attn", dict(RING, wo="k_matres")),
    # the transposing score path of k_attn (slices too long for k_attn2), kv_len 5001 = 312 blocks of 16 and 9 positions
    "attn-l8-16k": (replace(mg.SPECS["attn-l8"], n_layers=1), 16384, [(17, 5000), (9, 16383)], "k_attn", dict(REG, wo="k_matres_ring")),
    # the register-fed matvecs at a real width: Qwen2-0.5B (dim 896, hidden 4864, 14 / 2 heads of 64, qkv bias, tied, fp16)
    "qwen2-0.5b": (replace(mg.SPECS["qwen2-0.5b-fp16"], n_layers=1, vocab_size=V4K), 512, [(17, 0), (9, 200), (3, 511)], "k_attn", REG),
    "tiny-moe-gf4": (replace(mg.SPECS["tiny-moe-gf4"], n_layers=1), 64, [(17, 0), (9, 40), (300, 63)], "k_attn", REG),
    # Mixtral widths: two tokens, two expert pairs
    "mixtral": (replace(mg.SPECS["mixtral-8x7b-fp8"], n_layers=1, vocab_size=V4K), 4096, [(17, 0), (9, 1000), (1234, 4095)], "k_attn2", REG),
    # a residual stream of 16384 rows: 63 row pairs per k_matres_ring CTA on 132 SMs, more than its shared-memory fold holds,
    # so w2 runs both 2 KB chunks of a row in one task (S = cpt)
    "wide-16384": (replace(_RING, dim=16384, hidden_dim=4096), 512, [(17, 0), (9, 300)], "k_attn2", RING),
}
DECODE.update({"switch-" + k: (replace(v[0], n_layers=1, vocab_size=V4K), 512, [(17, 0), (9, 200), (5, ("kv", 16))], "k_attn2", RING) for k, v in VARIANTS.items()})


@pytest.mark.parametrize("kvbits", [16, 8])
def test_llama3_8b_widths_every_stage(kvbits, capfd, monkeypatch):
    """k_qkv, k_attn2<4, 128>, the ring kernels with 2 KB chunks (w2 in 7 K-slices): the edges of the attention's slices
    (positions 0, 15, 16, 17, 255: most slices own no block, or a partial one), a partial last bulk copy at seq_len 4009,
    the last slot, and the rolled-over cache with its re-rotated sinks."""
    model = run_decode(L8B, 1, 4096, kvbits, [(17, 0), (9, 15), (3, 16), (5, 17), (7, 255), (11, 4095)] + [(13, r) for r in ROLLED],
                       "k_attn2", RING, capfd, monkeypatch, "llama3-8b")
    run_decode(L8B, 1, 4009, kvbits, [(17, 4008), (9, ("kv", 2)), (3, ("kv", "last-slice")), (5, ("kv", -1))], "k_attn2", RING, capfd, monkeypatch,
               "llama3-8b seq_len 4009", model=model)


def test_classifier_at_the_real_vocabulary(capfd, monkeypatch):
    """k_output over Llama-3's 128256 rows."""
    run_decode(replace(L8B, vocab_size=128256), 2, 4096, 16, [(100000, 0), (9, 3000)], "k_attn2", RING, capfd, monkeypatch, "llama3-8b vocab 128256")


@pytest.mark.parametrize("case", sorted(DECODE))
def test_decode_every_stage(case, capfd, monkeypatch):
    spec, seq_len, steps, attn_kernel, matvec = DECODE[case]
    kvbits = 8 if case in ("mistral-gf4", "hd64-kvmul4", "kvmul3", "switch-layernorm") else 16
    run_decode(spec, 3, seq_len, kvbits, steps, attn_kernel, matvec, capfd, monkeypatch, case)


# ---- the prompt pass: (spec, kvbits, n, pos0)
PREFILL = {
    "llama3-8b n300": (L8B, 16, 300, 0),
    "mistral-gf4 n200": (DECODE["mistral-gf4"][0], 8, 200, 0),
    "pf-tiny-fp16 n129": (replace(mg.SPECS["pf-tiny"], n_layers=1, dtype="fp16"), 16, 129, 0),
    "pf-tiny-hd128 pos0 37": (replace(mg.SPECS["pf-tiny-hd128"], n_layers=1), 16, 150, 37),  # a warm cache, qkv bias
    "switch-gelu-clip-rot64 n150": (DECODE["switch-gelu-clip-rot64"][0], 16, 150, 0),
    "switch-layernorm-par n150": (DECODE["switch-layernorm-par"][0], 8, 150, 0),
}
PREFILL.update({k + " n150": (replace(GROUPINGS[k], n_layers=1), 16, 150, 0) for k in ("kv1-hd64", "kv7-hd64", "kv1-hd128", "kv7-hd128")})


@pytest.mark.parametrize("case", sorted(PREFILL))
def test_prefill_every_stage(case, capfd):
    """forward_prefill_cuda's n rows of Q, attention output, hidden and residual, and the cache entries of every position of
    the block, each from the device's own previous stage (PF_QKV, k_pf_attn, PF_WO + PF_UP, PF_DOWN of k_pf_gemm)."""
    spec, kvbits, n, pos0 = PREFILL[case]
    tensors, w = make_model(spec, 4)
    toks = mg.teacher_tokens(spec.vocab_size, n)
    hd, kv_mul = spec.head_dim, spec.n_heads // spec.n_kv_heads
    with lib.DeviceModel(spec, tensors, seq_len=512, kvbits=kvbits) as dm, capfd.disabled():
        dm.fill_kv(pos0, seed=6)
        assert dm.prefill(toks, pos0) == 1
        X = dm.read_state("pf_x").reshape(-1, spec.dim)[:n]
        Q = dm.read_state("pf_q").reshape(-1, spec.q_dim)[:n]
        A = dm.read_state("pf_att").reshape(-1, spec.q_dim)[:n]
        H = dm.read_state("pf_hb").reshape(-1, spec.hidden_dim)[:n]
        keys, values = layer_cache(dm, spec)
    label = f"prompt pass {case} kv{kvbits}"
    X0 = w.mat("model.embed.weight")[toks].astype(np.float64)
    q_ref, k_ref, v_ref, xn = sr.qkv(w, 0, X0, pos0 + np.arange(n))
    report(label, "Q", "k_pf_gemm QKV", Q, q_ref, np.abs(q_ref).max(), lambda i: f"token row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_q", pf_tol(spec.dim))
    for name, dev, ref in (("K", keys, k_ref), ("V", values, v_ref)):
        got = dev[:, pos0:pos0 + n].transpose(1, 0, 2).reshape(n, -1)
        check_entries(label, name, "k_pf_gemm QKV", got, ref, kvbits, lambda i: f"token row {i[0]} kv head {i[1] // hd} dim {i[1] % hd}", "pf_kv", pf_tol(spec.dim))
    a_ref = np.stack([sr.attention(spec, Q[t], keys, values, pos0 + t + 1) for t in range(n)])
    vmax = np.repeat(np.maximum.accumulate(np.abs(values[:, :pos0 + n]).max(2), 1)[:, pos0:].T, kv_mul * hd, 1)  # [n, q_dim]: max |V| of the head so far
    report(label, "A", "k_pf_attn", A, a_ref, vmax, lambda i: f"token row {i[0]} head {i[1] // hd} dim {i[1] % hd}", "pf_att")
    x1 = sr.wo(w, 0, X0, A)
    h_ref = sr.ffn_up(w, 0, sr.ffn_input(w, 0, x1, xn))
    report(label, "H", "k_pf_gemm WO+UP", H, h_ref, np.abs(h_ref).max(), lambda i: f"token row {i[0]} hidden row {i[1]}", "pf_hb", pf_tol(max(spec.dim, spec.q_dim)))
    x_ref = sr.ffn_down(w, 0, x1, H)
    report(label, "X", "k_pf_gemm DOWN", X, x_ref, np.abs(x_ref).max(), lambda i: f"token row {i[0]} row {i[1]}", "pf_x", pf_tol(spec.hidden_dim))


def test_zz_summary_of_largest_errors():
    """Runs last in this file: one line with the largest error each stage showed in this session, beside its bound."""
    if not worst_seen:
        pytest.skip("the stage tests did not run in this session")
    print("\n  largest share of its bound per stage: " + ", ".join(f"{k} {e:.2e} of {tol:.1e}" for k, (e, tol, _) in sorted(worst_seen.items())))
    assert all(e <= tol for e, tol, _ in worst_seen.values())
