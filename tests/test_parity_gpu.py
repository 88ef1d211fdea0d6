"""GPU parity tests: the CUDA path, called through the C ABI exactly as the reference driver calls its
backend (upload_cuda -> prepare_cuda -> forward_cuda per token), against
  (1) the CPU oracle (oracle/calm_oracle.c) on the same seeded model,
  (2) the committed golden fixtures produced by the unmodified reference, and
  (3) logits of the unmodified reference on further seeds and positions (tests/golden/reference-cpu.npz).
Tolerance (stated, DESIGN.md): |dlogit| <= 5e-3 * std(logits); argmax identical on every step whose
reference top-2 margin exceeds twice that; KV entries within fp16 rounding."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import KV_ATOL, KV_RTOL, ROOT, TOL_SIGMA, golden  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden import GOLDEN_SPECS, model_digest  # noqa: E402

pytestmark = pytest.mark.gpu


def run_device(spec, seed, tokens, pos0=0, seq_len=None, kvbits=16):
    host = mg.HostModel(spec, seed=seed, seq_len=seq_len)
    with lib.DeviceModel(spec, host.tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        logits = np.stack([dm.forward(t, pos0 + i) for i, t in enumerate(tokens)])
    return logits


@pytest.mark.parametrize("name", GOLDEN_SPECS)
def test_logits_match_golden_and_oracle(oracle_pkg, name):
    g = golden(name)
    spec = mg.SPECS[name]
    host = mg.HostModel(spec, seed=0)
    assert model_digest(host) == str(g["sha256"])
    toks = [int(t) for t in g["tokens"]]
    ck = oracle_pkg.Checker("port")
    ref = oracle_pkg.teacher_forced(ck, host, toks)
    with lib.DeviceModel(spec, host.tensors) as dm:
        got = np.stack([dm.forward(t, i) for i, t in enumerate(toks)])
        sigma = float(ref.std())
        tol = TOL_SIGMA * sigma
        err_oracle = np.abs(got - ref).max()
        err_golden = np.abs(got[g["steps"]] - g["logits"]).max()
        print(f"{name}: sigma {sigma:.3f} |cuda-oracle| {err_oracle:.2e} |cuda-golden(reference)| {err_golden:.2e} tol {tol:.2e}")
        assert err_oracle <= tol
        assert err_golden <= tol
        safe = g["margin"] > 2 * tol
        assert (got.argmax(1)[safe] == g["argmax"][safe]).all()
        assert safe.sum() >= len(toks) // 2
        for l in range(spec.n_layers):
            for i, p in enumerate(g["kvpos"]):
                k, v = dm.read_kv(l, int(p))
                np.testing.assert_allclose(k, g["k"][l, i], rtol=KV_RTOL, atol=KV_ATOL)
                np.testing.assert_allclose(v, g["v"][l, i], rtol=KV_RTOL, atol=KV_ATOL)
    ck.release(host)


def test_against_live_reference(oracle_pkg):
    """The unmodified reference CPU backend (logits stored from a run of it by tools/make_reference_golden.py), different
    seed / positions."""
    for name in ("tiny-llama", "tiny-moe", "tiny-gf4"):
        spec = mg.SPECS[name]
        toks = mg.teacher_tokens(spec.vocab_size, 20, start=50)
        ref = golden("reference-cpu")["parity-" + name]
        got = run_device(spec, 5, toks)
        tol = TOL_SIGMA * ref.std()
        assert np.abs(got - ref).max() <= tol, name


def test_kv_only_flag_and_prompt_pipeline(oracle_pkg):
    """FF_UPDATE_KV_ONLY returns NULL, still advances the cache (reference infer.cu:724-727), and a
    prompt fed that way gives the same final logits as feeding it with logits requested."""
    spec = mg.SPECS["tiny-fp8"]
    toks = mg.teacher_tokens(spec.vocab_size, 16)
    host = mg.HostModel(spec, seed=2)
    full = run_device(spec, 2, toks)
    with lib.DeviceModel(spec, host.tensors) as dm:
        for i, t in enumerate(toks[:-1]):
            assert dm.forward(t, i, FF_UPDATE_KV_ONLY) is None
        last = dm.forward(toks[-1], len(toks) - 1)
    np.testing.assert_array_equal(last, full[-1])  # same kernels, same order: bit-identical


def test_rolling_cache_with_sinks(oracle_pkg):
    """pos >= seq_len: ring buffer with 2 pinned, re-rotated sinks (reference infer.c:330-332, 384-394)."""
    spec = mg.SPECS["tiny-fp8"]
    toks = mg.teacher_tokens(spec.vocab_size, 40)
    host = mg.HostModel(spec, seed=1, seq_len=16)
    ref = oracle_pkg.teacher_forced(oracle_pkg.Checker("port"), host, toks)
    got = run_device(spec, 1, toks, seq_len=16)
    # the sinks are re-rounded to fp16 every step, which compounds; allow 4x the base tolerance
    assert np.abs(got - ref).max() <= 4 * TOL_SIGMA * ref.std()


def test_device_argmax_and_greedy_loop(oracle_pkg):
    """Device-side greedy pick == host argmax with the reference tie rule (sampler.c:34-42), and the
    device-resident decode loop reproduces the host-stepped loop token for token."""
    spec = mg.SPECS["tiny-llama"]
    host = mg.HostModel(spec, seed=4)
    with lib.DeviceModel(spec, host.tensors) as dm:
        tok, seq = 5, []
        for pos in range(20):
            logits = dm.forward(tok, pos)
            tok = int(np.argmax(logits))  # numpy argmax: first maximum
            seq.append(tok)
    with lib.DeviceModel(spec, host.tensors) as dm:
        tok, seq2 = 5, []
        for pos in range(20):
            tok = dm.forward_argmax(tok, pos)
            seq2.append(tok)
    with lib.DeviceModel(spec, host.tensors) as dm:
        seq3 = list(dm.decode_greedy(5, 0, 20))
    assert seq == seq2 == seq3


@pytest.mark.parametrize("dbits,n,d", [(8, 4096, 512), (16, 896, 130), (4, 4096, 96), (8, 14336, 64), (16, 4096, 33), (4, 1792, 40), (8, 32, 8)])
def test_matvec_kernel_vs_oracle(oracle_pkg, dbits, n, d):
    """The matvec kernel alone against reference infer.c:209-221 (via the oracle), ragged row counts and
    row lengths that are not a multiple of the 512-byte warp stride."""
    dtype = {16: "fp16", 8: "fp8", 4: "gf4"}[dbits]
    g = torch.Generator().manual_seed(dbits * 1000 + n + d)
    w = mg.quantize(0.02 * torch.randn(d, n, generator=g), dtype).contiguous()
    x = torch.randn(n, generator=g).numpy()
    L = lib.load()
    dev = L.upload_cuda(w.data_ptr(), w.numel() * w.element_size())
    y, _ = lib.matvec(dbits, dev, x, n, d)
    L.calm_b200_free(dev)
    wn = w.numpy() if dbits != 16 else w.view(torch.int16).numpy()
    ref = oracle_pkg.Checker("port").matvec(dbits, wn, x, n, d)
    ref64 = oracle_pkg.Checker("port_f64").matvec(dbits, wn, x, n, d)
    scale = np.abs(ref64).max() + 1e-6
    assert np.abs(y - ref64).max() <= 2e-5 * scale * np.sqrt(n / 32)
    assert np.abs(y - ref).max() <= 4e-5 * scale * np.sqrt(n / 32)


def test_full_size_matvec_properties(oracle_pkg):
    """BASELINE-sized matrix (Llama-3-8B w1: 14336 x 4096 fp8): size-independent properties --
    linearity in x, a row subset against the oracle, and zero input -> exact zeros."""
    n, d = 4096, 14336
    g = torch.Generator(device="cuda").manual_seed(0)
    w = (0.02 * torch.randn(d, n, generator=g, device="cuda")).to(torch.float8_e5m2).view(torch.uint8)
    x1 = np.random.default_rng(0).standard_normal(n).astype(np.float32)
    x2 = np.random.default_rng(1).standard_normal(n).astype(np.float32)
    y1, _ = lib.matvec(8, w.data_ptr(), x1, n, d)
    y2, _ = lib.matvec(8, w.data_ptr(), x2, n, d)
    y12, _ = lib.matvec(8, w.data_ptr(), x1 + x2, n, d)
    y0, _ = lib.matvec(8, w.data_ptr(), np.zeros(n, np.float32), n, d)
    assert (y0 == 0).all()
    assert np.abs(y12 - (y1 + y2)).max() <= 1e-4 * np.abs(y12).max()
    rows = np.r_[0:8, 7000:7008, d - 8:d]
    wsub = w[torch.from_numpy(rows).cuda()].cpu().numpy()
    ref = oracle_pkg.Checker("port_f64").matvec(8, wsub, x1, n, len(rows))
    assert np.abs(y1[rows] - ref).max() <= 1e-4 * np.abs(ref).max()


def test_full_size_layer_count_independent_shapes(oracle_pkg):
    """Llama-3-8B widths (dim 4096, hidden 14336, 32/8 heads of 128, vocab 128256) with 2 layers: the
    real row lengths / head shapes at a depth the oracle finishes in seconds."""
    spec = mg.SPECS["llama3-8b-fp8"]
    from dataclasses import replace

    spec = replace(spec, name="llama3-8b-2l", n_layers=2, max_seq_len=256)
    toks = mg.teacher_tokens(spec.vocab_size, 6)
    host = mg.HostModel(spec, seed=0)
    ref = oracle_pkg.teacher_forced(oracle_pkg.Checker("port"), host, toks)
    with lib.DeviceModel(spec, host.tensors) as dm:
        got = np.stack([dm.forward(t, i) for i, t in enumerate(toks)])
    tol = TOL_SIGMA * ref.std()
    print(f"llama3-8b widths, 2 layers: |cuda-oracle| {np.abs(got - ref).max():.2e} tol {tol:.2e}")
    assert np.abs(got - ref).max() <= tol
    srt = np.sort(ref, 1)
    safe = (srt[:, -1] - srt[:, -2]) > 2 * tol
    assert (got.argmax(1)[safe] == ref.argmax(1)[safe]).all()


def test_long_context_is_idempotent():
    """Attention over a long, synthetic cache: the same token at the same position twice gives bit-identical logits
    (the cache slot is rewritten identically and the split over CTAs is deterministic).  The VALUES at long context are
    checked against the oracle in tests/test_scale_gpu.py."""
    spec = mg.SPECS["tiny-llama"]
    host = mg.HostModel(spec, seed=7, seq_len=2048)
    with lib.DeviceModel(spec, host.tensors, seq_len=2048) as dm:
        dm.fill_kv(2000, seed=3)
        a = dm.forward(3, 2000)
        b = dm.forward(3, 2000)
        np.testing.assert_array_equal(a, b)
        assert np.isfinite(a).all()
