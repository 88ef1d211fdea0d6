"""The float64 stage references of tests/stage_ref.py, composed into whole tokens, against the double-precision build of
the CPU oracle: rotated queries, attention output and residual stream of every layer (oracle_forward_taps) and the logits,
for every model switch, both cache formats and a rolled-over cache.  The yardstick of tests/test_stages_gpu.py is proven
here, without a GPU."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_ref as sr  # noqa: E402

from calm_b200 import modelgen as mg  # noqa: E402

# the referee keeps its activations in fp32 between stages; three layers of that against float64 throughout
TOL = 2e-6
SEQ_LEN, N_TOKENS = 12, 16  # positions 12 .. 15 land in slots 2 .. 5 of a rolled-over cache, with re-rotated sinks

CASES = [(name, 16) for name in ("tiny-llama", "tiny-qwen", "tiny-gelu-clip", "tiny-ln", "tiny-lnpar", "tiny-moe", "tiny-moe-gf4", "tiny-gf4",
                                 "tiny-mha", "tiny-hd256", "tiny-fp16")] + [("tiny-llama", 8), ("tiny-qwen", 8), ("tiny-moe", 8)]


@pytest.mark.parametrize("name,kvbits", CASES)
def test_composed_stages_vs_f64_oracle(oracle_pkg, name, kvbits):
    spec = mg.SPECS[name]
    host = mg.HostModel(spec, seed=3, seq_len=SEQ_LEN, kvbits=kvbits)
    ck = oracle_pkg.Checker("port_f64")
    ck.prepare(host)
    w = sr.Weights(spec, host.tensors)
    cache = sr.Cache(spec, SEQ_LEN, kvbits)
    worst = {}
    for pos, tok in enumerate(mg.teacher_tokens(spec.vocab_size, N_TOKENS)):
        want = ck.forward_taps(host, tok, pos)
        slot = sr.kv_slot(pos, SEQ_LEN)[0]

        def adopt_entries(l):
            """The sinks and this token's slot: the referee's entry, or its neighbour where the referee's fp32 value sat on
            a tie (near zero, where the spacing is as fine as the referee's fp32 noise: that noise besides).  The referee's entries are then adopted, so the attention check is not charged for such a flip."""
            for p in {0, 1, slot}:
                for mine, ref in zip((cache.k[l, :, p], cache.v[l, :, p]), ck.read_kv(host, l, p)):
                    ref = ref.reshape(mine.shape)
                    d = np.abs(mine - ref)
                    assert (d <= sr.ulp(ref, kvbits) + TOL * np.abs(ref).max()).all() and (d == 0).mean() >= 0.98, (name, kvbits, pos, l, p)
                    mine[:] = ref

        got = sr.forward(w, cache, tok, pos, adopt_entries)
        for what, a, b in zip(("logits", "q", "att", "x"), got, want):
            err = float(np.abs(a - b).max() / np.abs(b).max())
            worst[what] = max(worst.get(what, 0.0), err)
            assert err <= TOL, (name, kvbits, pos, what, err)
    ck.release(host)
    print(f"{name} kv{kvbits}: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


def test_cache_rounding_is_nearest_even():
    """round_kv against torch's casts over normals, subnormals, ties and the e5m2 saturation."""
    import torch

    rng = np.random.default_rng(0)
    v = np.concatenate([rng.standard_normal(20000) * 10.0 ** rng.integers(-7, 4, 20000), [0.0, 1.25, 1.75, 2.5, 3.5, 6e-8, 2.3e-5, 1e-7]])
    t = torch.from_numpy(v.astype(np.float32))
    v = t.numpy().astype(np.float64)
    np.testing.assert_array_equal(sr.round_kv(v, 16), t.to(torch.float16).double().numpy())
    np.testing.assert_array_equal(sr.round_kv(v, 8), t.to(torch.float8_e5m2).double().numpy())
    assert sr.round_kv(np.array([6e4, -1e9]), 8).tolist() == [57344.0, -57344.0]
