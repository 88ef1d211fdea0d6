"""The tensor-core decode attention (k_attn2) at long context for the query-head groupings and head widths the headline
model does not use: 8 query heads per kv head at head_dim 128, and 4 or 8 at head_dim 64.  Device vs the CPU oracle on
identical cache contents (fp16 and e5m2), at context lengths that end inside a 16-position block."""
import os
import sys
from dataclasses import replace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import TOL_SIGMA  # noqa: E402
from test_scale_gpu import TOL8_SIGMA, fill_oracle_cache  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402

pytestmark = pytest.mark.gpu

_BASE = mg.SPECS["attn-l8"]
SHAPES = {
    "hg8-hd128": replace(_BASE, name="attn-hg8-hd128", n_heads=16, n_kv_heads=2, head_dim=128),  # 2 units x 36 slices
    "hg4-hd64": replace(_BASE, name="attn-hg4-hd64", n_heads=32, n_kv_heads=8, head_dim=64),
    "hg8-hd64": replace(_BASE, name="attn-hg8-hd64", n_heads=32, n_kv_heads=4, head_dim=64),
}


@pytest.mark.parametrize("kvbits", [16, 8])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_attn2_shapes_vs_oracle(oracle_pkg, shape, kvbits):
    spec = SHAPES[shape]
    seq_len = 4096
    host = mg.HostModel(spec, seed=13, seq_len=seq_len, kvbits=kvbits)
    ck = oracle_pkg.Checker("port")
    tol = TOL_SIGMA if kvbits == 16 else TOL8_SIGMA
    with lib.DeviceModel(spec, host.tensors, seq_len=seq_len, kvbits=kvbits) as dm:
        # kv_len = pos + 1: none a multiple of 16; pos 5094 is past seq_len (a rolled-over cache, this token in slot 1000)
        for pos in (40, 1000, 2900, 4094, 5094):
            ck.prepare(host)
            fill_oracle_cache(host, min(pos, seq_len), seed=7, kvbits=kvbits)
            want = ck.forward(host, 19, pos)
            ck.release(host)
            dm.fill_kv(min(pos, seq_len), seed=7)
            got = dm.forward(19, pos)
            sigma = float(want.std())
            err = float(np.abs(got - want).max())
            print(f"{shape} kv{kvbits} pos {pos}: |cuda-oracle| {err:.2e} = {err / sigma:.1e} sigma")
            assert err <= tol * sigma, (pos, err, sigma)
