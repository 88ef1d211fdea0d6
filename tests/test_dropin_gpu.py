"""The drop-in behaviour on the GPU: the backend, driven the way the UNMODIFIED reference driver (run.c) drives it, decodes a
.calm file's model greedily into the same tokens the reference program printed on its own CPU path (stored in
tests/golden/reference-cpu.npz by tools/make_reference_golden.py) and as the oracle; and CALM_B200_PERF=1 makes the
library print perf_cuda()'s per-stage table when the process exits, as the reference prints its own (run.c:630-632)."""
import hashlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT, golden  # noqa: E402

from calm_b200 import lib  # noqa: E402
from calm_b200 import modelgen as mg  # noqa: E402
from calm_b200.cstructs import FF_UPDATE_KV_ONLY  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["tiny-llama", "tiny-gf4", "tiny-moe"])
def test_reference_driver_with_our_backend(tmp_path, oracle_pkg, name):
    spec = mg.SPECS[name]
    g = golden("reference-cpu")
    model = mg.HostModel(spec, seed=0)
    path = str(tmp_path / "m.calm")
    mg.write_calm(path, spec, model.tensors)
    assert hashlib.sha256(open(path, "rb").read()).hexdigest() == str(g[f"dropin-{name}-sha256"])  # the file the driver decoded
    driver = [int(t) for t in g[f"dropin-{name}-tokens"]]  # the prompt tokens after BOS, then the generated ones
    # run.c: the prompt through forward(FF_UPDATE_KV_ONLY) except its last token, then greedy steps on host logits
    prompt = [spec.bos_id, 7, 8]
    gpu = []
    with lib.DeviceModel(spec, model.tensors) as dm:
        for i, t in enumerate(prompt[:-1]):
            assert dm.forward(t, i, FF_UPDATE_KV_ONLY) is None
        tok, pos = prompt[-1], len(prompt) - 1
        for _ in range(len(driver) - 2):
            tok = int(np.argmax(dm.forward(tok, pos)))
            gpu.append(tok)
            pos += 1
    assert driver[:2] == [7, 8]
    assert gpu == driver[2:], (gpu, driver)
    # and the oracle's greedy continuation of BOS, 7, 8
    ck = oracle_pkg.Checker("port")
    m2 = mg.HostModel(spec, seed=0)
    ck.prepare(m2)
    for i, t in enumerate(prompt):
        logits = ck.forward(m2, t, i)
    gen, pos = [], len(prompt)
    for _ in range(8):
        nxt = int(logits.argmax())
        gen.append(nxt)
        logits = ck.forward(m2, nxt, pos)
        pos += 1
    assert gpu[:len(gen)] == gen[:len(gpu)]


def test_perf_table_through_the_reference_driver(tmp_path):
    """CALM_B200_PERF=1: a process that decodes and exits without releasing the model (as the reference driver does,
    run.c:636) ends with perf_cuda()'s per-stage table; timings come from inside the production graph."""
    code = ("from calm_b200 import lib, modelgen as mg\n"
            "spec = mg.SPECS['tiny-llama']\n"
            "dm = lib.DeviceModel(spec, mg.HostModel(spec, seed=0).tensors)\n"
            "tok = 7\n"
            "for i in range(16):\n"
            "    tok = int(dm.forward(tok, i).argmax())\n")
    env = dict(os.environ, PYTHONPATH=ROOT, CALM_B200_PERF="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-800:]
    assert "forward breakdown" in r.stdout and "matmul_ffn_up" in r.stdout and "GB/s" in r.stdout, r.stdout[-600:]
    rows = re.findall(r"\[(\d)\]\s+(\w+):\s+([0-9.]+)%;\s+([0-9.]+) usec/run", r.stdout)
    assert len(rows) >= 5 and abs(sum(float(x[2]) for x in rows) - 100.0) < 1.0
