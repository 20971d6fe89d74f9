"""Per-warp staging of the sliced native build (scalar form, Next kernels): an emit site puts its successor into its
warp's shared-memory buffer, and the whole warp fingerprints, probes and appends the staged successors together.  A
lane that finds the buffer full probes where it is, as without staging.  Counts, per-level sizes and digests must not
move with staging at its compiled size, switched off (TLAG_SL_STAGE=0) or capped at one warp's worth of slots
(TLAG_SL_STAGE=32: flushes and full buffers both happen).  On the CPU: the Next kernels of the bench model still fit
4 CTAs per SM with no local memory."""
import os
import re
import shutil
import subprocess

import pytest

import test_sliced_self_loops as self_loops
from conftest import GOLDEN
from tla_rust_b200.compiled import load_compiled


def _resource_usage(so):
    """{kernel name: {REG, STACK, SHARED, LOCAL}} from cuobjdump"""
    out = subprocess.run([shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump", "--dump-resource-usage", so],
                         capture_output=True, text=True, check=True).stdout
    usage, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            usage[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", line)}
            name = None
    return usage


def test_staged_next_kernels_keep_four_ctas_per_sm():
    from tla_rust_b200 import engine
    cm, _, _, _ = load_compiled(os.path.join(GOLDEN, "MCPaxos3_b4.tlagz"))
    so = engine.sliced_library_path(cm)
    if not os.path.exists(so):
        pytest.skip(f"{so} is not built (build())")
    if not (shutil.which("cuobjdump") or os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("no cuobjdump")
    nxt = {k: v for k, v in _resource_usage(so).items() if "k_sl_next_" in k}
    assert nxt
    for name, u in nxt.items():
        assert u["REG"] <= 64, (name, u)              # 65536 registers / (256 threads x 4 CTAs)
        assert u["LOCAL"] == 0, (name, u)             # no spills
        assert u["SHARED"] > 0, (name, u)             # the staging buffer is compiled in
        assert 4 * u["SHARED"] <= 228 * 1024, (name, u)


@pytest.mark.gpu
@pytest.mark.parametrize("stage,skip_self", [(None, "1"), ("0", "1"), ("32", "1"), ("32", "0")])
@pytest.mark.parametrize("name,max_levels", self_loops.CASES)
def test_sliced_kernels_match_the_oracle_with_staging(monkeypatch, name, max_levels, stage, skip_self):
    if stage is None:
        monkeypatch.delenv("TLAG_SL_STAGE", raising=False)
    else:
        monkeypatch.setenv("TLAG_SL_STAGE", stage)
    self_loops.test_sliced_kernels_match_the_oracle_with_and_without_the_filter(monkeypatch, name, max_levels, skip_self)
