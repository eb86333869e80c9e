"""The split-bf16 GEMM kernels release ring stages without a GPU-scope fence.

A stage release is a plain `mbarrier` arrive on the `empty` barrier of each CTA of the pair: SASS
`SYNCS.ARRIVE.TRANS64.RED.A1T0` on a CTA of the cluster, `SYNCS.ARRIVE.TRANS64.A1T0` on the CTA's own barrier (the producer's
arrive with an expected byte count has a register operand instead).
Arriving with `.release.cluster` semantics makes ptxas put `MEMBAR.ALL.CTA; MEMBAR.ALL.GPU` in front of it, which waits for
every global store the thread has in flight and sits on the critical path of every k block.  The only fence these kernels
may keep is the once-per-kernel one of the entry and exit `barrier.cluster` (a MEMBAR followed by `UCGABAR_ARV`).
"""
import os
import re
import shutil
import subprocess

import pytest

from qagnn_b200 import _lib

WINDOW = 8  # instructions before a release arrive that must hold no MEMBAR


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def kernels():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    if not os.path.exists(_lib.LIB_PATH):
        from qagnn_b200 import build
        build.build()
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        if "gemm_tc_kernel" not in name and "mlp_tc_kernel" not in name:
            continue
        # "/*0a60*/   @!P1 MEMBAR.ALL.GPU ;   /* encoding */" -> "MEMBAR.ALL.GPU"
        ops = []
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops.append(m.group(1))
        out[name] = ops
    return out


def test_every_gemm_instantiation_is_found(kernels):
    # 3 activations x 4 tile widths x {single CTA, CTA pair}, and 3 activations x 2 for the fused MLP
    assert sum("gemm_tc_kernel" in n for n in kernels) == 24
    assert sum("mlp_tc_kernel" in n for n in kernels) == 6


def test_stage_release_carries_no_fence(kernels):
    bad = []
    for name, ops in kernels.items():
        releases = [i for i, op in enumerate(ops) if op.startswith("SYNCS.ARRIVE.TRANS64") and op.endswith(".A1T0")]
        assert releases, f"{name}: no stage-release arrive found"
        for i in releases:
            for j in range(max(0, i - WINDOW), i):
                if not ops[j].startswith("MEMBAR"):
                    continue
                if "UCGABAR_ARV" in ops[j + 1:j + 5]:
                    continue  # the entry / exit cluster barrier
                bad.append(f"{name}: {ops[j]} {i - j} instructions before {ops[i]}")
    assert not bad, "\n".join(bad[:10])
