"""`proj_resident_kernel` releases its ring stages without a GPU-scope fence, keeps its mainloop's wgmma unserialised and
stores through TMA.

The stage-release rule is the one of test_gemm_sass_cpu.py: no MEMBAR in the instructions before an
`SYNCS.ARRIVE.TRANS64[.RED].A1T0`, except the entry / exit `barrier.cluster`'s.
"""
import os
import re
import shutil
import subprocess

import pytest

from qagnn_b200 import _lib

WINDOW = 8  # instructions before a release arrive that must hold no MEMBAR
NAME = "proj_resident_kernel"


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
        if NAME not in name:
            continue
        ops = []
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops.append(m.group(1))
        out[name] = ops
    return out


def test_both_cta_settings_are_compiled(kernels):
    assert len(kernels) == 2, sorted(kernels)


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


def test_epilogue_stores_with_tma(kernels):
    for name, ops in kernels.items():
        assert any(op.startswith("UTMASTG") for op in ops), f"{name}: no TMA store"


def test_mma_chains_at_n104(kernels):
    """Three HGMMAs per k16 step: 4 steps in the full k blocks' chain and 1 + 2 + 3 + 4 in the K-tail switch (ptxas may keep
    one or two instructions outside the chains, e.g. a chain's first MMA peeled)."""
    for name, ops in kernels.items():
        n = sum(op.startswith("HGMMA") for op in ops)
        assert abs(n - 3 * (4 + 1 + 2 + 3 + 4)) <= 2, f"{name}: {n} HGMMA"

def test_ptxas_reports_no_spills_or_serialised_wgmma():
    log = os.path.join(os.path.dirname(_lib.LIB_PATH), "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log")
    text = open(log).read()
    assert not re.search(r"C7520.*" + NAME, text), "ptxas serialised the resident kernel's wgmma"
    props = re.findall(r"Function properties for \S*" + NAME + r"\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", text)
    assert len(props) == 2 and all(p == ("0", "0", "0") for p in props), props
