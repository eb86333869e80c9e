"""The deterministic backward of the message-passing core sums the edge-table gradients without float atomics.

Its table-kernel instantiations (mp_bwd_table_kernel<H, CH, S, true>) and the combine kernel that adds the per-run slots
must store with plain STG: a floating-point RED or ATOM in their SASS makes d_ke / d_me depend on scheduling again.  The
default instantiations (<..., false>) keep their RED.ADD.F32 and are the control that the check sees atomics at all.
"""
import os
import re
import shutil
import subprocess

import pytest

from qagnn_b200 import _lib

HEADS, CHUNKS, STORAGE = (1, 2, 4, 8, 16), (1, 2, 4, 8), 3


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
        if "mp_bwd_table" not in name:
            continue
        ops = []
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops.append(m.group(1))
        out[name] = ops
    return out


def _float_atomics(ops):
    """Global or generic reductions / atomics on a floating-point type, e.g. REDG.E.ADD.F32.FTZ.RN.STRONG.GPU."""
    return [op for op in ops if op.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG") and re.search(r"\.(F32|F16|BF16|F64)", op)]


def _split(kernels):
    # mp_bwd_table_kernel<H, CH, S, kDet>: the mangled name ends its template arguments with Lb1E (true) or Lb0E (false)
    det = {n: o for n, o in kernels.items() if "mp_bwd_table_kernel" in n and "Lb1E" in n}
    dflt = {n: o for n, o in kernels.items() if "mp_bwd_table_kernel" in n and "Lb0E" in n}
    combine = {n: o for n, o in kernels.items() if "mp_bwd_table_combine_kernel" in n}
    return det, dflt, combine


def test_every_table_instantiation_is_found(kernels):
    det, dflt, combine = _split(kernels)
    n = len(HEADS) * len(CHUNKS) * STORAGE
    assert len(det) == n and len(dflt) == n, (len(det), len(dflt))
    assert len(combine) == 1


def test_default_table_kernels_keep_their_atomics(kernels):
    _, dflt, _ = _split(kernels)
    assert all(_float_atomics(ops) for ops in dflt.values()), "the atomic check no longer sees the default path's RED"


def test_deterministic_table_and_combine_kernels_have_no_float_atomics(kernels):
    det, _, combine = _split(kernels)
    bad = {n: sorted(set(_float_atomics(ops))) for n, ops in {**det, **combine}.items() if _float_atomics(ops)}
    assert not bad, "\n".join(f"{n}: {ops}" for n, ops in list(bad.items())[:10])
