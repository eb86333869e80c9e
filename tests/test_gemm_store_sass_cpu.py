"""The split-bf16 GEMM kernels store their epilogue with TMA.

Every `gemm_tc_kernel` and `mlp_tc_kernel` instantiation must contain the bulk tensor store from shared memory (SASS
`UTMASTG`, from `cp.async.bulk.tensor ... global.shared::cta`); the direct-store epilogue, kept for comparison behind
QAGNN_TC_STORE=direct, stores with STG only.
"""
import os
import re
import shutil
import subprocess

import pytest

from qagnn_b200 import _lib


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_every_gemm_instantiation_stores_with_tma():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    if not os.path.exists(_lib.LIB_PATH):
        from qagnn_b200 import build
        build.build()
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    seen, missing = 0, []
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        if "gemm_tc_kernel" not in name and "mlp_tc_kernel" not in name:
            continue
        seen += 1
        if not re.search(r"\bUTMASTG\b", body):
            missing.append(name)
    assert seen == 30, f"expected 24 gemm_tc_kernel and 6 mlp_tc_kernel instantiations, found {seen}"
    assert not missing, "no TMA store in: " + ", ".join(missing[:5])
