"""The single-pass bf16 GEMM kernels (`gemm_bf16_kernel`, `mlp_bf16_kernel`) of the eval forward under bf16 autocast.

They are the split-bf16 kernels' body with the lo passes dropped: one HGMMA per k16 step instead of three, the same stage
release without a GPU-scope fence (the rule of test_gemm_sass_cpu.py), and the same TMA-store epilogue.
"""
import os
import re
import shutil
import subprocess

import pytest

from qagnn_b200 import _lib

WINDOW = 8  # instructions before a release arrive that must hold no MEMBAR
NAMES = ("gemm_tc_kernel", "mlp_tc_kernel", "gemm_bf16_kernel", "mlp_bf16_kernel")


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
        if not any(n in name for n in NAMES):
            continue
        ops = []
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops.append(m.group(1))
        out[name] = ops
    return out


def _single(kernels):
    return {n: ops for n, ops in kernels.items() if "gemm_bf16_kernel" in n or "mlp_bf16_kernel" in n}


def _split_twin(name):
    # _ZN...16gemm_bf16_kernelILi2ELi208ELi1EEEv... -> _ZN...14gemm_tc_kernelILi2ELi208ELi1EEEv...
    return name.replace("16gemm_bf16_kernel", "14gemm_tc_kernel").replace("15mlp_bf16_kernel", "13mlp_tc_kernel")


def test_every_single_pass_instantiation_is_found(kernels):
    # 3 activations x 4 tile widths x {single CTA, CTA pair}, and 3 activations x 2 for the fused MLP
    single = _single(kernels)
    assert sum("gemm_bf16_kernel" in n for n in single) == 24
    assert sum("mlp_bf16_kernel" in n for n in single) == 6
    for n in single:
        assert _split_twin(n) in kernels, f"{n}: no split-bf16 counterpart"


def test_stage_release_carries_no_fence(kernels):
    bad = []
    for name, ops in _single(kernels).items():
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
    for name, ops in _single(kernels).items():
        assert any(op.startswith("UTMASTG") for op in ops), f"{name}: no TMA store"


def test_a_third_of_the_mma_instructions(kernels):
    """One HGMMA per k16 step where the split kernel issues three (hi*hi, hi*lo, lo*hi)."""
    for name, ops in _single(kernels).items():
        n1 = sum(op.startswith("HGMMA") for op in ops)
        n3 = sum(op.startswith("HGMMA") for op in kernels[_split_twin(name)])
        assert n1 > 0
        # every MMA chain the split kernel unrolls has a single-pass counterpart of a third of its length; ptxas may keep
        # one or two instructions outside the chains (e.g. a chain's first MMA peeled)
        assert abs(3 * n1 - n3) <= 3, f"{name}: {n1} HGMMA vs {n3} in the split kernel"
