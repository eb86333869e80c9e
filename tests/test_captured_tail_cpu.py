"""optim.CapturedTail without a GPU: its refusals, the C entries in the header and the ctypes binding, the compiled tail
kernels (0 spills, vector loads, no floating-point atomics) and the bytes per parameter the benchmark counts from shapes."""
import collections
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

from qagnn_b200 import _lib, build, optim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("qagnn_step_tail_block_bytes", "qagnn_step_tail_fill", "qagnn_step_tail")
TAIL_KERNELS = {"tail_norm_kernel", "tail_radam_kernel", "tail_adamw_kernel", "tail_adam_kernel", "tail_sgd_kernel"}


def test_torch_sgd_and_adam_are_sent_to_the_eager_tail():
    p = torch.zeros(3, requires_grad=True)
    for opt in (torch.optim.SGD([p], lr=0.1), torch.optim.Adam([p])):
        with pytest.raises(ValueError, match="eager tail"):
            optim.CapturedTail(opt)


def test_cpu_tensors_are_refused():
    p = torch.zeros(3, requires_grad=True)
    p.grad = torch.ones(3)
    with pytest.raises(TypeError, match="CUDA device"):
        optim.CapturedTail(optim.RAdam([p]), max_grad_norm=1.0)()


def test_no_gradient_is_refused():
    p = torch.zeros(3, requires_grad=True)
    with pytest.raises(RuntimeError, match="no parameter has a gradient"):
        optim.CapturedTail(optim.AdamW([p]))()


def test_a_prior_unscale_is_refused():
    p = torch.zeros(3, requires_grad=True)
    opt = optim.RAdam([p])
    scaler = torch.amp.GradScaler("cpu")
    scaler.scale(p.sum()).backward()
    scaler.unscale_(opt)
    with pytest.raises(RuntimeError, match="unscale_"):
        optim.CapturedTail(opt, scaler=scaler, max_grad_norm=1.0)()


def test_a_disabled_scaler_counts_as_none():
    p = torch.zeros(3, requires_grad=True)
    tail = optim.CapturedTail(optim.RAdam([p]), scaler=torch.amp.GradScaler("cuda", enabled=False))
    assert tail.scaler is None


def test_mixed_devices_are_refused(monkeypatch):
    # two CUDA devices are not needed to reach the check: every tensor check passes and the devices differ
    p, q = torch.zeros(3, requires_grad=True), torch.zeros(3, device="meta", requires_grad=True)
    p.grad, q.grad = torch.ones(3), torch.ones(3, device="meta")
    monkeypatch.setattr(optim, "_check_tensor", lambda *a: None)
    with pytest.raises(ValueError, match="one device"):
        optim.CapturedTail(optim.RAdam([p, q]))()


def test_entries_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    for name in ENTRIES:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert name in _lib.EXPORTS, name
    assert "QAGNN_RULE_RADAM = 0" in header and "QAGNN_RULE_ADAMW = 1" in header


def test_bytes_per_parameter_from_shapes():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        from bench_tail import traffic
    finally:
        sys.path.pop(0)
    assert traffic("eager", clip=True, scaler=True) == 48  # unscale 8, norm 4, scale 8, step 28
    assert traffic("captured", clip=True, scaler=True) == 36  # pass 1 reads 4, pass 2 moves 32
    assert traffic("eager", clip=False, scaler=True) == traffic("captured", clip=False, scaler=True) - 4 == 32
    assert traffic("eager", clip=False, scaler=False) == traffic("captured", clip=False, scaler=False) == 28


# ---- the compiled kernels ------------------------------------------------------------------------------------------

def _tool(name):
    for cand in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """csrc/tail.cu cross-compiled with the library's flags: (ptxas report, {kernel: opcode counts})."""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("no nvcc / cuobjdump")
    obj = str(tmp_path_factory.mktemp("tail") / "tail.o")
    r = subprocess.run([nvcc, "-c", os.path.join(build.CSRC, "tail.cu"), "-o", obj] + build.NVCC_FLAGS,
                       capture_output=True, text=True, check=True)
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        ops = collections.Counter()
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops[m.group(1)] += 1
        kernels[re.search(r"tail_(?:norm|radam|adamw|adam|sgd)_kernel", body.split("\n", 1)[0]).group(0)] = ops
    return r.stdout + r.stderr, kernels


def test_no_tail_kernel_of_any_rule_spills(compiled):
    report, _ = compiled
    props = re.findall(r"Function properties for \S*(tail_(?:norm|radam|adamw|adam|sgd)_kernel)\S*\n\s*(\d+) bytes stack "
                       r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert {name for name, *_ in props} == TAIL_KERNELS, report
    for name, stack, stores, loads in props:
        assert int(stack) == int(stores) == int(loads) == 0, (name, report)


def test_every_tail_kernel_takes_vector_loads_and_no_floating_point_atomics(compiled):
    _, kernels = compiled
    assert set(kernels) == TAIL_KERNELS
    for name, ops in kernels.items():
        atomics = [op for op in ops if op.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG", "ATOMS")]
        assert not [op for op in atomics if re.search(r"\.F(16|32|64)", op)], (name, atomics)
        assert sum(ops[op] for op in atomics) == 1, (name, atomics)  # the arrival counter
        assert ops["LDG.E.128"] >= 1, name
    for name in ("tail_radam_kernel", "tail_adamw_kernel"):
        assert kernels[name]["LDG.E.128"] == 4 and kernels[name]["STG.E.128"] >= 3, name
    assert kernels["tail_norm_kernel"]["DFMA"] >= 4
