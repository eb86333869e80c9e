"""qagnn_b200.optim.clip_grad_norm_ without a GPU: the restated summation order (tests/clip_oracle.py) against a literal
per-thread, per-lane simulation of the kernel and against math.fsum; the coefficient against torch's CPU ops on the same
total; the refusals and the empty case; and the compiled kernels (no floating-point RED / ATOM, no spills)."""
import collections
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from qagnn_b200 import build, optim
from tests import clip_oracle as CO

SIZES = [[0], [1], [3], [8193], [5, 8192 * 2 + 7, 1, 0, 4099], [70_001], [1023, 1024, 1025]]


def _tensors(sizes, seed, spread=True):
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(sizes):
        x = rng.standard_normal(n).astype(np.float32)
        out.append(x * np.float32(10.0 ** (i % 5 - 2)) if spread else x)
    return out


def _shfl_down_tree(vals):
    """lane 0 of 32 lanes after __shfl_down_sync(v, o) for o = 16 .. 1; a lane past 31 reads its own value."""
    v = list(vals)
    for o in (16, 8, 4, 2, 1):
        v = [v[l] + (v[l + o] if l + o < 32 else v[l]) for l in range(32)]
    return v[0]


def _block_sum(partials):
    warps = [_shfl_down_tree(partials[32 * w:32 * w + 32]) for w in range(8)]
    return _shfl_down_tree(warps + [0.0] * 24)


def _simulate(tensors):
    """The kernel's loops written out one thread at a time, in Python floats (IEEE fp64)."""
    slots = []
    for x in tensors:
        x = [float(v) for v in x]
        for c0 in range(0, len(x), CO.CHUNK):
            g = x[c0:c0 + CO.CHUNK]
            n4 = len(g) // 4
            partials = []
            for t in range(CO.THREADS):
                acc = 0.0
                for j in range(t, n4, CO.THREADS):
                    for e in range(4):
                        acc = acc + g[4 * j + e] * g[4 * j + e]
                if 4 * n4 + t < len(g):
                    acc = acc + g[4 * n4 + t] * g[4 * n4 + t]
                partials.append(acc)
            slots.append(_block_sum(partials))
    partials = []
    for t in range(CO.THREADS):
        acc = 0.0
        for s in range(t, len(slots), CO.THREADS):
            acc = acc + slots[s]
        partials.append(acc)
    return _block_sum(partials)


@pytest.mark.parametrize("sizes", SIZES[:5], ids=lambda s: "-".join(map(str, s)))
def test_the_oracle_is_the_kernels_order(sizes):
    ts = _tensors(sizes, 1)
    assert CO.sum_squares(ts) == _simulate(ts)


def test_the_slot_sum_takes_the_kernels_order_past_256_slots():
    # 300 one-chunk tensors: thread t adds slots t and t + 256
    ts = _tensors([5 + i for i in range(300)], 2)
    assert CO.sum_squares(ts) == _simulate(ts)


@pytest.mark.parametrize("sizes", SIZES + [[8192] * 600, [3_000_001, 17]], ids=lambda s: f"{len(s)}x{max(s)}")
def test_the_norm_is_within_one_ulp_of_the_exact_norm(sizes):
    ts = _tensors(sizes, 3)
    exact = math.fsum(float(v) * float(v) for x in ts for v in x.astype(np.float64))  # squares exact, one rounding
    s = CO.sum_squares(ts)
    assert abs(s - exact) <= 1e-14 * exact
    norm = CO.total_norm(ts)
    assert norm.dtype == np.float32
    assert abs(float(norm) - math.sqrt(exact)) <= float(np.spacing(norm))


def test_the_norm_of_nothing_and_of_non_finite_values():
    assert CO.total_norm([]) == 0 and CO.total_norm([np.zeros(0, np.float32)]) == 0
    assert CO.total_norm([np.array([3.0, np.inf], np.float32)]) == np.inf
    assert np.isnan(CO.total_norm([np.array([3.0, np.nan], np.float32), np.array([np.inf], np.float32)]))
    # fp32 squares would overflow; the fp64 sum does not
    assert CO.total_norm([np.array([3e19, 4e19], np.float32)]) == np.float32(5e19)


TOTALS = [0.0, 1e-30, 1e-6, 0.25, 0.999999, 1.0, 1.0000001, 3.7, 12345.678, 1e30, 3.4e38, np.inf, np.nan]


@pytest.mark.parametrize("max_norm", [1.0, 0.1, 5.0, 1e-7, 0.0, 1e9])
def test_the_coefficient_is_torchs_on_the_same_total(max_norm):
    for t in TOTALS:
        total = torch.tensor(t, dtype=torch.float32)
        want = torch.clamp(max_norm / (total + 1e-6), max=1.0)  # torch.nn.utils.clip_grad_norm_'s ops
        got = CO.coefficient(np.float32(t), max_norm)
        assert np.array(got).view(np.int32) == want.numpy().view(np.int32), (max_norm, t, got, want)


# ---- the Python entry's refusals ---------------------------------------------------------------------------------

def test_no_gradient_returns_a_cpu_zero_as_torch_does():
    ps = [torch.nn.Parameter(torch.zeros(3)), torch.nn.Parameter(torch.zeros(2))]
    for arg in (ps, iter(ps), ps[0], []):
        out = optim.clip_grad_norm_(arg, 1.0)
        ref = torch.nn.utils.clip_grad_norm_(arg if not hasattr(arg, "__next__") else iter(ps), 1.0)
        assert out.device == ref.device and out.dtype == ref.dtype and float(out) == float(ref) == 0.0


def test_refusals():
    p = torch.nn.Parameter(torch.zeros(3))
    p.grad = torch.zeros(3)
    for kw, exc, msg in [(dict(norm_type=1.0), ValueError, r"only the L2 norm \(norm_type=2\)"),
                         (dict(norm_type=float("inf")), ValueError, "only the L2 norm"),
                         (dict(error_if_nonfinite=True), ValueError, "error_if_nonfinite=True needs a host read")]:
        with pytest.raises(exc, match=msg):
            optim.clip_grad_norm_([p], 1.0, **kw)
    with pytest.raises(TypeError, match=r"qagnn_b200\.optim\.clip_grad_norm_: the gradient must live on a CUDA device"):
        optim.clip_grad_norm_([p], 1.0)
    p.grad = torch.zeros(3).to_sparse()
    with pytest.raises(TypeError, match=r"clip_grad_norm_: the gradient must be dense \(got torch.sparse_coo\)"):
        optim.clip_grad_norm_([p], 1.0)
    assert torch.equal(p.grad.to_dense(), torch.zeros(3))


def test_it_is_exported_next_to_the_optimiser_table():
    from qagnn_b200.optim import OPTIMIZER_CLASSES, clip_grad_norm_  # noqa: F401
    assert clip_grad_norm_.__name__ == "clip_grad_norm_"


# ---- the compiled kernels ------------------------------------------------------------------------------------------

def _tool(name):
    for cand in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """csrc/clip.cu cross-compiled with the library's flags: (ptxas report, {kernel: opcode counts})."""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("no nvcc / cuobjdump")
    obj = str(tmp_path_factory.mktemp("clip") / "clip.o")
    r = subprocess.run([nvcc, "-c", os.path.join(build.CSRC, "clip.cu"), "-o", obj] + build.NVCC_FLAGS,
                       capture_output=True, text=True, check=True)
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        ops = collections.Counter()
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops[m.group(1)] += 1
        kernels[re.search(r"clip_(?:norm|scale)_kernel", body.split("\n", 1)[0]).group(0)] = ops
    return r.stdout + r.stderr, kernels


def test_neither_kernel_spills(compiled):
    report, _ = compiled
    props = re.findall(r"Function properties for \S*(clip_(?:norm|scale)_kernel)\S*\n\s*(\d+) bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert {name for name, *_ in props} == {"clip_norm_kernel", "clip_scale_kernel"}, report
    for name, stack, stores, loads in props:
        assert int(stack) == int(stores) == int(loads) == 0, (name, report)


def test_no_floating_point_atomics_and_vector_loads(compiled):
    _, kernels = compiled
    assert set(kernels) == {"clip_norm_kernel", "clip_scale_kernel"}
    for name, ops in kernels.items():
        atomics = [op for op in ops if op.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG", "ATOMS")]
        assert not [op for op in atomics if re.search(r"\.F(16|32|64)", op)], (name, atomics)
        assert ops["LDG.E.128"] >= 1, name
    assert sum(n for op, n in kernels["clip_norm_kernel"].items() if op.startswith(("ATOM", "RED"))) == 1  # the counter
    assert not [op for op in kernels["clip_scale_kernel"] if op.startswith(("ATOM", "RED"))]
    assert kernels["clip_norm_kernel"]["DFMA"] >= 4 and kernels["clip_scale_kernel"]["STG.E.128"] >= 1
