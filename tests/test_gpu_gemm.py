"""The split-bf16 wgmma GEMM (`gemm_tc_kernel`) on its own, through `ops.linear_bf16x3`, against fp64.

    out = act([A1 | A2] @ W^T + b)

Operands are split into bf16 hi + lo planes (16 mantissa bits) and every k16 step issues hi*hi, hi*lo, lo*hi, so the error
of an output element is bounded by 2^-15 * (|A| . |W|^T) plus the fp32 roundings of bias and activation.  That bound is far
below the contribution of any single k16 step, so a dropped or repeated step fails it (`test_bound_detects_one_k_column`).
Every case runs with CTA pairs (QAGNN_TC_2CTA=1, W multicast) and single CTAs (QAGNN_TC_2CTA=0) and requires the two
results to be bitwise equal: both run the same k16 steps in the same order.
"""
import pytest
import torch

DEV = "cuda:0"
ACTS = ("none", "relu", "gelu")


def _inputs(M, N, K1, K2, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a1 = torch.randn(M, K1, device=DEV, generator=g) * 0.5
    a2 = torch.randn(M, K2, device=DEV, generator=g) * 0.5 if K2 else None
    w = torch.randn(N, K1 + K2, device=DEV, generator=g) / (K1 + K2) ** 0.5
    b = torch.randn(N, device=DEV, generator=g) * 0.1
    return a1, a2, w, b


def _reference(a1, a2, w, b, act):
    """fp64 result and the per-element error bound of the split-bf16 product."""
    A = torch.cat([a1, a2], 1) if a2 is not None else a1
    pre = A.double() @ w.double().t() + b.double()
    mag = A.double().abs() @ w.double().abs().t()
    ref = pre
    if act == "relu":
        ref = pre.relu()
    elif act == "gelu":
        ref = torch.nn.functional.gelu(pre, approximate="tanh")
    # GELU's slope stays below 1.13; the fast tanh form is good to ~1e-6 absolute; bias add and activation round in fp32
    bound = 1.13 * 2.0 ** -15 * mag + 2e-6 + 2.0 ** -22 * ref.abs()
    return ref, bound


def _run(monkeypatch, a1, a2, w, b, act):
    from qagnn_b200 import ops
    outs = []
    for ctas in ("1", "0"):
        monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
        outs.append(ops.linear_bf16x3(a1, w, b, a2, act))
    torch.cuda.synchronize()
    return outs


def _check(monkeypatch, M, N, K1, K2, act, seed=0):
    a1, a2, w, b = _inputs(M, N, K1, K2, seed)
    pair, single = _run(monkeypatch, a1, a2, w, b, act)
    assert torch.equal(pair, single), "CTA-pair and single-CTA results differ"
    ref, bound = _reference(a1, a2, w, b, act)
    err = (pair.double() - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"M={M} N={N} K={K1}+{K2} act={act}: {int(bad.sum())} elements outside the bound; "
                                 f"max err {err.max().item():.3e}, max err/bound {(err / bound).max().item():.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("N", [8, 40, 64, 120, 200, 208, 256, 600, 624])
def test_tile_widths(monkeypatch, N):
    """Every compiled wgmma width (64, 128, 208, 256) and the n tiles that cut them short."""
    _check(monkeypatch, 257, N, 200, 104, ACTS[N % 3])


@pytest.mark.gpu
@pytest.mark.parametrize("K2", [0, 104, 200])
@pytest.mark.parametrize("K1", [8, 72, 96, 200, 248, 304])
def test_k_segments(monkeypatch, K1, K2):
    """One and two A segments with K off the k-block grid: the last block of each segment runs only the k16 steps that
    reach its K, and the second segment's weight columns start at K1."""
    _check(monkeypatch, 129, 200, K1, K2, "none")


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 127, 128, 129, 255, 257, 64000])
def test_ragged_rows(monkeypatch, M):
    """Row counts around the 128-row tile and the 256-row CTA pair, and the projection's full size."""
    _check(monkeypatch, M, 624, 304, 0, "none")


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_activations(monkeypatch, act):
    _check(monkeypatch, 1000, 208, 200, 200, act, seed=1)


@pytest.mark.gpu
def test_bound_detects_one_k_column(monkeypatch):
    """The bound is tight enough to see one k column: a result computed without the last column's contribution (the one k16
    step of a tail block) fails it.  The kernel runs on weights whose last column is perturbed; the reference keeps them."""
    M, N, K1 = 257, 200, 200
    a1, _, w, b = _inputs(M, N, K1, 0, 3)
    w_bad = w.clone()
    w_bad[:, K1 - 1] += 0.05
    pair, single = _run(monkeypatch, a1, None, w_bad, b, "none")
    assert torch.equal(pair, single)
    ref, bound = _reference(a1, None, w, b, "none")
    assert bool(((pair.double() - ref).abs() > bound).any())
