"""The fp64 references of tests/ragged_pool_oracle.py against autograd of the fp64 MultiheadAttPoolLayer, and the rows of
tests/test_gpu_ragged_ends.py against the shared-memory limits of qagnn_b200/csrc/pool.cu, without a GPU.

Once the closed-form backward equals autograd to 1e-10 of its magnitude (a fully masked graph, a length-1 graph and a head
width of 5 included), a GPU test that fails against it can only be failing on the kernel."""
import os
import re

import pytest
import torch

from oracle import qagnn_oracle as O
from qagnn_b200.layers import MultiheadAttPoolLayer
from tests import ragged_pool_oracle as RP
from tests import test_gpu_ragged_ends as RE

F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(nh, D, n, S, lens, seed):
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    lens = torch.tensor(lens)
    nt = torch.randint(0, 4, (B, n), generator=g)
    nt[:, 0] = 3
    nt[1, :] = 3  # graph 1: every node a context node, so every position is masked and node 0 is kept
    X = torch.randn(B, n, D, generator=g, dtype=F64)
    X[torch.arange(n) >= lens.unsqueeze(1)] = 0.0  # the re-padded layout of a ragged batch
    torch.manual_seed(seed)
    pool = MultiheadAttPoolLayer(nh, D, D).double().eval()
    with torch.no_grad():  # w_qs = identity: q is the kernel's qs
        pool.w_qs.weight.copy_(torch.eye(D, dtype=F64))
        pool.w_qs.bias.zero_()
        pool.w_ks.bias.normal_(0, 0.5, generator=g)
        pool.w_vs.bias.normal_(0, 0.5, generator=g)
    qs = torch.randn(B, D, generator=g, dtype=F64)
    dconcat = torch.randn(B, 2 * D + S, generator=g, dtype=F64)
    return pool, qs, X, RP.tail_mask(lens, nt), dconcat


@pytest.mark.parametrize("nh,D,n,S,lens", [
    (3, 15, 6, 4, [1, 4, 6, 9, 2]),    # dk = 5; graph 0 of length 1, graph 3 longer than n
    (1, 8, 1, 0, [1, 1]),              # n = 1, S = 0
    (4, 64, 40, 7, [40, 13, 1, 27]),
    (8, 200, 33, 5, [33, 2, 17]),
])
def test_closed_form_backward_equals_fp64_autograd(nh, D, n, S, lens):
    pool, qs, X, mask, dconcat = _case(nh, D, n, S, lens, seed=nh * 100 + n)
    q, x = qs.clone().requires_grad_(True), X.clone().requires_grad_(True)
    pooled, attn = pool(q, x, mask)
    (pooled * dconcat[:, :D]).sum().add_((x[:, 0] * dconcat[:, D + S:]).sum()).backward()
    # the folded forward is the layer's forward
    p2, a2 = RP.pool_forward(qs, X, mask, pool.w_ks.weight, pool.w_ks.bias, pool.w_vs.weight, pool.w_vs.bias, nh)
    assert torch.allclose(p2, pooled.detach(), rtol=1e-12, atol=1e-12) and torch.allclose(a2, attn.detach(), rtol=0, atol=1e-14)
    assert bool((a2.view(nh, -1, n)[:, 1, 1:] == 0).all()) and bool((a2.view(nh, -1, n)[:, 1, 0] == 1).all())
    r = RP.pool_backward(qs, X, attn.detach(), dconcat, pool.w_ks.weight, pool.w_ks.bias, pool.w_vs.weight, nh, S)
    for name, got in (("dX", x.grad), ("dqs", q.grad), ("dwk", pool.w_ks.weight.grad), ("dbk", pool.w_ks.bias.grad),
                      ("dwv", pool.w_vs.weight.grad), ("dbv", pool.w_vs.bias.grad)):
        val, mag = r[name][0], r["mag"][name]
        err = (val - got).abs()
        assert bool((err <= 1e-10 * mag + 1e-300).all()), f"{name}: closed form off autograd by {float(err.max()):.3e}"
    # softmax is shift invariant: the key bias gets no gradient, and its bar holds 0 as well
    assert float(pool.w_ks.bias.grad.abs().max()) <= float(r["dbk"][1].max())


def test_folded_forward_equals_the_oracle_pooler():
    nh, D, n, S = 5, 100, 30, 12
    g = torch.Generator().manual_seed(3)
    pool = MultiheadAttPoolLayer(nh, S, D).double().eval()
    sd = {"pooler." + k: v.detach() for k, v in pool.state_dict().items()}
    q, X = torch.randn(4, S, generator=g, dtype=F64), torch.randn(4, n, D, generator=g, dtype=F64)
    mask = RP.tail_mask(torch.tensor([1, 30, 7, 40]), torch.randint(0, 4, (4, n), generator=g))
    ref_p, ref_a = O.multihead_att_pool(sd, "pooler", q, X, mask, nh)
    qs = pool.w_qs(q).detach()
    p, a = RP.pool_forward(qs, X, mask, pool.w_ks.weight, pool.w_ks.bias, pool.w_vs.weight, pool.w_vs.bias, nh)
    assert torch.allclose(p, ref_p, rtol=1e-12, atol=1e-12) and torch.allclose(a, ref_a, rtol=0, atol=1e-14)


def test_pack_and_repad_are_inverse():
    lens, n = torch.tensor([1, 5, 9, 3]), 5
    node_ptr, N_cap, rows = RP.ragged_layout(lens, n, tail_rows=7)
    assert node_ptr.tolist() == [0, 1, 6, 11, 14] and N_cap == 21
    X = torch.randn(4, n, 3, dtype=F64)
    tail = torch.randn(7, 3, dtype=F64)
    Xp = RP.pack(X, rows, N_cap, tail)
    assert torch.equal(Xp[14:], tail) and torch.equal(Xp[1:6], X[1])
    fill = torch.randn(4, n, 3, dtype=F64)
    Y = RP.repad(Xp, rows, 4, n, fill)
    valid = torch.arange(n) < lens.clamp(max=n).unsqueeze(1)
    assert torch.equal(Y[valid], X[valid]) and torch.equal(Y[~valid], fill[~valid])


# ---- the shared-memory limits of pool.cu, and the table rows that straddle them ----------------------------------------
def _pool_cu_constants():
    src = open(os.path.join(ROOT, "qagnn_b200", "csrc", "pool.cu")).read()
    cap = re.search(r"constexpr size_t kPoolSmemCap = (\d+) \* 1024;", src)
    thr = re.search(r"constexpr int kPoolThreads = (\d+);", src)
    bthr = re.search(r"constexpr int kPoolBwdThreads = (\d+);", src)
    fwd = re.search(r"pool_smem_bytes\(int n, int D, int nh\) \{\s*return \(\(size_t\)2 \* nh \* D \+ \(size_t\)nh \* n \+ nh \+ 16 \+ "
                    r"\(size_t\)\(kPoolThreads / 32\) \* nh \* D\) \* sizeof\(float\);", src)
    bwd = re.search(r"pool_backward_smem_bytes\(int D\) \{ return \(\(size_t\)3 \* D \+ kPoolBwdThreads / 32\) \* sizeof\(float\); \}",
                    src)
    refuse = re.search(r"if \(pool_smem_bytes\(n, D, n_head\) > kPoolSmemCap\) return QAGNN_ERR_UNSUPPORTED;  // the forward", src)
    assert cap and thr and bthr and fwd and bwd and refuse, "pool.cu's shared-memory formulas changed: update this test"
    return int(cap.group(1)) * 1024, int(thr.group(1)), int(bthr.group(1))


def test_limit_formulas_match_pool_cu():
    cap, thr, bthr = _pool_cu_constants()
    assert cap == RE.POOL_SMEM_CAP
    for nh in range(1, 9):
        for D in (nh, 8 * nh, 200 - 200 % nh, 1024 - 1024 % nh, 5000 - 5000 % nh):
            for n in (1, 257, 4000, 50000):
                fwd = (2 * nh * D + nh * n + nh + 16 + (thr // 32) * nh * D) * 4
                bwd = (3 * D + bthr // 32) * 4
                assert fwd == RE.pool_smem(n, D, nh) and bwd == RE.pool_bwd_smem(D)
                # the backward's shared memory never exceeds the forward's: it takes every shape the forward takes
                assert bwd < fwd


def test_every_limit_has_a_row_at_it_and_one_past_it():
    rows = {(r[0], r[1], r[2]) for r in RE.LIMIT_CASES}
    for nh in range(1, 9):
        for D in (RE.limit_D(D, nh) for D in RE.LIMIT_DS):
            assert D % nh == 0
            nmax = RE.max_pool_len(D, nh)
            if nmax >= 1:
                assert RE.pool_smem(nmax, D, nh) <= RE.POOL_SMEM_CAP < RE.pool_smem(nmax + 1, D, nh)
                assert (nh, D, nmax) in rows and (nh, D, nmax + 1) in rows, (nh, D)
            else:  # no node count fits: n = 1 is already refused
                assert RE.pool_smem(1, D, nh) > RE.POOL_SMEM_CAP and (nh, D, 1) in rows, (nh, D)
    for nh, D, n, accepted in RE.LIMIT_CASES:
        assert accepted == (RE.pool_smem(n, D, nh) <= RE.POOL_SMEM_CAP), (nh, D, n)


def test_the_case_table_covers_every_branch():
    cases = RE.TAIL_CASES
    assert {c.nh for c in cases} == set(range(1, 9))
    dks = {c.D // c.nh for c in cases}
    assert any(dk % 4 for dk in dks) and any(dk % 32 and dk % 4 == 0 for dk in dks)
    Ds = {c.D for c in cases}
    assert min(Ds) < 128 and any(128 < D <= 256 for D in Ds) and max(Ds) > 256
    assert {1, 2, 3, 4, 5, 255, 256, 257, 1000} <= {c.n for c in cases}
    Ss = {c.S for c in cases}
    assert 0 in Ss and any(S % 2 for S in Ss) and max(Ss) >= 1024
    Bs = {c.B for c in cases}
    assert 1 in Bs and max(Bs) >= 100
    assert {"none", "few", "many"} == {c.tail for c in cases}
    assert {torch.float32, torch.bfloat16} == {c.xdtype for c in cases}
    for c in cases:
        assert c.name, c
        lens, nt = RE.lengths_and_types(c)
        assert lens.numel() == c.B and int(lens.min()) >= 1
        _, N_cap, rows = RP.ragged_layout(lens, c.n, RE.tail_rows(c))
        if c.tail == "many":
            assert N_cap - rows.numel() > c.B  # the head kernel's r += B loop runs more than once
        if c.B >= 4:  # every length edge: length 1, length n (or more), a graph of context nodes only
            assert 1 in lens.tolist() and int(lens.max()) >= c.n
            assert any(bool((nt[b, :min(int(lens[b]), c.n)] == 3).all()) for b in range(c.B))
