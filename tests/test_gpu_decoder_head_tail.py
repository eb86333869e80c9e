"""The decoder's two ends against fp64: the attention pooling of csrc/pool.cu in both of its modes and the decoder head.

`attention_pool_kernel` is launched with an explicit mask (qagnn_attention_pool, MultiheadAttPoolLayer.forward) or with the
mask derived from adj_lengths / node_type, writing cat(graph_vecs, sent_vecs, Z) (qagnn_decoder_tail,
MultiheadAttPoolLayer.pool_concat).  It branches on what these tests sweep: heads in passes of four (nh = 5..8 take a
second pass, nh = 1, 3 a partial one), head widths that are not a multiple of 4 or 32, nodes in steps of four per warp,
columns in steps of 128 per warp, more than 48 KB of dynamic shared memory (opt-in), and a refusal above 200 KB after
which the module pools with its einsum path.  `decoder_head_kernel` (qagnn_decoder_head) writes the context node and the
gathered concept rows and normalises the node scores.

References, all fp64 on the CPU: O.multihead_att_pool (pooling), O.decoder_pool_mask (the tail's mask) and
O.decoder_head (the head).  Tolerances: attn |err| <= 2e-6 + 1e-4 |ref|; pooled vectors and scores
|err| <= 2e-5 max|ref| + 1e-4 |ref|; copies bit for bit.  Positions where the reference is NaN must be NaN, no others.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle import qagnn_oracle as O
from qagnn_b200 import _lib
from qagnn_b200.layers import MultiheadAttPoolLayer
from tests import helpers as Hh

pytestmark = pytest.mark.gpu

F64 = torch.float64
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POOL_SMEM_CAP = 200 * 1024  # kPoolSmemCap, qagnn_b200/csrc/pool.cu


def pool_smem(n, D, nh):
    """pool_smem_bytes of qagnn_b200/csrc/pool.cu: qk, xs [nh, D], logits [nh, n], constants, 8 warps' partial sums."""
    return (2 * nh * D + nh * n + nh + 16 + 8 * nh * D) * 4


def max_pool_len(D, nh):
    """The largest node count the pooling kernel takes at (D, nh)."""
    return (POOL_SMEM_CAP // 4 - 10 * nh * D - nh - 16) // nh


# ---------------------------------------------------------------------------------------------------------------------
# tolerances
# ---------------------------------------------------------------------------------------------------------------------
def _split_nan(got, ref, what):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    nan_g, nan_r = torch.isnan(got), torch.isnan(ref)
    assert torch.equal(nan_g, nan_r), f"{what}: NaN at {int((nan_g & ~nan_r).sum())} positions the reference has none, " \
                                      f"and missing at {int((nan_r & ~nan_g).sum())}"
    assert torch.isfinite(got[~nan_g]).all(), f"{what}: infinite values"
    return got[~nan_g], ref[~nan_r]


def attn_excess(got, ref, what="attn"):
    """max(|err| - (2e-6 + 1e-4 |ref|)) over the non-NaN positions: <= 0 within the bar."""
    g, r = _split_nan(got, ref, what)
    return float(((g - r).abs() - (2e-6 + 1e-4 * r.abs())).max()) if r.numel() else -1.0


def value_excess(got, ref, what="value"):
    """max(|err| - (2e-5 max|ref| + 1e-4 |ref|)) over the non-NaN positions: <= 0 within the bar."""
    g, r = _split_nan(got, ref, what)
    return float(((g - r).abs() - (2e-5 * float(r.abs().max()) + 1e-4 * r.abs())).max()) if r.numel() else -1.0


def assert_attn(got, ref, what):
    ex = attn_excess(got, ref, what)
    assert ex <= 0, f"{what}: exceeds 2e-6 + 1e-4|ref| by {ex:.3e}"


def assert_value(got, ref, what):
    ex = value_excess(got, ref, what)
    assert ex <= 0, f"{what}: exceeds 2e-5 max|ref| + 1e-4|ref| by {ex:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# inputs, references and the two ways in (module, C ABI)
# ---------------------------------------------------------------------------------------------------------------------
def make_pooler(nh, S, D, seed):
    torch.manual_seed(seed)
    return MultiheadAttPoolLayer(nh, S, D).eval()


def pooler_sd(pool, dtype=F64):
    return {"pooler." + k: v.detach().cpu().to(dtype) for k, v in pool.state_dict().items()}


def make_mask(kind, B, n, g):
    if kind == "random":   # 40 % masked, node 0 open so that no row is fully masked
        m = torch.rand(B, n, generator=g) < 0.4
        m[:, 0] = False
    elif kind == "prefix":  # adj_length style: the first L_b nodes open
        m = torch.arange(n) >= torch.randint(1, n + 1, (B, 1), generator=g)
    elif kind == "first":
        m = torch.ones(B, n, dtype=torch.bool)
        m[:, 0] = False
    elif kind == "last":
        m = torch.ones(B, n, dtype=torch.bool)
        m[:, -1] = False
    else:
        raise ValueError(kind)
    return m


def tail_inputs(B, n, g):
    """adj_lengths cycling over 0, 1, n, n + 5 and random values; node_type per row: type 3 on node 0 only, type 3 on
    every node within the length, or mixed types with 3 anywhere.  B = 15 runs every combination of the two."""
    lens = torch.randint(0, n + 6, (B,), generator=g)
    for b, v in zip(range(B), (0, 1, n, n + 5)):
        lens[b::5] = v
    node_type = torch.randint(0, 3, (B, n), generator=g)
    node_type[:, 0] = 3
    for b in range(B):
        if b % 3 == 1:
            node_type[b, :min(int(lens[b]), n)] = 3
        elif b % 3 == 2:
            node_type[b] = torch.randint(0, 4, (n,), generator=g)
    return lens, node_type


def ref_pool_given_qs(pool, qs, X, mask):
    """O.multihead_att_pool in fp64 with w_qs = identity: the reference of the kernel call that receives qs itself."""
    sd = pooler_sd(pool)
    D = X.size(2)
    sd["pooler.w_qs.weight"], sd["pooler.w_qs.bias"] = torch.eye(D, dtype=F64), torch.zeros(D, dtype=F64)
    return O.multihead_att_pool(sd, "pooler", qs.double(), X.double(), mask, pool.n_head)


def _weights(pool):
    return [_lib.ptr(t.detach()) for t in (pool.w_ks.weight, pool.w_ks.bias, pool.w_vs.weight, pool.w_vs.bias)]


SENTINEL = 3.0e38  # outputs start out as this: an element the kernel does not write fails every comparison


def abi_attention_pool(pool, qs, X, mask):
    B, n, D = X.shape
    nh = pool.n_head
    Xd, qd, m8 = X.to(DEV).contiguous(), qs.to(DEV).contiguous(), mask.to(DEV).to(torch.uint8).contiguous()
    pooled = torch.full((B, D), SENTINEL, device=DEV)
    attn = torch.full((nh * B, n), SENTINEL, device=DEV)
    lib = _lib.load()
    st = lib.qagnn_attention_pool(B, n, D, nh, _lib.ptr(Xd), _lib.ptr(qd), _lib.ptr(m8), *_weights(pool), _lib.ptr(pooled),
                                  _lib.ptr(attn), _lib.stream_ptr(torch.device(DEV)))
    _lib.check(st, "qagnn_attention_pool")
    return pooled.cpu(), attn.cpu()


def abi_decoder_tail(pool, qs, X, node_type, lens, sent):
    B, n, D = X.shape
    S, nh = sent.size(1), pool.n_head
    Xd, qd, sd_ = X.to(DEV).contiguous(), qs.to(DEV).contiguous(), sent.to(DEV).contiguous()
    nt, al = node_type.to(DEV).contiguous(), lens.to(DEV).contiguous()
    concat = torch.full((B, 2 * D + S), SENTINEL, device=DEV)
    attn = torch.full((nh * B, n), SENTINEL, device=DEV)
    lib = _lib.load()
    st = lib.qagnn_decoder_tail(B, n, D, nh, S, _lib.ptr(Xd), _lib.ptr(qd), _lib.ptr(nt), _lib.ptr(al), _lib.ptr(sd_),
                                *_weights(pool), _lib.ptr(concat), _lib.ptr(attn), _lib.stream_ptr(torch.device(DEV)))
    _lib.check(st, "qagnn_decoder_tail")
    return concat.cpu(), attn.cpu()


def launches():
    torch.cuda.synchronize()
    return _lib.load().qagnn_launch_count()


def module_forward(pool, q, X, mask):
    """pool.forward on the GPU; returns (pooled, attn, library launches it made)."""
    c0 = launches()
    with torch.no_grad():
        out, attn = pool(q.to(DEV), X.to(DEV), mask.to(DEV))
    return out.cpu(), attn.cpu(), launches() - c0


def module_pool_concat(pool, q, X, node_type, lens):
    c0 = launches()
    with torch.no_grad():
        r = pool.pool_concat(q.to(DEV), X.to(DEV), node_type.to(DEV), lens.to(DEV))
    return (None if r is None else tuple(t.cpu() for t in r)), launches() - c0


def check_tail(concat, attn, ref_pooled, ref_attn, X, sent, what):
    B, n, D = X.shape
    S = sent.size(1)
    assert concat.shape == (B, 2 * D + S) and attn.shape == ref_attn.shape
    assert_attn(attn, ref_attn, f"{what} attn")
    assert_value(concat[:, :D], ref_pooled, f"{what} graph_vecs")
    assert torch.equal(concat[:, D:D + S], sent), f"{what}: sent_vecs not copied bit for bit"
    assert torch.equal(concat[:, D + S:], X[:, 0]), f"{what}: Z = X[:, 0] not copied bit for bit"


# ---------------------------------------------------------------------------------------------------------------------
# 1. explicit-mask pooling
# ---------------------------------------------------------------------------------------------------------------------
# (nh, D, n, B, X scale, mask): every nh in 1..8 the kernel's passes distinguish, dk % 4 != 0 (5, 25) or dk % 32 != 0,
# D = 1024 above 48 KB of shared memory, n around the 4-node and 32-lane steps, B = 600 > 4 CTAs x 132 SMs
POOL_CASES = [
    (1, 8, 1, 7, 1.0, "first"),
    (1, 8, 1000, 7, 3.0, "random"),
    (1, 8, 31, 1, 3.0, "prefix"),
    (2, 200, 33, 600, 1.0, "random"),
    (2, 200, 200, 7, 3.0, "prefix"),
    (3, 96, 31, 600, 3.0, "last"),
    (3, 96, 3, 7, 1.0, "prefix"),
    (4, 64, 33, 7, 1.0, "random"),
    (5, 100, 200, 7, 3.0, "random"),
    (5, 100, 3, 600, 1.0, "first"),
    (8, 200, 1000, 7, 1.0, "random"),
    (8, 200, 31, 600, 3.0, "prefix"),
    (8, 200, 1, 1, 3.0, "first"),
    (8, 200, 33, 600, 1.0, "last"),
    (2, 1024, 200, 7, 1.0, "random"),
    (2, 1024, 1000, 1, 3.0, "last"),
    (4, 1024, 33, 7, 3.0, "prefix"),
    (4, 1024, 1, 1, 1.0, "first"),
]


@pytest.mark.parametrize("nh,D,n,B,scale,mask_kind", POOL_CASES)
def test_attention_pool_matches_fp64(nh, D, n, B, scale, mask_kind):
    S = 48
    g = torch.Generator().manual_seed(nh * 1000 + n + B)
    pool = make_pooler(nh, S, D, seed=n + D).to(DEV)
    q, X = torch.randn(B, S, generator=g), torch.randn(B, n, D, generator=g) * 0.7 * scale
    mask = make_mask(mask_kind, B, n, g)
    # module: w_qs on the GPU, then the fused kernel (one library launch)
    got_out, got_attn, nl = module_forward(pool, q, X, mask)
    assert nl == 1, f"the fused kernel did not run ({nl} launches)"
    ref_out, ref_attn = O.multihead_att_pool(pooler_sd(pool), "pooler", q.double(), X.double(), mask, nh)
    assert_attn(got_attn, ref_attn, "module attn")
    assert_value(got_out, ref_out, "module pooled")
    # C ABI with the query given
    qs = torch.randn(B, D, generator=g)
    got_out, got_attn = abi_attention_pool(pool, qs, X, mask)
    ref_out, ref_attn = ref_pool_given_qs(pool, qs, X, mask)
    assert_attn(got_attn, ref_attn, "abi attn")
    assert_value(got_out, ref_out, "abi pooled")


def test_fully_masked_rows_give_nan_where_the_reference_does():
    """A row with every node masked: the reference's softmax over -inf gives NaN for that graph's attention and pooled
    vector.  The kernel must give NaN at exactly those positions and match everywhere else."""
    nh, D, n, B, S = 3, 96, 33, 7, 48
    g = torch.Generator().manual_seed(5)
    pool = make_pooler(nh, S, D, seed=5).to(DEV)
    q, X = torch.randn(B, S, generator=g), torch.randn(B, n, D, generator=g) * 0.7
    mask = make_mask("random", B, n, g)
    mask[2] = True
    mask[5] = True
    ref_out, ref_attn = O.multihead_att_pool(pooler_sd(pool), "pooler", q.double(), X.double(), mask, nh)
    assert torch.isnan(ref_out[2]).all() and torch.isnan(ref_attn[5::B]).all() and not torch.isnan(ref_out[0]).any()
    got_out, got_attn, nl = module_forward(pool, q, X, mask)
    assert nl == 1
    assert_attn(got_attn, ref_attn, "attn")
    assert_value(got_out, ref_out, "pooled")


# ---------------------------------------------------------------------------------------------------------------------
# 2. tail mode: mask from adj_lengths / node_type, cat(graph_vecs, sent_vecs, Z)
# ---------------------------------------------------------------------------------------------------------------------
TAIL_CASES = [  # (nh, D, n, B, S, X scale)
    (2, 200, 200, 15, 1024, 3.0),
    (1, 8, 1, 15, 8, 1.0),
    (3, 96, 33, 15, 8, 3.0),
    (5, 100, 31, 600, 8, 1.0),
    (8, 200, 1000, 15, 1024, 1.0),
    (4, 1024, 3, 15, 8, 3.0),
    (2, 1024, 257, 15, 1024, 1.0),
]


@pytest.mark.parametrize("nh,D,n,B,S,scale", TAIL_CASES)
def test_decoder_tail_matches_fp64(nh, D, n, B, S, scale):
    g = torch.Generator().manual_seed(nh * 1000 + n + S)
    pool = make_pooler(nh, S, D, seed=n + S).to(DEV)
    sent, X = torch.randn(B, S, generator=g), torch.randn(B, n, D, generator=g) * 0.7 * scale
    lens, node_type = tail_inputs(B, n, g)
    mask = O.decoder_pool_mask(lens, node_type)
    assert not mask.all(1).any()
    # module (pool_concat): w_qs on the GPU, then the fused tail (one library launch)
    r, nl = module_pool_concat(pool, sent, X, node_type, lens)
    assert r is not None and nl == 1
    ref_out, ref_attn = O.multihead_att_pool(pooler_sd(pool), "pooler", sent.double(), X.double(), mask, nh)
    check_tail(*r, ref_out, ref_attn, X, sent, "module")
    # C ABI with the query given; attn head-major [nh * B, n] as the reference lays it out
    qs = torch.randn(B, D, generator=g)
    concat, attn = abi_decoder_tail(pool, qs, X, node_type, lens, sent)
    ref_out, ref_attn = ref_pool_given_qs(pool, qs, X, mask)
    check_tail(concat, attn, ref_out, ref_attn, X, sent, "abi")


# ---------------------------------------------------------------------------------------------------------------------
# 3. head: context node, concept rows, score normalisation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [4, 8, 100, 200, 1024])
@pytest.mark.parametrize("n", [1, 2, 257, 1000])
def test_decoder_head_matches_fp64(n, D):
    B, S, n_concept = 6, 24, 50
    g = torch.Generator().manual_seed(n * 7 + D)
    sd = {"svec2nvec.weight": torch.randn(D, S, generator=g, dtype=F64) / S ** 0.5,
          "svec2nvec.bias": torch.randn(D, generator=g, dtype=F64) * 0.1,
          "concept_emb.emb.weight": torch.randn(n_concept, D, generator=g).double()}  # fp32 values: gathered exactly
    sent = torch.randn(B, S, generator=g, dtype=F64)
    # the kernel's inputs: the fp32 context rows and the table the caller has already projected
    ctx = O.gelu_tanh(O.linear(sent, sd, "svec2nvec")).float()
    table = sd["concept_emb.emb.weight"].float()
    cid = torch.randint(1, n_concept + 1, (B, n), generator=g)
    cid[:, 0] = 0  # the context node's id is never read
    if n > 1:  # both ends of the id range
        cid[0::2, 1] = 1
        cid[1::2, n - 1] = n_concept
    lens = torch.randint(1, n + 4, (B,), generator=g)
    lens[:4] = torch.tensor([0, 1, n, n + 3])
    scores = torch.randn(B, n, generator=g)
    H_out = torch.full((B, n, D), SENTINEL, device=DEV)
    s_out = torch.full((B, n), SENTINEL, device=DEV)
    cd, td, cxd, sc, al = (t.to(DEV).contiguous() for t in (cid, table, ctx, scores, lens))
    st = _lib.load().qagnn_decoder_head(B, n, D, _lib.ptr(cd), n_concept, _lib.ptr(td), _lib.ptr(cxd), _lib.ptr(sc),
                                        _lib.ptr(al), _lib.ptr(H_out), _lib.ptr(s_out), _lib.stream_ptr(torch.device(DEV)))
    _lib.check(st, "qagnn_decoder_head")
    ref_H, ref_s = O.decoder_head(sd, sent, cid, scores.unsqueeze(2).double(), lens, F64)
    H_out, s_out = H_out.cpu(), s_out.cpu()
    assert torch.equal(H_out[:, 0], ctx), "context rows are not bit copies of ctx"
    assert torch.equal(H_out[:, 1:], table[cid[:, 1:] - 1]), "concept rows are not bit copies of the table rows"
    assert torch.equal(H_out, ref_H.float())  # the reference's rows, which are exactly these fp32 values
    assert torch.isnan(ref_s[0]).all() and torch.isnan(s_out[0]).all(), "adj_lengths = 0: the reference's scores are NaN"
    assert_value(s_out, ref_s.squeeze(2), "scores")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the shared-memory boundary
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh,D", [(2, 200), (2, 1024), (8, 512)])
def test_shared_memory_boundary(nh, D):
    """At the largest node count the kernel takes it runs (one launch) and matches fp64; one node more, the module pools
    with its einsum path (no launch) and still matches."""
    nmax = max_pool_len(D, nh)
    assert pool_smem(nmax, D, nh) <= POOL_SMEM_CAP < pool_smem(nmax + 1, D, nh)
    B, S = 2, 16
    g = torch.Generator().manual_seed(nh + D)
    pool = make_pooler(nh, S, D, seed=nh + D).to(DEV)
    q = torch.randn(B, S, generator=g)
    for n, fused in ((nmax, True), (nmax + 1, False)):
        X = torch.randn(B, n, D, generator=g) * 0.7
        lens, node_type = torch.tensor([n, n // 3]), torch.randint(0, 4, (B, n), generator=g)
        mask = O.decoder_pool_mask(lens, node_type)
        ref_out, ref_attn = O.multihead_att_pool(pooler_sd(pool), "pooler", q.double(), X.double(), mask, nh)
        got_out, got_attn, nl = module_forward(pool, q, X, mask)
        assert nl == int(fused), f"n = {n}: {nl} launches"
        assert_attn(got_attn, ref_attn, f"forward attn n={n}")
        assert_value(got_out, ref_out, f"forward pooled n={n}")
        r, nl = module_pool_concat(pool, q, X, node_type, lens)
        assert nl == int(fused) and (r is not None) == fused, f"n = {n}: {nl} launches"
        if fused:
            check_tail(*r, ref_out, ref_attn, X, q, f"pool_concat n={n}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. / 6. regressions: the shared-memory limit both entry points rely on, and fallback after one refused shape
# ---------------------------------------------------------------------------------------------------------------------
def tail_pool_tail_sequence():
    """nh = 2, D = 1024 (81 992 + 8 n bytes of shared memory): the tail at n = 2000, the explicit-mask pool at n = 200,
    the tail at n = 1000, each once.  Returns the worst excess of each call (<= 0 within the bars)."""
    nh, D, S, B = 2, 1024, 32, 2
    g = torch.Generator().manual_seed(11)
    pool = make_pooler(nh, S, D, seed=11).to(DEV)
    sd = pooler_sd(pool)
    q = torch.randn(B, S, generator=g)
    result = []
    for kind, n in (("tail", 2000), ("pool", 200), ("tail", 1000)):
        X = torch.randn(B, n, D, generator=g) * 0.7
        lens, node_type = torch.tensor([n, n // 2]), torch.randint(0, 4, (B, n), generator=g)
        mask = O.decoder_pool_mask(lens, node_type)
        ref_out, ref_attn = O.multihead_att_pool(sd, "pooler", q.double(), X.double(), mask, nh)
        if kind == "tail":
            r, nl = module_pool_concat(pool, q, X, node_type, lens)
            assert r is not None
            out, attn = r[0][:, :D], r[1]
        else:
            out, attn, nl = module_forward(pool, q, X, mask)
        result.append({"call": f"{kind} n={n}", "launches": nl, "attn": attn_excess(attn, ref_attn),
                       "pooled": value_excess(out, ref_out)})
    return result


def test_tail_then_pool_then_tail_in_one_process():
    """Both entry points launch one kernel; a limit set for one must not undercut the other.  Run in a fresh process, so
    that what earlier tests set does not hide the sequence."""
    code = ("import json, sys; sys.path.insert(0, %r); from tests import test_gpu_decoder_head_tail as T; "
            "print(json.dumps(T.tail_pool_tail_sequence()))" % ROOT)
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    calls = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(calls) == 3
    for c in calls:
        assert c["launches"] == 1 and c["attn"] <= 0 and c["pooled"] <= 0, c


@pytest.mark.parametrize("entry", ["forward", "pool_concat"])
def test_a_refused_length_does_not_turn_the_kernel_off(entry):
    """One refused node count sends that length to the einsum path; a shorter batch after it still runs the kernel."""
    nh, D, S, B = 8, 512, 16, 2
    g = torch.Generator().manual_seed(12)
    pool = make_pooler(nh, S, D, seed=12).to(DEV)
    sd = pooler_sd(pool)
    q = torch.randn(B, S, generator=g)
    for n, fused in ((max_pool_len(D, nh) + 1, False), (200, True)):
        X = torch.randn(B, n, D, generator=g) * 0.7
        lens, node_type = torch.tensor([n, n // 2]), torch.randint(0, 4, (B, n), generator=g)
        mask = O.decoder_pool_mask(lens, node_type)
        ref_out, ref_attn = O.multihead_att_pool(sd, "pooler", q.double(), X.double(), mask, nh)
        if entry == "forward":
            out, attn, nl = module_forward(pool, q, X, mask)
        else:
            r, nl = module_pool_concat(pool, q, X, node_type, lens)
            assert (r is not None) == fused
            if r is None:  # the caller pools with forward, which the other parameter checks
                assert nl == 0
                continue
            out, attn = r[0][:, :D], r[1]
        assert nl == int(fused), f"n = {n}: {nl} launches, expected {int(fused)}"
        assert_attn(attn, ref_attn, f"attn n={n}")
        assert_value(out, ref_out, f"pooled n={n}")


# ---------------------------------------------------------------------------------------------------------------------
# 7. the bars are sharp
# ---------------------------------------------------------------------------------------------------------------------
def test_bars_detect_an_open_masked_node_swapped_heads_and_a_perturbed_value_weight():
    nh, D, n, B, S = 4, 200, 33, 7, 48
    g = torch.Generator().manual_seed(13)
    pool = make_pooler(nh, S, D, seed=13).to(DEV)
    q, X = torch.randn(B, S, generator=g), torch.randn(B, n, D, generator=g) * 2.1
    mask = make_mask("random", B, n, g)
    sd = pooler_sd(pool)
    got_out, got_attn, nl = module_forward(pool, q, X, mask)
    assert nl == 1
    ref_out, ref_attn = O.multihead_att_pool(sd, "pooler", q.double(), X.double(), mask, nh)
    assert attn_excess(got_attn, ref_attn) <= 0 and value_excess(got_out, ref_out) <= 0
    # a reference with one masked node left open
    m2 = mask.clone()
    b, i = (int(v) for v in mask.nonzero()[0])
    m2[b, i] = False
    o2, a2 = O.multihead_att_pool(sd, "pooler", q.double(), X.double(), m2, nh)
    assert attn_excess(got_attn, a2) > 0 and value_excess(got_out, o2) > 0
    # heads 0 and 1 swapped
    dk = D // nh
    perm = torch.tensor([1, 0, 2, 3])
    assert attn_excess(got_attn, ref_attn.view(nh, B, n)[perm].reshape(nh * B, n)) > 0
    assert value_excess(got_out, ref_out.view(B, nh, dk)[:, perm].reshape(B, D)) > 0
    # one column of w_vs moved by 1e-3
    sd3 = dict(sd)
    sd3["pooler.w_vs.weight"] = sd["pooler.w_vs.weight"].clone()
    sd3["pooler.w_vs.weight"][:, 17] += 1e-3
    o3, _ = O.multihead_att_pool(sd3, "pooler", q.double(), X.double(), mask, nh)
    assert value_excess(got_out, o3) > 0


# ---------------------------------------------------------------------------------------------------------------------
# the whole decoder through the module API (fused head and tail) against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_decoder_module_with_five_pool_heads_matches_fp64():
    import qagnn_b200
    B, n, e, D, k, S, n_concept, nh = 6, 40, 120, 100, 1, 40, 300, 5
    inp = O.synth_graph_batch(B, n, e, D, 38, seed=21, realistic=True)
    g = torch.Generator().manual_seed(21)
    lens = inp["adj_lengths"].clone()
    lens[:3] = torch.tensor([1, n, n + 5])
    node_type = inp["node_type"].clone()
    node_type[3, :int(lens[3])] = 3
    sent = torch.randn(B, S, generator=g)
    cid = torch.randint(1, n_concept + 1, (B, n), generator=g)
    cid[0, 1], cid[1, 1] = 1, n_concept
    torch.manual_seed(21)
    dec = qagnn_b200.QAGNN(None, k, 4, 38, S, n_concept, D, 32, nh, D, 1, 0.2, 0.2, 0.2, init_range=0).eval()
    sd = {kk: v.detach().clone() for kk, v in dec.state_dict().items()}
    ref_logits, ref_attn, _ = O.qagnn_decoder_forward(sd, sent, cid, node_type, inp["node_score"], lens, inp["edge_index"],
                                                      inp["edge_type"], k, 4, 38, nh, 1, dtype=F64)
    dec = dec.to(DEV)
    args = (sent.to(DEV), cid.to(DEV), node_type.to(DEV), inp["node_score"].to(DEV), lens.to(DEV),
            (inp["edge_index"].to(DEV), inp["edge_type"].to(DEV)))
    with torch.no_grad():
        logits, attn = dec(*args)  # fused head, message passing, fused tail
    Hh.assert_close(attn, ref_attn, "pool_attn")
    Hh.assert_close(logits, ref_logits, "logits")
