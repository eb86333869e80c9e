"""The ragged decoder's two ends against fp64: qagnn_decoder_head_ragged (decoder_head_ragged_kernel), the ragged tail
qagnn_decoder_tail_ragged (attention_pool_kernel<XT, true>) and its backward qagnn_attention_pool_backward_ragged
(pool_backward_head_kernel, pool_backward_rows_kernel, pool_backward_weights_kernel), all in qagnn_b200/csrc/pool.cu.

One case table, every entry run through the tail forward and the backward.  Across its rows it takes every head count 1..8
(the forward's passes of four heads), head widths that are not a multiple of 4 or of 32, D under one 128-column step, over
one and over two, node counts around the 4-node, 32-lane and 256-thread steps (n = 255, 256, 257, 1000 run the backward's
thread-stride loops), S = 0 (the C entries only), odd and 1024, one graph and hundreds, X in fp32 and bf16, and every length edge: length 1,
length n and more, a graph of context nodes only (node 0 kept), a batch that ends exactly at the node capacity, tail rows
fewer and more than the graphs (the head kernel's r += B loop), and graphs that own rows past their length.

References (tests/ragged_pool_oracle.py, fp64 on the CPU): the forward re-padded through the folded pooling with the padded
test's bars (tests/test_gpu_decoder_head_tail.py); the backward's closed form with a magnitude bar per element, on exactly
the kernel's inputs; the head through O.decoder_head.  Outputs start as a sentinel, so an element never written fails.
Needs a GPU: run with -m gpu."""
import collections

import pytest
import torch

from oracle import qagnn_oracle as O
from qagnn_b200 import _lib
from qagnn_b200.layers import MultiheadAttPoolLayer
from tests import ragged_pool_oracle as RP
from tests.test_gpu_decoder_head_tail import assert_attn, assert_value, attn_excess, value_excess

pytestmark = pytest.mark.gpu

F64 = torch.float64
DEV = "cuda:0"
SENTINEL = 3.0e38
UNSUPPORTED = -5
POOL_SMEM_CAP = 200 * 1024  # kPoolSmemCap, qagnn_b200/csrc/pool.cu


def pool_smem(n, D, nh):
    """pool_smem_bytes of pool.cu: the forward's dynamic shared memory."""
    return (2 * nh * D + nh * n + nh + 16 + 8 * nh * D) * 4


def pool_bwd_smem(D):
    """pool_backward_smem_bytes of pool.cu: qk, dxs, dqk [D] and 8 warps' partial sums."""
    return (3 * D + 8) * 4


def max_pool_len(D, nh):
    """The largest node count the ragged forward (and so the backward) takes at (D, nh); < 1 when it takes none."""
    return (POOL_SMEM_CAP // 4 - 10 * nh * D - nh - 16) // nh


# ---------------------------------------------------------------------------------------------------------------------
# the case table
# ---------------------------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", "name nh D n B S xdtype tail slack")
f32, bf16 = torch.float32, torch.bfloat16
TAIL_CASES = [
    Case("one graph of one node, S = 0, D under a column step", 1, 8, 1, 1, 0, f32, "many", 0),
    Case("dk = 100: 32-lane remainder, D over one column step, odd S, n = 257", 2, 200, 257, 40, 33, f32, "few", 0),
    Case("dk = 5, 600 graphs of n = 5, bf16", 3, 15, 5, 600, 7, bf16, "many", 0),
    Case("dk = 25, n = 256, S = 1024, batch ends at the capacity", 4, 100, 256, 9, 1024, f32, "none", 0),
    Case("five heads (second pass), D over two column steps, n = 1000, bf16", 5, 320, 1000, 6, 1, bf16, "few", 0),
    Case("six heads, dk = 16, n = 2, rows past the lengths", 6, 96, 2, 33, 0, f32, "many", 1),
    Case("seven heads, dk = 40, n = 255, batch ends at the capacity", 7, 280, 255, 12, 5, f32, "none", 0),
    Case("eight heads, dk = 25, n = 3, bf16", 8, 200, 3, 200, 16, bf16, "few", 0),
    Case("four heads, dk = 256, D = 1024 (over 48 KB of shared memory), n = 4", 4, 1024, 4, 3, 1024, f32, "many", 0),
    Case("one head, n = 1000, rows past the lengths", 1, 100, 1000, 5, 9, f32, "few", 7),
    Case("two heads, dk = 32, n = 257, bf16, one graph", 2, 64, 257, 1, 3, bf16, "none", 0),
]


def tail_rows(c):
    return {"none": 0, "few": max(1, c.B // 2), "many": 2 * c.B + 3}[c.tail]


def lengths_and_types(c):
    """adj_lengths cycling over 1, n, n + 5 and random values (graph 0 of a single-graph batch has length n), and padded node
    types with node 0 a context node; every third graph from graph 2 on has only context nodes within its length."""
    g = torch.Generator().manual_seed(c.nh * 7919 + c.D * 31 + c.n + c.B)
    lens = torch.randint(1, c.n + 1, (c.B,), generator=g)
    for b, v in zip(range(min(c.B, 4)), (c.n, 1, c.n + 5, 1)):
        lens[b] = v
    nt = torch.randint(0, 4, (c.B, c.n), generator=g)
    nt[:, 0] = 3
    for b in range(2, c.B, 3):
        nt[b] = 3
    return lens, nt


def make_inputs(c):
    """Everything one case runs on: the pooler (weights in fp32), the ragged layout and its packed tensors, the padded
    references' inputs, and a random dconcat."""
    lens, nt = lengths_and_types(c)
    g = torch.Generator().manual_seed(c.B * 13 + c.n)
    torch.manual_seed(c.n + c.D)
    pool = MultiheadAttPoolLayer(c.nh, c.S, c.D).eval()
    with torch.no_grad():
        for p in (pool.w_ks.bias, pool.w_vs.bias):
            p.normal_(0, 0.5, generator=g)
    node_ptr, N_cap, rows = RP.ragged_layout(lens, c.n, tail_rows(c), c.slack)
    X = (torch.randn(c.B, c.n, c.D, generator=g) * 1.5).to(c.xdtype)
    tail = (torch.randn(N_cap - rows.numel(), c.D, generator=g) * 1.5).to(c.xdtype)
    Xp = RP.pack(X, rows, N_cap, tail)
    ntp = RP.pack(nt.unsqueeze(-1), rows, N_cap).squeeze(-1)
    ntp[rows.numel():] = 2
    valid = torch.arange(c.n) < lens.clamp(max=c.n).unsqueeze(1)
    X64 = torch.where(valid.unsqueeze(-1), X.double(), 0.0)  # the reference's padded X: zero past each length
    return {"pool": pool, "lens": lens, "nt": nt, "node_ptr": node_ptr, "N_cap": N_cap, "rows": rows, "X": X, "Xp": Xp,
            "ntp": ntp, "valid": valid, "X64": X64, "mask": RP.tail_mask(lens, nt),
            "qs": torch.randn(c.B, c.D, generator=g), "sent": torch.randn(c.B, c.S, generator=g),
            "dconcat": torch.randn(c.B, 2 * c.D + c.S, generator=g)}


def weights(pool):
    return [t.detach().cpu() for t in (pool.w_ks.weight, pool.w_ks.bias, pool.w_vs.weight, pool.w_vs.bias)]


def launches():
    torch.cuda.synchronize()
    return _lib.load().qagnn_launch_count()


# ---------------------------------------------------------------------------------------------------------------------
# the C entry points
# ---------------------------------------------------------------------------------------------------------------------
def _d(*ts):
    return [t.to(DEV).contiguous() for t in ts]


def _sent(sent):
    """sent_vecs on the device; at S = 0 a one-element buffer, as the entry points refuse a null pointer (nothing is read)."""
    return sent.to(DEV).contiguous() if sent.numel() else torch.zeros(1, device=DEV)


def abi_tail_ragged(nh, n, Xp, node_ptr, qs, ntp, lens, sent, w, status=False):
    """(concat [B, 2D + S], attn [nh * B, n]) of qagnn_decoder_tail_ragged, or its status when `status`."""
    B, (N_cap, D), S = lens.numel(), Xp.shape, sent.size(1)
    Xd, npd, qd, ntd, ld = _d(Xp, node_ptr, qs, ntp, lens)
    sd_, wd = _sent(sent), _d(*w)
    concat = torch.full((B, 2 * D + S), SENTINEL, device=DEV)
    attn = torch.full((nh * B, n), SENTINEL, device=DEV)
    st = _lib.load().qagnn_decoder_tail_ragged(_lib.DTYPE_CODES[Xp.dtype], B, n, D, nh, S, N_cap, _lib.ptr(Xd), _lib.ptr(npd),
                                               _lib.ptr(qd), _lib.ptr(ntd), _lib.ptr(ld), _lib.ptr(sd_), *map(_lib.ptr, wd),
                                               _lib.ptr(concat), _lib.ptr(attn), _lib.stream_ptr(torch.device(DEV)))
    if status:
        return st
    _lib.check(st, "qagnn_decoder_tail_ragged")
    return concat.cpu(), attn.cpu()


def abi_tail_padded(nh, X, qs, nt, lens, sent, w):
    B, n, D = X.shape
    S = sent.size(1)
    Xd, qd, ntd, ld = _d(X, qs, nt, lens)
    sd_, wd = _sent(sent), _d(*w)
    concat = torch.full((B, 2 * D + S), SENTINEL, device=DEV)
    attn = torch.full((nh * B, n), SENTINEL, device=DEV)
    st = _lib.load().qagnn_decoder_tail_typed(_lib.DTYPE_CODES[X.dtype], B, n, D, nh, S, _lib.ptr(Xd), _lib.ptr(qd), _lib.ptr(ntd),
                                              _lib.ptr(ld), _lib.ptr(sd_), *map(_lib.ptr, wd), _lib.ptr(concat), _lib.ptr(attn),
                                              _lib.stream_ptr(torch.device(DEV)))
    _lib.check(st, "qagnn_decoder_tail_typed")
    return concat.cpu(), attn.cpu()


def abi_backward(nh, n, S, Xp, node_ptr, lens, qs, w, attn, dconcat, status=False):
    """{dX, dqs, dwk, dbk, dwv, dbv} of qagnn_attention_pool_backward_ragged (every output a sentinel first), or its status."""
    B, (N_cap, D) = lens.numel(), Xp.shape
    Xd, npd, ld, qd, ad, gd = _d(Xp, node_ptr, lens, qs, attn, dconcat)
    wk, bk, wv, _ = _d(*w)
    out = {"dX": torch.full((N_cap, D), SENTINEL, device=DEV), "dqs": torch.full((B, D), SENTINEL, device=DEV),
           "dwk": torch.full((D, D), SENTINEL, device=DEV), "dbk": torch.full((D,), SENTINEL, device=DEV),
           "dwv": torch.full((D, D), SENTINEL, device=DEV), "dbv": torch.full((D,), SENTINEL, device=DEV)}
    lib = _lib.load()
    nbytes = lib.qagnn_attention_pool_backward_ragged_scratch_bytes(B, n, D, nh)
    scratch = torch.full((max(nbytes // 4, 1),), SENTINEL, device=DEV)
    st = lib.qagnn_attention_pool_backward_ragged(_lib.DTYPE_CODES[Xp.dtype], B, n, D, nh, S, N_cap, _lib.ptr(Xd), _lib.ptr(npd),
                                                  _lib.ptr(ld), _lib.ptr(qd), _lib.ptr(wk), _lib.ptr(bk), _lib.ptr(wv), _lib.ptr(ad),
                                                  _lib.ptr(gd), *(_lib.ptr(out[k]) for k in ("dX", "dqs", "dwk", "dbk", "dwv", "dbv")),
                                                  _lib.ptr(scratch), nbytes, _lib.stream_ptr(torch.device(DEV)))
    if status:
        return st
    _lib.check(st, "qagnn_attention_pool_backward_ragged")
    return {k: v.cpu() for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------------------------
# checks shared by the table and the limit rows
# ---------------------------------------------------------------------------------------------------------------------
def check_forward(c, inp, concat, attn, what):
    """concat / attn of the ragged tail against the fp64 folded pooling, the copies bit for bit, attn 0 past the lengths."""
    D, S, nh, n = c.D, c.S, c.nh, c.n
    ref_p, ref_a = RP.pool_forward(inp["qs"], inp["X64"], inp["mask"], *weights(inp["pool"]), nh)
    assert_attn(attn, ref_a, f"{what} attn")
    assert_value(concat[:, :D], ref_p, f"{what} graph_vecs")
    assert torch.equal(concat[:, D:D + S], inp["sent"]), f"{what}: sent_vecs not copied bit for bit"
    Z = inp["Xp"][inp["node_ptr"][:-1]].float()
    assert torch.equal(concat[:, D + S:], Z), f"{what}: Z is not each graph's first packed row, bit for bit"
    past = ~inp["valid"].repeat(nh, 1)
    assert bool((attn[past] == 0).all()), f"{what}: attention past a graph's length is not exactly 0"


def backward_ref(c, inp, attn, qs=None, dconcat=None):
    return RP.pool_backward(inp["qs"] if qs is None else qs, inp["X64"], attn, inp["dconcat"] if dconcat is None else dconcat,
                            *weights(inp["pool"])[:3], c.nh, c.S, n_rows=int(inp["lens"].clamp(max=c.n).max()))


def backward_excess(got, ref, inp, B, n):
    """{name: excess over the bar}; dX compared on the re-padded layout of the rows that hold a graph's node."""
    rows, valid = inp["rows"], inp["valid"]
    ex = {}
    for k in ("dqs", "dwk", "dbk", "dwv", "dbv"):
        ex[k] = RP.excess(got[k], *ref[k])
    dXg = RP.repad(got["dX"].double(), rows, B, n)
    ex["dX"] = RP.excess(dXg[valid], ref["dX"][0][valid], ref["dX"][1][valid])
    return ex


def check_backward(c, inp, got, ref, what):
    ex = backward_excess(got, ref, inp, c.B, c.n)
    bad = {k: v for k, v in ex.items() if v > 0}
    assert not bad, f"{what}: outside the magnitude bars by {bad}"
    # softmax is shift invariant: the key bias's gradient is zero up to rounding, and so within its bar of 0
    assert bool((got["dbk"].double().abs() <= ref["dbk"][1]).all()), f"{what}: dL/db_k is not within its bar of 0"
    # the tail rows and the rows a graph owns past its length get exactly 0
    nv = int(inp["node_ptr"][-1])
    pos, gb = inp["rows"] % c.n, inp["rows"] // c.n
    past = (pos >= inp["lens"].clamp(max=c.n)[gb]).nonzero().squeeze(-1)
    assert bool((got["dX"][nv:] == 0).all()), f"{what}: a tail row got a gradient"
    assert bool((got["dX"][past] == 0).all()), f"{what}: a row past a graph's length got a gradient"


# ---------------------------------------------------------------------------------------------------------------------
# 1. the table: tail forward and backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", TAIL_CASES, ids=[c.name for c in TAIL_CASES])
def test_ragged_tail_forward_and_backward_match_fp64(c):
    inp = make_inputs(c)
    w = weights(inp["pool"])
    args = (inp["Xp"], inp["node_ptr"], inp["qs"], inp["ntp"], inp["lens"], inp["sent"], w)
    concat, attn = abi_tail_ragged(c.nh, c.n, *args)
    check_forward(c, inp, concat, attn, "forward")
    # DESIGN §5.5: the padded tail on the re-padded batch gives the same bits.  The padded rows past each length hold finite
    # random values, so the equality shows they get weight exactly 0.
    fill = (torch.randn(c.B, c.n, c.D, generator=torch.Generator().manual_seed(c.n)) * 4).to(c.xdtype)
    Xpad = RP.repad(inp["Xp"], inp["rows"], c.B, c.n, fill)
    Xpad = torch.where(inp["valid"].unsqueeze(-1), Xpad, fill)
    pc, pa = abi_tail_padded(c.nh, Xpad, inp["qs"], inp["nt"], inp["lens"], inp["sent"], w)
    assert torch.equal(concat, pc) and torch.equal(attn, pa), "the ragged tail is not the padded tail bit for bit"

    got = abi_backward(c.nh, c.n, c.S, inp["Xp"], inp["node_ptr"], inp["lens"], inp["qs"], w, attn, inp["dconcat"])
    ref = backward_ref(c, inp, attn)
    check_backward(c, inp, got, ref, "backward")
    again = abi_backward(c.nh, c.n, c.S, inp["Xp"], inp["node_ptr"], inp["lens"], inp["qs"], w, attn, inp["dconcat"])
    for k in got:
        assert torch.equal(got[k], again[k]), f"{k} differs between two runs"

    # dZ alone: dX is dZ on each graph's first row, bit for bit, and zero everywhere else
    dz = torch.zeros_like(inp["dconcat"])
    dz[:, c.D + c.S:] = inp["dconcat"][:, c.D + c.S:]
    gz = abi_backward(c.nh, c.n, c.S, inp["Xp"], inp["node_ptr"], inp["lens"], inp["qs"], w, attn, dz)
    want = torch.zeros(inp["N_cap"], c.D)
    want[inp["node_ptr"][:-1]] = dz[:, c.D + c.S:]
    assert torch.equal(gz["dX"], want), "dZ does not land on each graph's row 0 alone"

    # the graphs in another order: dX rows and dqs permute bit for bit
    if c.B > 1:
        perm = torch.randperm(c.B, generator=torch.Generator().manual_seed(c.B))
        counts = inp["node_ptr"].diff()
        pnp = torch.zeros(c.B + 1, dtype=torch.long)
        pnp[1:] = counts[perm].cumsum(0)
        src = torch.cat([torch.arange(int(inp["node_ptr"][b]), int(inp["node_ptr"][b + 1])) for b in perm.tolist()])
        nv = int(inp["node_ptr"][-1])
        pXp = torch.cat([inp["Xp"][src], inp["Xp"][nv:]])
        pnt = torch.cat([inp["ntp"][src], inp["ntp"][nv:]])
        pc2, pa2 = abi_tail_ragged(c.nh, c.n, pXp, pnp, inp["qs"][perm], pnt, inp["lens"][perm], inp["sent"][perm], w)
        assert torch.equal(pa2.view(c.nh, c.B, c.n), attn.view(c.nh, c.B, c.n)[:, perm])
        gp = abi_backward(c.nh, c.n, c.S, pXp, pnp, inp["lens"][perm], inp["qs"][perm], w, pa2, inp["dconcat"][perm])
        assert torch.equal(gp["dX"][:nv], got["dX"][src]), "permuting the graphs does not permute dX bit for bit"
        assert torch.equal(gp["dqs"], got["dqs"][perm]), "permuting the graphs does not permute dqs bit for bit"


MODULE_CASES = [c for c in TAIL_CASES if c.S > 0]  # the module's w_qs needs a query of at least one feature


@pytest.mark.parametrize("c", MODULE_CASES, ids=[c.name for c in MODULE_CASES])
def test_pool_concat_ragged_module_matches_the_c_entry(c):
    """pool_concat_ragged (w_qs on the GPU, then the ragged tail, differentiable through qagnn_attention_pool_backward_ragged)
    gives the C entry's values on the same qs, and gradients within the closed form's bars; a bf16 k gets a bf16 gradient
    within the bar plus half a bf16 ulp."""
    inp = make_inputs(c)
    pool = inp["pool"].to(DEV)
    sent, Xp = inp["sent"].to(DEV).requires_grad_(True), inp["Xp"].to(DEV).requires_grad_(True)
    concat, attn = pool.pool_concat_ragged(sent, Xp, inp["node_ptr"].to(DEV), inp["ntp"].to(DEV), inp["lens"].to(DEV), c.n)
    (concat * inp["dconcat"].to(DEV)).sum().backward()
    with torch.no_grad():
        qs = pool.w_qs(sent).float().cpu()
    inp["qs"] = qs
    w = [t.cpu() for t in weights(pool)]
    c2, a2 = abi_tail_ragged(c.nh, c.n, inp["Xp"], inp["node_ptr"], qs, inp["ntp"], inp["lens"], inp["sent"], w)
    assert torch.equal(concat.detach().cpu(), c2) and torch.equal(attn.cpu(), a2)
    assert Xp.grad.dtype == c.xdtype
    ref = backward_ref(c, inp, a2)
    dX = RP.repad(Xp.grad.cpu().double(), inp["rows"], c.B, c.n)[inp["valid"]]
    r, b = ref["dX"][0][inp["valid"]], ref["dX"][1][inp["valid"]]
    half_ulp = 0.0 if c.xdtype == f32 else 2.0 ** -8 * r.abs()
    assert RP.excess(dX, r, b + half_ulp) <= 0, "dL/dk outside the bar"
    for name, p in (("dwk", pool.w_ks.weight), ("dbk", pool.w_ks.bias), ("dwv", pool.w_vs.weight), ("dbv", pool.w_vs.bias)):
        assert RP.excess(p.grad, *ref[name]) <= 0, f"{name} outside the bar"
    # dL/dsent = w_qs^T dqs + the gradient of the copied sent_vecs
    want = ref["dqs"][0] @ pool.w_qs.weight.detach().double().cpu() + inp["dconcat"][:, c.D:c.D + c.S].double()
    mag = ref["mag"]["dqs"] @ pool.w_qs.weight.detach().double().abs().cpu() + inp["dconcat"][:, c.D:c.D + c.S].double().abs()
    assert RP.excess(sent.grad, want, RP.bar(mag, 4 * c.D + 2 * c.n + 8)) <= 0, "dL/dsent_vecs outside the bar"


def test_fp16_k_is_widened_exactly():
    """An fp16 k (the autograd decoder under fp16 autocast) runs the fp32 kernels on its exact widening: the same values as
    an fp32 k holding them, and its gradient is that gradient rounded to fp16."""
    c = TAIL_CASES[1]
    inp = make_inputs(c)
    pool = inp["pool"].to(DEV)
    res = []
    for dt in (torch.float16, torch.float32):
        pool.zero_grad(set_to_none=True)
        k = inp["Xp"].half().to(dt).to(DEV).requires_grad_(True)
        concat, attn = pool.pool_concat_ragged(inp["sent"].to(DEV), k, inp["node_ptr"].to(DEV), inp["ntp"].to(DEV),
                                               inp["lens"].to(DEV), c.n)
        (concat * inp["dconcat"].to(DEV)).sum().backward()
        res.append((concat.detach(), attn, k.grad, pool.w_ks.weight.grad.clone(), pool.w_vs.weight.grad.clone()))
    (c16, a16, g16, wk16, wv16), (c32, a32, g32, wk32, wv32) = res
    assert g16.dtype == torch.float16 and torch.equal(g16, g32.half())
    assert torch.equal(c16, c32) and torch.equal(a16, a32) and torch.equal(wk16, wk32) and torch.equal(wv16, wv32)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the bars reject perturbed references
# ---------------------------------------------------------------------------------------------------------------------
def test_bars_reject_perturbed_references():
    c = TAIL_CASES[1]  # nh = 2, D = 200, n = 257, 40 graphs
    inp = make_inputs(c)
    w = weights(inp["pool"])
    concat, attn = abi_tail_ragged(c.nh, c.n, inp["Xp"], inp["node_ptr"], inp["qs"], inp["ntp"], inp["lens"], inp["sent"], w)
    got = abi_backward(c.nh, c.n, c.S, inp["Xp"], inp["node_ptr"], inp["lens"], inp["qs"], w, attn, inp["dconcat"])
    ref = backward_ref(c, inp, attn)
    assert max(backward_excess(got, ref, inp, c.B, c.n).values()) <= 0
    D, nh, dk, B, n = c.D, c.nh, c.D // c.nh, c.B, c.n

    def rejects(r, names):
        ex = backward_excess(got, r, inp, B, n)
        for k in names:
            assert ex[k] > 0, f"{k}: the perturbed reference passes ({ex[k]:.3e})"

    # one graph's last valid node (an open one, with weight in every head) dropped from the node sums xs and dqk
    A = attn.view(nh, B, n)
    b = next(b for b in range(B) if int(inp["lens"][b]) > 8 and bool((A[:, b, min(int(inp["lens"][b]), n) - 1] > 0).all()))
    last = min(int(inp["lens"][b]), n) - 1
    X2 = inp["X64"].clone()
    X2[b, last] = 0
    inp2 = dict(inp, X64=X2)
    r = backward_ref(c, inp2, attn)
    rejects(r, ["dwv", "dwk", "dqs"])
    # sdot omitted from the logit gradient: g_i = a_i da_i / sqrt(dk)
    parts = ref["parts"]
    a = attn.double().view(nh, B, n).permute(1, 0, 2)
    da = torch.einsum("bhj,bij->bhi", parts["dxs"], inp["X64"])
    g_bad = a * da / dk ** 0.5
    dX_bad = torch.einsum("bhi,bhj->bij", a, parts["dxs"]) + torch.einsum("bhi,bhj->bij", g_bad, parts["qk"])
    dX_bad[:, 0] += inp["dconcat"][:, D + c.S:].double()
    rejects(dict(ref, dX=(dX_bad, ref["dX"][1])), ["dX"])
    # dZ added to row 1 as well as row 0
    dX_z = ref["dX"][0].clone()
    dX_z[:, 1] += inp["dconcat"][:, D + c.S:].double()
    rejects(dict(ref, dX=(dX_z, ref["dX"][1])), ["dX"])
    # heads 0 and 1 swapped
    sw = lambda t, dim: torch.cat([t.narrow(dim, dk, dk), t.narrow(dim, 0, dk)], dim)
    rejects(dict(ref, dqs=(sw(ref["dqs"][0], 1), ref["dqs"][1]), dwv=(sw(ref["dwv"][0], 0), ref["dwv"][1])), ["dqs", "dwv"])
    # one graph left out of the dW_v sum
    dp = inp["dconcat"][:, :D].double().view(B, nh, dk)
    dwv_bad = ref["dwv"][0] - torch.einsum("hr,hj->hrj", dp[b], parts["xs"][b]).reshape(D, D)
    rejects(dict(ref, dwv=(dwv_bad, ref["dwv"][1])), ["dwv"])
    # a ragged reference one row off: every graph's rows read from one row later
    Xoff = RP.repad(torch.cat([inp["Xp"][1:], inp["Xp"][:1]]).double(), inp["rows"], B, n)
    Xoff = torch.where(inp["valid"].unsqueeze(-1), Xoff, 0.0)
    r = backward_ref(c, dict(inp, X64=Xoff), attn)
    rejects(r, ["dX", "dqs", "dwk", "dwv"])
    ref_p, ref_a = RP.pool_forward(inp["qs"], Xoff, inp["mask"], *w, nh)
    assert attn_excess(attn, ref_a) > 0 and value_excess(concat[:, :D], ref_p) > 0


# ---------------------------------------------------------------------------------------------------------------------
# 3. the shared-memory limits: at the forward's largest n both directions run; one node more, both refuse before a launch
# ---------------------------------------------------------------------------------------------------------------------
# each head count takes the largest multiple of itself at or below these; at D = 4800 the backward needs 56 KB (its opt-in)
LIMIT_DS = (200, 1024, 4800)


def limit_D(D, nh):
    return D - D % nh


LIMIT_CASES = []  # (nh, D, n, accepted)
for _nh in range(1, 9):
    for _D in (limit_D(D, _nh) for D in LIMIT_DS):
        _m = max_pool_len(_D, _nh)
        LIMIT_CASES += [(_nh, _D, _m, True), (_nh, _D, _m + 1, False)] if _m >= 1 else [(_nh, _D, 1, False)]


@pytest.mark.parametrize("nh,D,n,accepted", LIMIT_CASES, ids=[f"nh{r[0]}-D{r[1]}-n{r[2]}" for r in LIMIT_CASES])
def test_shared_memory_limits(nh, D, n, accepted):
    c = Case("limit", nh, D, n, 1, 3, f32, "few", 0)  # one graph of length n and one tail row
    lens = torch.tensor([n])
    g = torch.Generator().manual_seed(nh * 10 + D)
    nt = torch.randint(0, 3, (1, n), generator=g)
    nt[:, 0] = 3
    node_ptr, N_cap, rows = RP.ragged_layout(lens, n, tail_rows(c))
    Xp = torch.randn(N_cap, D, generator=g)
    ntp = RP.pack(nt.unsqueeze(-1), rows, N_cap).squeeze(-1)
    torch.manual_seed(nh + D)
    pool = MultiheadAttPoolLayer(nh, 3, D).eval()
    w = weights(pool)
    qs, sent, dconcat = torch.randn(1, D, generator=g), torch.randn(1, 3, generator=g), torch.randn(1, 2 * D + 3, generator=g)
    if not accepted:
        c0 = launches()
        st_f = abi_tail_ragged(nh, n, Xp, node_ptr, qs, ntp, lens, sent, w, status=True)
        attn = torch.zeros(nh, n)
        st_b = abi_backward(nh, n, 3, Xp, node_ptr, lens, qs, w, attn, dconcat, status=True)
        assert st_f == UNSUPPORTED and st_b == UNSUPPORTED, (st_f, st_b)
        assert launches() == c0, "a refused shape launched a kernel"
        return
    valid = torch.arange(n) < lens.unsqueeze(1)
    X64 = torch.zeros(1, n, D, dtype=F64)
    X64[valid] = Xp[:rows.numel()].double()
    inp = {"pool": pool, "lens": lens, "nt": nt, "node_ptr": node_ptr, "N_cap": N_cap, "rows": rows, "Xp": Xp, "ntp": ntp,
           "valid": valid, "X64": X64, "mask": RP.tail_mask(lens, nt), "qs": qs, "sent": sent, "dconcat": dconcat}
    concat, attn = abi_tail_ragged(nh, n, Xp, node_ptr, qs, ntp, lens, sent, w)
    check_forward(c, inp, concat, attn, f"forward n={n}")
    got = abi_backward(nh, n, 3, Xp, node_ptr, lens, qs, w, attn, dconcat)
    check_backward(c, inp, got, backward_ref(c, inp, attn), f"backward n={n}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the ragged head
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [4, 8, 100, 200, 1024])
@pytest.mark.parametrize("n", [1, 2, 257, 1000])
def test_ragged_head_matches_fp64_and_the_grad_mode_head(n, D):
    import qagnn_b200
    B, S, n_concept = 7, 24, 50
    g = torch.Generator().manual_seed(n * 7 + D)
    torch.manual_seed(n + D)
    dec = qagnn_b200.QAGNN(None, 1, 4, 38, S, n_concept, D, D, 1, 8, 0, 0.0, 0.0, 0.0).eval()
    sent = torch.randn(B, S, generator=g)
    cid = torch.randint(1, n_concept + 1, (B, n), generator=g)
    cid[:, 0] = 0  # the context node's id is never read
    if n > 1:
        cid[0, 1], cid[1, n - 1] = 1, n_concept  # both ends of the table
    lens = torch.randint(1, n + 1, (B,), generator=g)
    lens[:4] = torch.tensor([1, n, n + 3, n + 50])  # adj_lengths past n
    scores = torch.randn(B, n, generator=g)
    nt = torch.randint(0, 4, (B, n), generator=g)
    tails = 2 * B + 5  # more tail rows than graphs: CTA b clears rows node_ptr[B] + b, + B, + 2B
    node_ptr, N_cap, rows = RP.ragged_layout(lens, n, tails)
    dec = dec.to(DEV)

    def run(ids):
        with torch.no_grad():
            ctx = dec.activation(dec.svec2nvec(sent.to(DEV))).float().contiguous()
            table = dec.concept_emb.projected_table()
        H = torch.full((N_cap, D), SENTINEL, device=DEV)
        s = torch.full((N_cap,), SENTINEL, device=DEV)
        t = torch.full((N_cap,), -7, dtype=torch.long, device=DEV)
        cd, sd_, ld, ntd, npd = _d(ids, scores, lens, nt, node_ptr)
        st = _lib.load().qagnn_decoder_head_ragged(B, n, D, N_cap, _lib.ptr(cd), table.size(0), _lib.ptr(table), _lib.ptr(ctx),
                                                   _lib.ptr(sd_), _lib.ptr(ld), _lib.ptr(ntd), _lib.ptr(npd), _lib.ptr(H),
                                                   _lib.ptr(s), _lib.ptr(t), _lib.stream_ptr(torch.device(DEV)))
        _lib.check(st, "qagnn_decoder_head_ragged")
        return H.cpu(), s.cpu(), t.cpu(), ctx.cpu(), table.cpu()

    H, s, t, ctx, table = run(cid)
    nv = rows.numel()
    # the tail rows: zeros, score 0, type 2
    assert bool((H[nv:] == 0).all()) and bool((s[nv:] == 0).all()) and bool((t[nv:] == 2).all())
    # against the fp64 oracle head, re-packed: rows bit for bit (gathers of fp32 values), scores within the padded test's bar
    sd = {"svec2nvec.weight": dec.svec2nvec.weight.detach().cpu().double(), "svec2nvec.bias": dec.svec2nvec.bias.detach().cpu().double(),
          "concept_emb.emb.weight": table.double()}
    ref_H, ref_s = O.decoder_head(sd, sent.double(), cid, scores.unsqueeze(2).double(), lens, F64)
    assert torch.equal(H[:nv, :], RP.pack(torch.cat([ctx.unsqueeze(1), table[cid[:, 1:] - 1]], 1), rows, nv)), "rows"
    assert_value(s[:nv], RP.pack(ref_s, rows, nv).squeeze(-1), "scores")
    Hr = RP.pack(ref_H, rows, nv)
    assert_value(H[:nv], Hr, "rows vs fp64")
    assert torch.equal(t[:nv], RP.pack(nt.unsqueeze(-1), rows, nv).squeeze(-1)), "types"
    # the grad-mode head (PyTorch ops, gathered into the packed layout): the same rows and types bit for bit
    with torch.no_grad():
        gi, gs, gt = dec._head_ragged(sent.to(DEV), cid.to(DEV), nt.to(DEV), scores.unsqueeze(2).to(DEV), lens.to(DEV),
                                      node_ptr.to(DEV), N_cap)
    assert torch.equal(gi.cpu(), H) and torch.equal(gt.cpu(), t), "rows / types differ from QAGNN._head_ragged"
    assert_value(gs.cpu().squeeze(-1)[:nv], RP.pack(ref_s, rows, nv).squeeze(-1), "grad-mode head scores")
    # concept ids past both ends of the table read its first and last rows
    if n > 1:
        bad = cid.clone()
        bad[0, 1], bad[1, n - 1] = 0, n_concept + 1
        bad[2, 1:] = -5
        H2 = run(bad)[0]
        assert torch.equal(H2[:nv], RP.pack(torch.cat([ctx.unsqueeze(1), table[bad[:, 1:].clamp(1, n_concept) - 1]], 1), rows, nv))


# ---------------------------------------------------------------------------------------------------------------------
# 5. the module: eval-mode ragged QAGNN gradients against fp64 autograd, in fp32 and under bf16 / fp16 autocast
# ---------------------------------------------------------------------------------------------------------------------
MANT = {torch.float16: 10, torch.bfloat16: 7}


@pytest.mark.parametrize("amp", [None, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_ragged_decoder_gradients_with_five_pool_heads_match_fp64(amp):
    """QAGNN in .eval() on a ragged batch, 5 pool heads and D = 100 (dk = 20), gradients of sent_vecs, node_scores and every
    parameter against autograd of the fp64 oracle decoder.  fp32 at tests/test_gpu_eval_grad.py's training bar; under
    autocast, as tests/test_gpu_eval_grad.py bounds autocast, the error may not exceed what the same autocast costs the
    padded batch plus one ulp of the dtype at the tensor's scale."""
    import qagnn_b200
    from tests.test_gpu_eval_grad import _edge_case_decoder_batch, _grad_close, _leaves64, _ragged_adj, _set_running_stats
    bt = _edge_case_decoder_batch()
    bt["D"] = 100
    T, R, nh, k = 4, 38, 5, 2
    torch.manual_seed(3)
    dec = qagnn_b200.QAGNN(None, k, T, R, bt["sent_vecs"].size(1), bt["n_concept"], 100, 100, nh, 100, 1, 0.3, 0.3, 0.3)
    sd = _set_running_stats(dict(dec.state_dict()), seed=4)
    dec.load_state_dict(sd)
    dec = dec.to(DEV).eval()
    W = torch.randn(bt["adj_lengths"].numel(), 1, generator=torch.Generator().manual_seed(6), dtype=F64)
    s64 = _leaves64(sd)
    s64["concept_emb.emb.weight"].requires_grad_(False)
    sv64, ns64 = bt["sent_vecs"].double().requires_grad_(True), bt["node_score"].double().requires_grad_(True)
    logits64, _, _ = O.qagnn_decoder_forward(s64, sv64, bt["concept_ids"], bt["node_type"], ns64, bt["adj_lengths"],
                                             bt["edge_index"], bt["edge_type"], k, T, R, nh, 1, dtype=F64)
    (logits64 * W).sum().backward()
    ref = {"sent_vecs": sv64.grad, "node_scores": ns64.grad}
    ref.update({kk: s64[kk].grad for kk, p in dec.named_parameters() if p.requires_grad})
    ragged = _ragged_adj(bt["edge_index"], bt["edge_type"], bt["adj_lengths"], bt["n"], extra_rows=23)
    padded = (bt["edge_index"].to(DEV), bt["edge_type"].to(DEV))

    def grads(adj, dt):
        dec.zero_grad(set_to_none=True)
        sv, ns = bt["sent_vecs"].to(DEV).requires_grad_(True), bt["node_score"].to(DEV).requires_grad_(True)
        with torch.autocast("cuda", dtype=dt or torch.float32, enabled=dt is not None):
            logits, _ = dec(sv, bt["concept_ids"].to(DEV), bt["node_type"].to(DEV), ns, bt["adj_lengths"].to(DEV), adj)
            loss = (logits.float() * W.float().to(DEV)).sum()
        loss.backward()
        out = {"sent_vecs": sv.grad, "node_scores": ns.grad}
        out.update({kk: p.grad for kk, p in dec.named_parameters() if p.requires_grad})
        return out

    got = grads(ragged, amp)
    gmax = max(float(g.abs().max()) for g in ref.values())
    if amp is None:
        for kk in ref:
            _grad_close(got[kk], ref[kk], f"ragged dL/d{kk}", floor=1e-2 * gmax)
        return
    # under autocast: no further from fp64 than the padded batch under the same autocast, plus one ulp of the dtype
    pad = grads(padded, amp)
    ulp = 2.0 ** -(MANT[amp] + 1)
    for kk in ref:
        g = got[kk]
        assert g is not None and bool(torch.isfinite(g).all()), f"dL/d{kk} is missing or not finite"
        scale = max(float(ref[kk].abs().max()), 1e-2 * gmax)
        err = float((g.double().cpu() - ref[kk]).abs().max())
        auto = float((pad[kk].double().cpu() - ref[kk]).abs().max())
        assert err <= auto + ulp * scale, f"{amp} ragged dL/d{kk}: max|err| {err:.3e}, padded's {auto:.3e}, scale {scale:.3e}"
