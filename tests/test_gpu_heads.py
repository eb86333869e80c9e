"""GATConvE at every head count and head width the message-passing kernels dispatch on, against fp64 references.

The kernels branch on the head count H and on the head width d = D/H: the tiled kernel pads d to DP (a multiple of 4),
the column-sliced kernels cut it into SL-column slices, and the basic and backward kernels give each lane CH = ceil(D/128)
float4 chunks, which straddle two heads when d % 4 != 0.  Every comparison here is against an fp64 restatement: the graph
part of a layer (`mp_core_ref`, pinned to the oracle by the one CPU test of this file) or the oracle's GATConvE.
GPU tests are marked one by one.
"""
import ctypes
import functools

import pytest
import torch

from oracle import qagnn_oracle as O
from tests import helpers as Hh

F64 = torch.float64
DEV = "cuda:0"
T, R = 4, 38
NC = R * T * T + T  # combos: rows of the edge tables


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference of the message-passing core
# ---------------------------------------------------------------------------------------------------------------------
def mp_core_ref(qkm, ke, me, src, tgt, combo, H):
    """The graph part of one GATConvE layer on node-level projections, in differentiable fp64 torch ops.

    qkm [N, 3D] = [Q / sqrt(d) | Kx | Mx]; ke / me [C, D] = the edge-table halves of linear_key / linear_msg (bias included)
    per combo; src / tgt / combo [E'] as O.graph_prep_oracle lays them out (self loops last).  Returns aggr [N, D] and
    alpha [E', H], the per-source softmax before the out-degree rescale."""
    N, D = qkm.size(0), qkm.size(1) // 3
    d = D // H
    Q, Kx, Mx = (qkm[:, i * D:(i + 1) * D].reshape(N, H, d) for i in range(3))
    s = (Q[src] * (Kx[tgt] + ke.reshape(-1, H, d)[combo])).sum(-1)                                   # [E', H]
    # per-source softmax; the shift by the segment maximum cancels, so it carries no gradient
    smax = torch.full((N, H), float("-inf"), dtype=s.dtype).scatter_reduce(0, src[:, None].expand(-1, H), s.detach(), "amax")
    e = torch.exp(s - smax[src])
    alpha = e / (torch.zeros(N, H, dtype=s.dtype).index_add(0, src, e)[src] + 1e-16)
    outdeg = torch.bincount(src, minlength=N).to(s.dtype)                                             # self loop included
    msg = (alpha * outdeg[src][:, None])[:, :, None] * (Mx[src] + me.reshape(-1, H, d)[combo])
    return torch.zeros(N, H, d, dtype=s.dtype).index_add(0, tgt, msg).reshape(N, D), alpha


def _edges(edge_index, edge_type, node_type, T, R):
    p = O.graph_prep_oracle(edge_index, edge_type, node_type, T, R)
    return tuple(torch.from_numpy(p[k]) for k in ("src", "tgt", "combo"))


def combo_parts(c, T, R):
    """(edge type, source type, target type) of combo ids c in graph prep's numbering; a self loop's edge type is R."""
    real = c < R * T * T
    et = torch.where(real, c // (T * T), torch.full_like(c, R))
    ts = torch.where(real, (c // T) % T, c - R * T * T)
    tt = torch.where(real, c % T, c - R * T * T)
    return et, ts, tt


def _combo_onehots(dtype, T, R):
    """[C, R+1+2T] one-hot edge features in graph prep's combo numbering."""
    C_ = R * T * T + T
    c = torch.arange(C_)
    et, ts, tt = combo_parts(c, T, R)
    tab = torch.zeros(C_, R + 1 + 2 * T, dtype=dtype)
    tab[c, et] = 1
    tab[c, R + 1 + ts] = 1
    tab[c, R + 1 + T + tt] = 1
    return tab


def _projections(sd, prefix, x, extra, H, dtype):
    """qkm, ke, me of one eval-mode layer, formed the way the training path forms them (qagnn_b200/training.py)."""
    D = x.size(1)
    W = lambda name: sd[f"{prefix}.{name}"].to(dtype)  # noqa: E731
    x2 = torch.cat([x, extra], 1).to(dtype)
    wk, wm = W("linear_key.weight"), W("linear_msg.weight")
    q = (x2 @ W("linear_query.weight").t() + W("linear_query.bias")) / (D // H) ** 0.5
    qkm = torch.cat([q, x2 @ wk[:, :2 * D].t(), x2 @ wm[:, :2 * D].t()], 1)
    tab = O.mlp_lin_bn_relu_lin(_combo_onehots(dtype, T, R), sd, prefix + ".edge_encoder")
    return qkm, tab @ wk[:, 2 * D:].t() + W("linear_key.bias"), tab @ wm[:, 2 * D:].t() + W("linear_msg.bias")


@pytest.mark.parametrize("H,D,seed", [(4, 24, 0), (2, 10, 1)])  # (2, 10): d = 5, not a multiple of 4
def test_mp_core_reference_equals_the_oracle(H, D, seed):
    """mp_core_ref on the layer's own projections gives the oracle's alpha and aggr to 1e-10, so a GPU mismatch against it
    can only come from a kernel."""
    b = O.synth_graph_batch(3, 12, 40, D, R, seed=seed)
    sd = O.random_state_dict(1, D, T, R, "peaky", seed=seed)
    x, nt = b["H"].reshape(-1, D), b["node_type"].reshape(-1)
    extra = torch.randn(x.shape, generator=torch.Generator().manual_seed(seed)) * 0.5
    _, _, alpha_o, aggr_o = O.gatconve_forward(sd, "gnn_layers.0", x, b["edge_index"], b["edge_type"], nt, extra, T, R,
                                               head_count=H, dtype=F64)
    qkm, ke, me = _projections(sd, "gnn_layers.0", x, extra, H, F64)
    aggr, alpha = mp_core_ref(qkm, ke, me, *_edges(b["edge_index"], b["edge_type"], nt, T, R), H)
    assert torch.allclose(alpha, alpha_o, rtol=0, atol=1e-10)
    assert torch.allclose(aggr, aggr_o, rtol=1e-10, atol=1e-10)


def test_gatconve_refuses_head_counts_no_kernel_set_supports():
    from qagnn_b200 import GATConvE
    D = 480  # divisible by every head count below
    enc = torch.nn.Sequential(torch.nn.Linear(R + 1 + 2 * T, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))
    for H in (3, 5, 6, 32):
        with pytest.raises(ValueError, match=r"head_count must be one of \(1, 2, 4, 8, 16\)"):
            GATConvE(None, D, T, R, enc, head_count=H)
    for H in (1, 2, 4, 8, 16):
        assert GATConvE(None, D, T, R, enc, head_count=H).head_count == H


# ---------------------------------------------------------------------------------------------------------------------
# kernel-level backward: qagnn_mp_core_forward / _backward through training._MPCore
# ---------------------------------------------------------------------------------------------------------------------
def _excess(got, ref, scale=0.0):
    """max(|got - ref| - (2e-5 max(max|ref|, scale) + 1e-4 |ref|)): <= 0 when `got` is within the tolerance of this file."""
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    return float(((got - ref).abs() - (2e-5 * max(float(ref.abs().max()), scale) + 1e-4 * ref.abs())).max())


def _assert_tight(got, ref, what, scale=0.0):
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    ex = _excess(got, ref, scale)
    err = (got.detach().cpu().double() - ref.detach().cpu().double()).abs().max().item()
    assert ex <= 0, f"{what}: max|err| {err:.3e} (ref scale {ref.abs().max().item():.3e}) exceeds 2e-5*max|ref| + 1e-4*|ref| by {ex:.3e}"


def _graph(kind, seed=0):
    """(N, edge_index [2, E], edge_type [E], node_type [N]) on the CPU."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda hi, n: torch.randint(0, hi, (n,), generator=g)  # noqa: E731
    if kind == "random":
        N, E = 300, 1200
        src, tgt = ri(N, E), ri(N, E)
    elif kind == "self_loops_only":
        N, src, tgt = 50, ri(1, 0), ri(1, 0)
    elif kind == "one_node":  # N = 1 with three 0 -> 0 edges next to its self loop
        N, src, tgt = 1, ri(1, 3), ri(1, 3)
    elif kind in ("source_hub", "target_hub"):  # one node with 3000 out- (in-) edges plus a random rest
        N = 200
        src, tgt = ri(N, 3400), ri(N, 3400)
        (src if kind == "source_hub" else tgt)[:3000] = 7
    elif kind == "duplicates":  # every edge four times, with the same relation
        N = 100
        src, tgt, et = ri(N, 200), ri(N, 200), ri(R, 200)
        return N, torch.stack([src, tgt]).repeat(1, 4), et.repeat(4), ri(T, N)
    elif kind == "isolated":  # nodes 80..399 have their self loop only
        N = 400
        src, tgt = ri(80, 300), ri(80, 300)
    elif kind == "cross_graph":  # five graphs of 40 nodes with 50 edges between different graphs
        N = 200
        g_of = ri(5, 200)
        src, tgt = g_of * 40 + ri(40, 200), g_of * 40 + ri(40, 200)
        cross = torch.arange(150, 200)
        tgt[cross] = (g_of[cross] + 1 + ri(4, 50)) % 5 * 40 + ri(40, 50)
    elif kind == "one_combo_flood":  # one relation, one node type: all 3000 real edges share ONE dKe / dMe row
        N = 150
        return N, torch.stack([ri(N, 3000), ri(N, 3000)]), torch.full((3000,), 5, dtype=torch.long), torch.full((N,), 2, dtype=torch.long)
    elif kind == "ragged":  # N + E = 311, not a multiple of the 64-edge runs of the table kernel
        N, E = 61, 250
        src, tgt = ri(N, E), ri(N, E)
    else:
        raise ValueError(kind)
    return N, torch.stack([src, tgt]), ri(R, src.numel()), ri(T, N)


@functools.lru_cache(maxsize=None)
def _core_case(H, D, kind):
    """Random fp32 leaves through the CUDA core (forward, then backward twice) and the fp64 reference on the same values."""
    from qagnn_b200 import training as TR
    from qagnn_b200.modeling_qagnn import GraphPrep
    N, ei, et, nt = _graph(kind)
    g = torch.Generator().manual_seed(H * 4096 + D)
    qkm = torch.randn(N, 3 * D, generator=g)
    qkm[:, :D] /= (D // H) ** 0.5  # Q / sqrt(d) as the layer scales it: logits stay O(1) at every head width
    ke, me = torch.randn(NC, D, generator=g), torch.randn(NC, D, generator=g)
    G = torch.randn(N, D, generator=g)
    prep = GraphPrep(ei.to(DEV), et.to(DEV), nt.to(DEV), T, R, n_per_graph=0)
    leaves = [t.to(DEV).requires_grad_(True) for t in (qkm, ke, me)]
    aggr, alpha = TR._MPCore.apply(*leaves, prep, (N, ei.size(1), D, H, T, R), True)
    grads = torch.autograd.grad(aggr, leaves, G.to(DEV), retain_graph=True)
    grads2 = torch.autograd.grad(aggr, leaves, G.to(DEV))
    ref_leaves = [t.double().requires_grad_(True) for t in (qkm, ke, me)]
    edges = _edges(ei, et, nt, T, R)
    raggr, ralpha = mp_core_ref(*ref_leaves, *edges, H)
    rgrads = torch.autograd.grad(raggr, ref_leaves, G.double())
    cpu = lambda ts: [t.detach().cpu() for t in ts]  # noqa: E731
    return dict(got=cpu([aggr, alpha, *grads]), again=cpu(grads2), ref=[raggr.detach(), ralpha.detach(), *rgrads],
                inputs=(qkm, ke, me, G, ei, et, nt))


def _check_core(case, D, kind):
    names = ("aggr", "alpha", "dQ", "dKx", "dMx", "d_ke", "d_me")
    aggr, alpha, d_qkm, d_ke, d_me = case["got"]
    raggr, ralpha, rd_qkm, rd_ke, rd_me = case["ref"]
    got = (aggr, alpha, *d_qkm.split(D, 1), d_ke, d_me)
    ref = (raggr, ralpha, *rd_qkm.split(D, 1), rd_ke, rd_me)
    scale = {}
    if kind == "one_node":
        # every edge runs 0 -> 0, so dKx[0] = Q[0] * sum(ds) is exactly 0 (the softmax gradient sums to zero over one
        # source): the kernel's value is the fp32 rounding of terms as large as dQ's, so it is judged on dQ's scale
        scale["dKx"] = float(rd_qkm[:, :D].abs().max())
    for name, g_, r_ in zip(names, got, ref):
        _assert_tight(g_, r_, name, scale.get(name, 0.0))
    # d_qkm comes from atomic-free kernels: bit-identical on a second backward; d_ke / d_me accumulate with atomics
    assert torch.equal(case["again"][0], d_qkm), "d_qkm differs between two backward calls"
    _assert_tight(case["again"][1], rd_ke, "d_ke (second backward)")
    _assert_tight(case["again"][2], rd_me, "d_me (second backward)")


# D per head count giving CH = ceil(D/128) = 1, 2, 4, 8 (in that order); several have d % 4 != 0, so float4 chunks
# straddle two heads: (2, 388) d = 194, (4, 100) d = 25, (4, 232) d = 58, (4, 1020) d = 255, (8, 200) d = 25,
# (8, 488) d = 61, (8, 1000) d = 125, (16, 208) d = 13, (16, 400) d = 25
BWD_SHAPES = [(1, 36), (1, 200), (1, 500), (1, 1020),
              (2, 40), (2, 200), (2, 388), (2, 1000),
              (4, 100), (4, 232), (4, 400), (4, 1020),
              (8, 64), (8, 200), (8, 488), (8, 1000),
              (16, 64), (16, 208), (16, 400), (16, 1024)]
EDGE_KINDS = ["self_loops_only", "one_node", "source_hub", "target_hub", "duplicates", "isolated", "cross_graph",
              "one_combo_flood", "ragged"]


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", BWD_SHAPES)
def test_core_forward_and_backward_every_instantiation(H, D):
    assert (D + 127) // 128 in (1, 2, 4, 8)
    _check_core(_core_case(H, D, "random"), D, "random")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", EDGE_KINDS)
@pytest.mark.parametrize("H,D", [(4, 200), (8, 1000)])
def test_core_backward_graph_edge_cases(H, D, kind):
    case = _core_case(H, D, kind)
    N, E = case["inputs"][0].size(0), case["inputs"][4].size(1)
    if kind == "ragged":
        assert (N + E) % 64 != 0
    _check_core(case, D, kind)


@pytest.mark.gpu
def test_core_tolerance_rejects_a_missing_edge_and_swapped_heads():
    """The comparison above is sharp enough to see one missing edge among 1500 or two heads' gradients swapped."""
    H, D = 4, 200
    case = _core_case(H, D, "random")
    aggr, _, d_qkm, d_ke, d_me = case["got"]
    raggr, _, rd_qkm, rd_ke, rd_me = case["ref"]
    assert max(_excess(g_, r_) for g_, r_ in zip((aggr, d_qkm, d_ke, d_me), (raggr, rd_qkm, rd_ke, rd_me))) <= 0
    qkm, ke, me, G, ei, et, nt = case["inputs"]
    # the reference of the same graph without its first edge
    leaves = [t.double().requires_grad_(True) for t in (qkm, ke, me)]
    paggr, _ = mp_core_ref(*leaves, *_edges(ei[:, 1:], et[1:], nt, T, R), H)
    pd_qkm, pd_ke, pd_me = torch.autograd.grad(paggr, leaves, G.double())
    for name, g_, r_ in (("aggr", aggr, paggr), ("d_qkm", d_qkm, pd_qkm), ("d_ke", d_ke, pd_ke), ("d_me", d_me, pd_me)):
        assert _excess(g_, r_.detach()) > 0, f"{name}: a reference missing one edge passes the tolerance"
    # heads 0 and 1 of the softmax gradient swapped: what a wrong head mapping of ds writes into dKe (and dQ / dKx)
    d = D // H
    perm = torch.tensor([1, 0, 2, 3])
    assert _excess(d_ke, rd_ke.view(NC, H, d)[:, perm].reshape(NC, D)) > 0
    assert _excess(d_qkm[:, :D], rd_qkm[:, :D].view(-1, H, d)[:, perm].reshape(-1, D)) > 0


# ---------------------------------------------------------------------------------------------------------------------
# eval forward of GATConvE on every path
# ---------------------------------------------------------------------------------------------------------------------
PATH_TILED, PATH_SLICE, PATH_BASIC = 0, 1, 2  # qagnn_mp_path (include/qagnn_b200.h)

# (H, D, tiled path taken with a per-graph prep, path taken without one; None = no kernel takes it)
EVAL_SHAPES = [
    (1, 8, True, PATH_BASIC),       # DP 8
    (1, 36, True, PATH_BASIC),      # DP 36: two float4 chunks per lane in the tiled kernel
    (1, 128, False, PATH_SLICE),    # d 128: two SL = 64 slices per head
    (1, 256, False, PATH_BASIC),    # too wide for tiles and slices
    (2, 10, True, None),            # d 5 -> DP 8; D % 4 != 0: only the tiled kernel takes it
    (2, 24, True, PATH_BASIC),      # DP 12
    (2, 64, True, PATH_SLICE),      # DP 32, SL 32
    (2, 104, True, PATH_BASIC),     # DP 52
    (8, 32, True, PATH_BASIC),      # DP 4
    (8, 128, True, PATH_SLICE),     # DP 16, SL 16
    (8, 160, True, PATH_BASIC),     # DP 20
    (8, 400, True, PATH_BASIC),     # DP 52, H * DP = 416 > 256: the projection GEMM splits a `which` over two n tiles
    (8, 1024, False, PATH_SLICE),   # d 128: two slices per head
    (16, 64, True, PATH_BASIC),     # DP 4
    (16, 192, True, PATH_BASIC),    # DP 12
    (16, 320, True, PATH_BASIC),    # DP 20, H * DP = 320 > 256
    (16, 512, True, PATH_SLICE),    # DP 32, SL 32, H * DP = 512
    (16, 576, True, PATH_BASIC),    # DP 36, H * DP = 576
]


def _enc(D):
    return torch.nn.Sequential(torch.nn.Linear(R + 1 + 2 * T, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))


def _layer(H, D, sd):
    from qagnn_b200 import GATConvE
    layer = GATConvE(None, D, T, R, _enc(D), head_count=H)
    layer.load_state_dict({k[len("gnn_layers.0."):]: v for k, v in sd.items() if k.startswith("gnn_layers.0.")}, strict=True)
    return layer.to(DEV)


@functools.lru_cache(maxsize=None)
def _eval_case(H, D):
    B, n, e = 6, 50, 150
    seed = 97 * H + D
    b = O.synth_graph_batch(B, n, e, D, R, seed=seed)
    sd = O.random_state_dict(1, D, T, R, "peaky", seed=seed)
    x, nt = b["H"].reshape(-1, D), b["node_type"].reshape(-1)
    extra = torch.randn(x.shape, generator=torch.Generator().manual_seed(seed)) * 0.5
    out, _, alpha, aggr = O.gatconve_forward(sd, "gnn_layers.0", x, b["edge_index"], b["edge_type"], nt, extra, T, R,
                                             head_count=H, dtype=F64)
    return dict(n=n, sd=sd, x=x, extra=extra, nt=nt, ei=b["edge_index"], et=b["edge_type"], ref=(out, alpha, aggr))


def _mp_path(prep, H, D):
    from qagnn_b200 import _lib
    with torch.cuda.device(DEV):
        return _lib.load().qagnn_mp_path(ctypes.byref(_lib.Shape(prep.N, prep.E, D, H, T, R, 1, prep.n_per_graph)))


@pytest.mark.gpu
@pytest.mark.parametrize("gemm", ["tc", "ffma"])
@pytest.mark.parametrize("H,D,tiled,general", EVAL_SHAPES)
def test_eval_forward_on_every_path(H, D, tiled, general, gemm, monkeypatch):
    from qagnn_b200 import _lib
    from qagnn_b200.modeling_qagnn import GraphPrep
    monkeypatch.delenv("QAGNN_MP_PATH", raising=False)
    if gemm == "ffma":
        monkeypatch.setenv("QAGNN_GEMM", "ffma")
    else:
        monkeypatch.delenv("QAGNN_GEMM", raising=False)
    c = _eval_case(H, D)
    layer = _layer(H, D, c["sd"]).eval()
    x, extra, nt = c["x"].to(DEV), c["extra"].to(DEV), c["nt"].to(DEV)
    ei, et = c["ei"].to(DEV), c["et"].to(DEV)
    ref_out, ref_alpha, ref_aggr = c["ref"]

    def run(prep, label, want_path):
        assert _mp_path(prep, H, D) == want_path, f"{label}: qagnn_mp_path says {_mp_path(prep, H, D)}, expected {want_path}"
        (out, (_, alpha)), aggr = layer(x, None, None, nt, extra, return_attention_weights=True, prep=prep, return_aggr=True)
        Hh.assert_close(out, ref_out, f"{label} out")
        Hh.assert_close(alpha, ref_alpha, f"{label} alpha")
        Hh.assert_close(aggr, ref_aggr, f"{label} aggr")

    prep_t = GraphPrep(ei, et, nt, T, R, n_per_graph=c["n"])
    assert prep_t.n_per_graph == c["n"]
    if tiled:
        run(prep_t, "tiled", PATH_TILED)
    else:
        assert _mp_path(prep_t, H, D) != PATH_TILED
    prep_c = GraphPrep(ei, et, nt, T, R, n_per_graph=0)
    if general is None:  # refused by status, before any message-passing launch
        with pytest.raises(_lib.QagnnError, match="unsupported shape"):
            layer(x, None, None, nt, extra, prep=prep_c)
        return
    run(prep_c, "general", general)
    if general == PATH_SLICE:
        monkeypatch.setenv("QAGNN_MP_PATH", "basic")
        run(prep_c, "basic", PATH_BASIC)


# ---------------------------------------------------------------------------------------------------------------------
# module-level training
# ---------------------------------------------------------------------------------------------------------------------
def _grad_close(got, ref, what, floor=0.0):
    # as tests/test_gpu_training.py: 1e-4 of the tensor's own scale (or of `floor` for a gradient that is zero up to
    # rounding, such as the bias in front of a BatchNorm) plus 1e-4 relative
    scale = max(float(ref.abs().max()), floor, 1e-6)
    Hh.assert_close(got, ref, what, atol=1e-4 * scale, rtol=1e-4)


# one CH = 1 and one CH >= 4 width per head count (H = 4 is covered in tests/test_gpu_training.py)
TRAIN_SHAPES = [(1, 64), (1, 512), (2, 100), (2, 400), (8, 64), (8, 488), (16, 128), (16, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", TRAIN_SHAPES)
def test_training_layer_matches_autograd_of_the_oracle(H, D):
    seed = 31 * H + D
    b = O.synth_graph_batch(3, 30, 90, D, R, seed=seed)
    sd = O.random_state_dict(1, D, T, R, "peaky", seed=seed)
    x, nt = b["H"].reshape(-1, D), b["node_type"].reshape(-1)
    g = torch.Generator().manual_seed(seed)
    extra = torch.randn(x.shape, generator=g) * 0.5
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items() if k.startswith("gnn_layers.0.") and v.is_floating_point()}
    x64, e64 = x.double().requires_grad_(True), extra.double().requires_grad_(True)
    ref_out, _, ref_alpha, _ = O.gatconve_forward(sd64, "gnn_layers.0", x64, b["edge_index"], b["edge_type"], nt, e64, T, R,
                                                  head_count=H, dtype=F64, train=True)
    G = torch.randn(ref_out.shape, generator=g)
    (ref_out * G.double()).sum().backward()

    layer = _layer(H, D, sd).train()
    xg, eg = x.to(DEV).requires_grad_(True), extra.to(DEV).requires_grad_(True)
    out, (_, alpha) = layer(xg, b["edge_index"].to(DEV), b["edge_type"].to(DEV), nt.to(DEV), eg, return_attention_weights=True)
    Hh.assert_close(out, ref_out.detach(), "train-mode out")
    Hh.assert_close(alpha, ref_alpha.detach(), "alpha")
    (out * G.to(DEV)).sum().backward()
    _grad_close(xg.grad, x64.grad, "dL/dx")
    _grad_close(eg.grad, e64.grad, "dL/dextra")
    params = dict(layer.named_parameters())
    refs = {name: sd64["gnn_layers.0." + name].grad for name in params}
    gmax = max(float(r.abs().max()) for r in refs.values())
    for name, p in params.items():
        assert p.grad is not None and refs[name] is not None, name
        _grad_close(p.grad, refs[name], f"dL/d{name}", floor=1e-2 * gmax)
