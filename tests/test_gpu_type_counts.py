"""Every message-passing path at node- and edge-type counts (T, R) other than the reference's (4, 38), on both sides of each
limit the combo count C = R*T*T + T decides.

C is the number of distinct one-hot edge features: a real edge (type r, source type ts, target type tt) has combo
(r*T + ts)*T + tt, the self loop of a type-t node R*T*T + t.  Every edge table has C rows, and these plan decisions depend on it:
  * the tiled kernel (mp_headtile.cu make_plan) addresses table rows through 16-bit words: (C - 1)*(DP/4)*8 <= 65535, DP the head
    width padded to a multiple of 4;
  * it keeps the table and two node tiles in shared memory: C*DP*4 + 2*n*DP*4 + 64 <= the device's opt-in shared memory;
  * the column-sliced kernels (mp_slice.cu make_slice_plan) keep an SL-column table slice there: C*SL*4 <= opt-in;
  * the combo sort of the training backward (combo_sort.cu) takes C <= 6144;
  * the packed and ragged graph preps store 16|16-bit (local id, combo) words: C <= 65536.
A plan that accepts one combo too many would read another in-bounds table row without any fault, one that refuses too early
would quietly lose the fast path.  Each row below states its expected path by hand; the tests check it with qagnn_mp_path and
with the kernels the profiler saw, and compare the result with an fp64 reference that gathers the edge encoder's first linear
instead of building one-hot rows (their width R + 1 + 2T is impractical at R = 65536).  tests/test_type_counts_cpu.py checks,
without a GPU, that every limit has a row exactly at it and one just past it.
"""
import ctypes

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import _lib
from qagnn_b200 import data as Dt
from tests import helpers as Hh
from tests.test_gpu_heads import _check_core, _edges, combo_parts, mp_core_ref

DEV = "cuda:0"
F64 = torch.float64
BF = torch.bfloat16
PATHS = {"tiled": 0, "slice": 1, "basic": 2}  # qagnn_mp_path (include/qagnn_b200.h)
PATH_KERNELS = {"tiled": "mp_headtile_kernel", "slice": "mp_slice_scores_kernel", "basic": "mp_scores_kernel"}
PREP_COMBO_MAX = 65536   # graph_prep.cu: combo ids of the packed / ragged preps are 16 bits
COMBO_SORT_MAX = 6144    # combo_sort.cu kMaxCombos


# ---------------------------------------------------------------------------------------------------------------------
# the rows
# ---------------------------------------------------------------------------------------------------------------------
def combos(T, R):
    return R * T * T + T


def head_dim_padded(H, D):
    return (D // H + 3) // 4 * 4


class Row:
    """One eval forward: GATConvE (H, D) and QAGNN_Message_Passing (k = 1) at (T, R) on graphs of n nodes, with the per-graph
    prep.  `limit` is the limit the row sits on ('offset', 'tile_smem', 'slice_smem') and `side` 'at' (the largest accepted
    value) or 'past' (one more); None for a row that covers something else.  `path` is the path the row must take."""

    def __init__(self, H, D, T, R, path, limit=None, side=None, n=40, fast=False, note=""):
        assert path in PATHS and side in (None, "at", "past")
        self.H, self.D, self.T, self.R, self.path, self.limit, self.side, self.n = H, D, T, R, path, limit, side, n
        self.fast, self.note = fast, note
        self.C, self.DP = combos(T, R), head_dim_padded(H, D)
        self.id = f"h{H}-d{D}-t{T}-r{R}" + (f"-n{n}" if n != 40 else "") + f"-{path}"


# The 16-bit table offset of the tiled kernel: (C - 1) * (DP / 4) * 8 <= 65535, so C <= 631 at DP 52, 1024 at DP 32, 2048 at
# DP 16 and 8192 at DP 4.  At T = 1 the limit is hit exactly; at T > 1, C moves in steps of T*T and the row is the largest R.
# A refused shape goes to the column-sliced kernels where its head width has slices (d 32 and 16), else to the basic ones.
OFFSET_ROWS = [
    Row(4, 200, 1, 630, "tiled", "offset", "at"),  Row(4, 200, 1, 631, "basic", "offset", "past"),    # d 50: no slices
    Row(4, 200, 4, 39, "tiled", "offset", "at"),   Row(4, 200, 4, 40, "basic", "offset", "past"),
    Row(2, 64, 1, 1023, "tiled", "offset", "at"),  Row(2, 64, 1, 1024, "slice", "offset", "past"),    # SL 32
    Row(2, 64, 2, 255, "tiled", "offset", "at"),   Row(2, 64, 2, 256, "slice", "offset", "past"),
    Row(8, 128, 1, 2047, "tiled", "offset", "at"), Row(8, 128, 1, 2048, "slice", "offset", "past"),   # SL 16
    Row(8, 128, 8, 31, "tiled", "offset", "at"),   Row(8, 128, 8, 32, "slice", "offset", "past"),
    Row(8, 32, 1, 8191, "tiled", "offset", "at"),  Row(8, 32, 1, 8192, "basic", "offset", "past"),    # d 4: no slices
    Row(8, 32, 16, 31, "tiled", "offset", "at"),   Row(8, 32, 16, 32, "basic", "offset", "past"),
]
# 64 node types on the fast projection: 64 per-type bias rows (fold.cu tbias), C = 4160
OTHER_ROWS = [Row(8, 32, 64, 1, "tiled", fast=True, note="64 per-type bias rows")]


def smem_rows(optin):
    """The rows of the two limits set by the opt-in shared memory per block `optin` (bytes): the tiled kernel's node tile at
    (4, 200), T = 4, R = 38 (n = 252 on a 227 KB H100), and the column-sliced table at SL 16 (8, 128) and SL 32 (2, 64)
    (C = optin / (4 SL): 3632 and 1816 on an H100).  T = 1, so C = R + 1 reaches every value."""
    C, DP = combos(4, 38), head_dim_padded(4, 200)
    n = (optin - 64 - C * DP * 4) // (2 * DP * 4)
    rows = [Row(4, 200, 4, 38, "tiled", "tile_smem", "at", n=n), Row(4, 200, 4, 38, "basic", "tile_smem", "past", n=n + 1)]
    for H, D, SL in ((8, 128, 16), (2, 64, 32)):
        Cmax = optin // (4 * SL)
        rows += [Row(H, D, 1, Cmax - 1, "slice", "slice_smem", "at"), Row(H, D, 1, Cmax, "basic", "slice_smem", "past")]
    return rows


# graph prep: the packed / ragged preps take C <= 65536 ((1, 65535): the top combo is 0xffff) and refuse (1, 65536)
PREP_CASES = [(1, 5), (7, 3), (16, 23), (16, 255), (1, 65535)]
PREP_REFUSED = (1, 65536)
COMBO_SORT_CASES = [((1, 6143), True), ((1, 6144), False)]  # C = 6144 sorted, 6145 refused


def _optin():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def batch(T, R, D, seed, B=4, n=40, e=120, lens=None):
    """B graphs of n padded nodes, node types over all of [0, T), edge types over all of [0, R), edges inside each graph's first
    lens[b] nodes, laid out graph by graph.  Forces the extreme combos: nodes 1 and 2 of graph 0 have type T - 1 and an edge
    1 -> 2 of type R - 1 (combo R*T*T - 1); node 1's self loop is combo C - 1."""
    g = torch.Generator().manual_seed(seed)
    lens = list(lens) if lens is not None else [n] * B
    nt = torch.randint(0, T, (B, n), generator=g)
    eis, ets = [], []
    for L_ in lens:
        m = e if L_ > 1 else 0
        eis.append(torch.randint(0, L_, (2, m), generator=g))
        ets.append(torch.randint(0, R, (m,), generator=g))
    nt[0, 1] = nt[0, 2] = T - 1
    eis[0] = torch.cat([eis[0], torch.tensor([[1], [2]])], 1)
    ets[0] = torch.cat([ets[0], torch.tensor([R - 1])])
    return {"H": torch.randn(B, n, D, generator=g) * 0.5, "extra": torch.randn(B * n, D, generator=g) * 0.5,
            "edge_index": torch.cat([e_ + b * n for b, e_ in enumerate(eis)], 1), "edge_type": torch.cat(ets),
            "node_type": nt, "node_score": torch.randn(B, n, 1, generator=g), "adj_lengths": torch.tensor(lens),
            "local": (eis, ets), "n": n}


def assert_extreme_combos(prep, T, R, what=""):
    """Both extreme combos occur in the prep's combo array: R*T*T - 1 (a real edge) and C - 1 (a self loop)."""
    c = prep.array("combo")[:prep.N + prep.E].cpu()
    for want in (R * T * T - 1, combos(T, R) - 1):
        assert bool((c == want).any()), f"{what}: combo {want} does not occur"
    assert int(c.max()) == combos(T, R) - 1 and int(c.min()) >= 0, what


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference in gather form
# ---------------------------------------------------------------------------------------------------------------------
def edge_tables(sd, prefix, ee, combo_ids, T, R, D):
    """ke, me [len(combo_ids), D]: the edge-table halves of linear_key / linear_msg (bias included) for the given combos.  The
    edge encoder's first linear of a one-hot row is a sum of three columns: W0[:, r] + W0[:, R+1+ts] + W0[:, R+1+T+tt] + b0."""
    et, ts, tt = combo_parts(combo_ids, T, R)
    W0 = sd[ee + ".0.weight"].to(F64)
    h = W0[:, et].t() + W0[:, R + 1 + ts].t() + W0[:, R + 1 + T + tt].t() + sd[ee + ".0.bias"].to(F64)
    emb = O.linear(torch.relu(O.batchnorm_eval(h, sd, ee + ".1")), sd, ee + ".3")
    W = lambda name: sd[f"{prefix}.{name}"].to(F64)  # noqa: E731
    return (emb @ W("linear_key.weight")[:, 2 * D:].t() + W("linear_key.bias"),
            emb @ W("linear_msg.weight")[:, 2 * D:].t() + W("linear_msg.bias"))


def layer_ref(sd, prefix, ee, x, extra, ei, et, nt, T, R, H, remap=None):
    """GATConvE in eval mode, fp64: (out, alpha, aggr).  remap(combo) -> combo seeds a fault: the table row each edge reads."""
    D = x.size(1)
    p = O.graph_prep_oracle(ei, et, nt, T, R)
    src, tgt, combo = (torch.from_numpy(p[k]) for k in ("src", "tgt", "combo"))
    if remap is not None:
        combo = remap(combo)
    used, row = torch.unique(combo, return_inverse=True)
    W = lambda name: sd[f"{prefix}.{name}"].to(F64)  # noqa: E731
    x2 = torch.cat([x, extra], 1).to(F64)
    q = (x2 @ W("linear_query.weight").t() + W("linear_query.bias")) / (D // H) ** 0.5
    qkm = torch.cat([q, x2 @ W("linear_key.weight")[:, :2 * D].t(), x2 @ W("linear_msg.weight")[:, :2 * D].t()], 1)
    ke, me = edge_tables(sd, prefix, ee, used, T, R, D)
    aggr, alpha = mp_core_ref(qkm, ke, me, src, tgt, row, H)
    return O.mlp_lin_bn_relu_lin(aggr, sd, prefix + ".mlp"), alpha, aggr


def mp_ref(sd, H_in, ei, et, nt, score, k, T, R, H):
    """QAGNN_Message_Passing in eval mode, fp64, layers by layer_ref: out [B*n, D]."""
    D = H_in.size(-1)
    extra = O.node_feature_extra(sd, nt, score, T, D, F64)
    X = H_in.reshape(-1, D).to(F64)
    for l_ in range(k):
        X = O.gelu_tanh(layer_ref(sd, f"gnn_layers.{l_}", "edge_encoder", X, extra, ei, et, nt.reshape(-1), T, R, H)[0])
    return O.gelu_tanh(O.linear(H_in.reshape(-1, D).to(F64), sd, "Vh") + O.linear(X, sd, "Vx"))


@pytest.mark.parametrize("T,R,H,D", [(1, 4, 4, 24), (3, 5, 2, 10), (6, 2, 4, 32)])
def test_gather_reference_equals_the_oracle(T, R, H, D):
    """The gather-form reference gives the oracle's one-hot GATConvE and message passing to 1e-10 at small (T, R), so a GPU
    mismatch against it at large R can only come from a kernel."""
    b = batch(T, R, D, seed=T * 100 + R, B=3, n=12, e=40)
    sd = O.random_state_dict(2, D, T, R, "peaky", seed=T + R)
    x, nt, ei, et = b["H"].reshape(-1, D), b["node_type"].reshape(-1), b["edge_index"], b["edge_type"]
    want = O.gatconve_forward(sd, "gnn_layers.0", x, ei, et, nt, b["extra"], T, R, head_count=H, dtype=F64)
    got = layer_ref(sd, "gnn_layers.0", "gnn_layers.0.edge_encoder", x, b["extra"], ei, et, nt, T, R, H)
    for name, g_, w_ in zip(("out", "alpha", "aggr"), got, (want[0], want[2], want[3])):
        assert torch.allclose(g_, w_, rtol=1e-10, atol=1e-10), name
    want = O.message_passing_forward(sd, b["H"], ei, et, b["node_type"], b["node_score"], 2, T, R, head_count=H, dtype=F64)
    got = mp_ref(sd, b["H"], ei, et, b["node_type"], b["node_score"], 2, T, R, H)
    assert torch.allclose(got, want.reshape(-1, D), rtol=1e-10, atol=1e-10)


# ---------------------------------------------------------------------------------------------------------------------
# modules and kernels
# ---------------------------------------------------------------------------------------------------------------------
def _enc(D, T, R):
    return torch.nn.Sequential(torch.nn.Linear(R + 1 + 2 * T, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))


def layer_module(H, D, T, R, sd):
    layer = qagnn_b200.GATConvE(None, D, T, R, _enc(D, T, R), head_count=H)
    layer.load_state_dict({k[len("gnn_layers.0."):]: v for k, v in sd.items() if k.startswith("gnn_layers.0.")}, strict=True)
    return layer.eval().to(DEV)


def mp_module(H, D, k, T, R, sd, dropout=0.1):
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, T, R, D, D, D, dropout=dropout)
    mod.gnn_layers = torch.nn.ModuleList([qagnn_b200.GATConvE(None, D, T, R, mod.edge_encoder, head_count=H) for _ in range(k)])
    mod.load_state_dict(sd, strict=True)
    return mod.to(DEV)


def mp_path(prep, H, D, T, R):
    with torch.cuda.device(DEV):
        return _lib.load().qagnn_mp_path(ctypes.byref(_lib.Shape(prep.N, prep.E, D, H, T, R, 1, prep.n_per_graph)))


def assert_path_ran(names, path, what):
    from tests.test_gpu_forward_plans import _has
    ran = [p for p, k in PATH_KERNELS.items() if _has(names, k)]
    assert ran == [path], f"{what}: the message-passing kernels of {ran} ran, expected {path}"


def _profiled(fn):
    """(fn(), kernel names) of a call after a first, unprofiled one that folds the weights."""
    from tests.test_gpu_forward_plans import _kernels
    fn()
    return _kernels(fn)


def _layer_call(layer, b, prep, dt=torch.float32):
    x, extra = b["H"].reshape(-1, layer.emb_dim).to(DEV, dt), b["extra"].to(DEV, dt)
    with torch.no_grad():
        (out, (_, alpha)), aggr = layer(x, None, None, b["node_type"].reshape(-1).to(DEV), extra, return_attention_weights=True,
                                        prep=prep, return_aggr=True)
    torch.cuda.synchronize()
    return out.cpu(), alpha.cpu(), aggr.cpu()


def _mp_call(mod, b, adj=None):
    adj = adj if adj is not None else (b["edge_index"].to(DEV), b["edge_type"].to(DEV))
    with torch.no_grad():
        out = mod(b["H"].to(DEV), adj, b["node_type"].to(DEV), b["node_score"].to(DEV))
    torch.cuda.synchronize()
    return out.reshape(-1, out.size(-1)).cpu()


def _prep(b, T, R, n_per_graph):
    from qagnn_b200.modeling_qagnn import GraphPrep
    return GraphPrep(b["edge_index"].to(DEV), b["edge_type"].to(DEV), b["node_type"].reshape(-1).to(DEV), T, R,
                     n_per_graph=n_per_graph)


def _row_case(r, seed):
    B = 2 if r.n > 100 else 4
    b = batch(r.T, r.R, r.D, seed, B=B, n=r.n, e=3 * r.n)
    sd = O.random_state_dict(1, r.D, r.T, r.R, "peaky", seed=seed)
    return b, sd


def _layer_refs(r, b, sd, remap=None):
    return layer_ref(sd, "gnn_layers.0", "gnn_layers.0.edge_encoder", b["H"].reshape(-1, r.D), b["extra"], b["edge_index"],
                     b["edge_type"], b["node_type"].reshape(-1), r.T, r.R, r.H, remap)


def _check_layer(got, ref, what):
    for name, g_, r_ in zip(("out", "alpha", "aggr"), got, ref):
        Hh.assert_close(g_, r_, f"{what} {name}")


# ---------------------------------------------------------------------------------------------------------------------
# eval forward on each side of every limit
# ---------------------------------------------------------------------------------------------------------------------
def _run_row(r, monkeypatch):
    for name in ("QAGNN_MP_PATH", "QAGNN_GEMM", "QAGNN_MP_FASTPROJ", "QAGNN_MP_WARPS"):
        monkeypatch.delenv(name, raising=False)
    seed = r.C + 7 * r.H + r.n
    b, sd = _row_case(r, seed)
    prep = _prep(b, r.T, r.R, b["n"])
    assert prep.n_per_graph == b["n"]
    assert_extreme_combos(prep, r.T, r.R, r.id)
    assert mp_path(prep, r.H, r.D, r.T, r.R) == PATHS[r.path], f"{r.id}: qagnn_mp_path {mp_path(prep, r.H, r.D, r.T, r.R)}"
    layer = layer_module(r.H, r.D, r.T, r.R, sd)
    got, names = _profiled(lambda: _layer_call(layer, b, prep))
    assert_path_ran(names, r.path, f"{r.id} layer")
    _check_layer(got, _layer_refs(r, b, sd), f"{r.id} layer")

    mod = mp_module(r.H, r.D, 1, r.T, r.R, sd).eval()
    out, names = _profiled(lambda: _mp_call(mod, b))
    assert_path_ran(names, r.path, f"{r.id} message passing")
    from tests.test_gpu_forward_plans import _has
    if r.fast:
        assert _has(names, "sin_basis_planes_kernel"), f"{r.id}: the fast-form projection did not run"
    ref = mp_ref(sd, b["H"], b["edge_index"], b["edge_type"], b["node_type"], b["node_score"], 1, r.T, r.R, r.H)
    Hh.assert_close(out, ref, f"{r.id} message passing out")
    return b, sd, got


@pytest.mark.gpu
@pytest.mark.parametrize("r", OFFSET_ROWS + OTHER_ROWS, ids=[r.id for r in OFFSET_ROWS + OTHER_ROWS])
def test_eval_forward_at_the_table_offset_limit(r, monkeypatch):
    _run_row(r, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(6))
def test_eval_forward_at_the_shared_memory_limits(i, monkeypatch):
    """Rows made from the device's opt-in shared memory: the tiled node tile and the column-sliced table, at and past."""
    r = smem_rows(_optin())[i]
    _run_row(r, monkeypatch)


def _find(H, D, T, R):
    return next(r for r in OFFSET_ROWS if (r.H, r.D, r.T, r.R) == (H, D, T, R))


@pytest.mark.gpu
def test_layer_bar_rejects_the_top_combo_reading_row_0(monkeypatch):
    """At C = 631 on the tiled kernel every self loop is combo C - 1: a reference that reads table row 0 for it fails."""
    r = _find(4, 200, 1, 630)
    b, sd, got = _run_row(r, monkeypatch)
    bad = _layer_refs(r, b, sd, remap=lambda c: torch.where(c == r.C - 1, torch.zeros_like(c), c))
    with pytest.raises(AssertionError):
        _check_layer(got, bad, "combo C - 1 read as row 0")


@pytest.mark.gpu
def test_layer_bar_rejects_swapped_self_loop_types(monkeypatch):
    """At T = 4, R = 39 (C = 628, tiled): a reference with the self-loop combos of types T - 1 and 0 swapped fails."""
    r = _find(4, 200, 4, 39)
    b, sd, got = _run_row(r, monkeypatch)
    lo, hi = r.R * r.T * r.T, r.C - 1
    bad = _layer_refs(r, b, sd, remap=lambda c: torch.where(c == lo, hi, torch.where(c == hi, lo, c)))
    with pytest.raises(AssertionError):
        _check_layer(got, bad, "self-loop types T - 1 and 0 swapped")


@pytest.mark.gpu
def test_bf16_autocast_layer_at_seven_node_types(monkeypatch):
    """(7, 3) under bf16 autocast on the tiled kernel and single-pass bf16 GEMMs, against the bf16 contract emulation of
    tests/test_gpu_eval_bf16.py with its bars."""
    from tests import test_gpu_eval_bf16 as E16
    from tests.test_gpu_forward_plans import _has
    for name in ("QAGNN_MP_PATH", "QAGNN_GEMM", "QAGNN_MP_FASTPROJ", "QAGNN_MP_WARPS"):
        monkeypatch.delenv(name, raising=False)
    T, R, H, D = 7, 3, 4, 200
    b = batch(T, R, D, seed=73)
    sd = O.random_state_dict(1, D, T, R, "peaky", seed=73)
    prep = _prep(b, T, R, b["n"])
    assert_extreme_combos(prep, T, R, "bf16")
    layer = layer_module(H, D, T, R, sd)

    def call():
        with torch.autocast("cuda", dtype=BF):
            return _layer_call(layer, b, prep)
    (out, _, _), names = _profiled(call)
    assert out.dtype == BF and _has(names, "gemm_bf16_kernel")
    assert_path_ran(names, "tiled", "bf16 layer")
    bf = lambda t: t.float().to(BF).double()  # noqa: E731
    emu, mag, rss = E16._emulate_layer(sd, "gnn_layers.0", "gnn_layers.0.edge_encoder", bf(b["H"].reshape(-1, D)), bf(b["extra"]),
                                       b["edge_index"], b["edge_type"], b["node_type"].reshape(-1), T, R, H, E16.Variant())
    ok, frac, worst = E16._bars_hold(out.reshape(-1, D), bf(emu), mag, rss, ulp_out=True)
    assert ok, f"bf16 layer at (7, 3): {frac:.3f} over the tight bar, worst {worst:.2f} of the loose bar"


@pytest.mark.gpu
def test_ragged_message_passing_at_seven_node_types(monkeypatch):
    """(7, 3) on a ragged batch: its rows equal the padded batch's on the same tiled plan bit for bit, and the fp64 reference."""
    from tests.test_gpu_ragged import ragged_inputs
    for name in ("QAGNN_MP_PATH", "QAGNN_GEMM", "QAGNN_MP_FASTPROJ", "QAGNN_MP_WARPS"):
        monkeypatch.delenv(name, raising=False)
    T, R, H, D, n = 7, 3, 4, 200, 40
    b = batch(T, R, D, seed=74, B=5, n=n, lens=[n, 9, 1, n - 3, 28])
    sd = O.random_state_dict(1, D, T, R, "peaky", seed=74)
    mod = mp_module(H, D, 1, T, R, sd).eval()
    padded = _mp_call(mod, b)
    adj, Hp, ntp, nsp, rows = ragged_inputs(b["H"], b["edge_index"], b["edge_type"], b["node_type"], b["node_score"],
                                            b["adj_lengths"], n, node_capacity=int(b["adj_lengths"].sum()) + 19)
    adj = adj.to(DEV)

    def call():
        with torch.no_grad():
            out = mod(Hp.to(DEV), adj, ntp.to(DEV), nsp.to(DEV))
        torch.cuda.synchronize()
        return out.cpu()
    rag, names = _profiled(call)
    assert any("mp_headtile_kernel" in s and "true>" in s for s in names), "the ragged tiled kernel did not run"
    assert_extreme_combos(mod._last_prep, T, R, "ragged")
    assert torch.equal(rag[:rows.numel()], padded[rows]), "ragged rows differ from the padded batch's"
    ref = mp_ref(sd, b["H"], b["edge_index"], b["edge_type"], b["node_type"], b["node_score"], 1, T, R, H)
    Hh.assert_close(rag[:rows.numel()], ref[rows], "ragged out")


# ---------------------------------------------------------------------------------------------------------------------
# graph prep
# ---------------------------------------------------------------------------------------------------------------------
PREP_KEYS = ("src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt", "csr_src_tgt", "csr_src_combo",
             "csr_tgt_src", "csr_tgt_combo", "csr_tgt_apos", "csr_src_tpos", "pk_src", "pk_tgt")


def _prep_arrays(prep):
    out = {k: prep.array(k).cpu().numpy().astype(np.int64) for k in PREP_KEYS}
    N = prep.N
    for k in ("order_src", "order_tgt"):
        off = getattr(prep.layout, k)
        out[k] = prep.buf[off:off + 4 * N].view(torch.int32).cpu().numpy().astype(np.int64)
    return out


def _check_prep_against_oracle(got, b, T, R, what, per_graph=True):
    """per_graph: also the words of the per-graph kernels (pk_src / pk_tgt, the degree orders), which a prep writes when it has
    n_per_graph and C <= 65536."""
    nt = b["node_type"].reshape(-1)
    ref = O.graph_prep_oracle(b["edge_index"], b["edge_type"], nt, T, R)
    for key in ("src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt"):
        assert np.array_equal(got[key], ref[key]), f"{what} {key}"
    ps, pt = ref["perm_src"], ref["perm_tgt"]
    assert np.array_equal(got["csr_src_tgt"], ref["tgt"][ps]) and np.array_equal(got["csr_src_combo"], ref["combo"][ps]), what
    assert np.array_equal(got["csr_tgt_src"], ref["src"][pt]) and np.array_equal(got["csr_tgt_combo"], ref["combo"][pt]), what
    inv = np.empty_like(ps)
    inv[ps] = np.arange(len(inv))
    assert np.array_equal(got["csr_tgt_apos"], inv[pt]), what
    inv_t = np.empty_like(pt)
    inv_t[pt] = np.arange(len(inv_t))
    assert np.array_equal(got["csr_src_tpos"], inv_t[ps]), what
    if not per_graph:
        return
    n = b["n"]  # (local endpoint << 16 | combo): the top combo 0xffff must survive the packing
    assert np.array_equal(got["pk_src"], ((ref["tgt"] % n) << 16 | ref["combo"])[ps]), f"{what} pk_src"
    assert np.array_equal(got["pk_tgt"], ((ref["src"] % n) << 16 | ref["combo"])[pt]), f"{what} pk_tgt"
    for name, deg in (("order_src", ref["outdeg"]), ("order_tgt", ref["indeg"])):
        for g in range(len(nt) // n):
            o = got[name][g * n:(g + 1) * n]
            assert sorted(o.tolist()) == list(range(n)), f"{what} {name}"
            assert (np.diff(np.minimum(deg[g * n + o], 255)) <= 0).all(), f"{what} {name}"


def _packed_preps(b, T, R):
    """(packed prep, ragged prep) of batch b; the ragged one at full-length graphs and no spare rows, so its layout is the
    padded one and every array must equal the packed prep's."""
    from qagnn_b200.modeling_qagnn import GraphPrep
    n, B = b["n"], b["node_type"].size(0)
    nt = b["node_type"].reshape(-1).to(DEV)
    pk = Dt.pack_adj(*b["local"], n, pin=False).to(DEV)
    rg = Dt.pack_adj(*b["local"], n, pin=False, adj_lengths=b["adj_lengths"], node_capacity=B * n).to(DEV)
    return (lambda: GraphPrep(pk.edge_index, pk.edge_type, nt, T, R, n, graph_ptr=pk.graph_ptr_dev, max_edges=pk.max_edges),
            lambda: GraphPrep(rg.edge_index, rg.edge_type, nt, T, R, n, graph_ptr=rg.graph_ptr_dev, max_edges=rg.max_edges,
                              node_ptr=rg.node_ptr_dev), rg)


@pytest.mark.gpu
@pytest.mark.parametrize("T,R", PREP_CASES)
def test_graph_prep_at_other_type_counts(T, R):
    b = batch(T, R, 8, seed=T * 7 + R, B=3, n=30, e=200)
    general = _prep(b, T, R, b["n"])
    assert_extreme_combos(general, T, R, "general")
    got = _prep_arrays(general)
    _check_prep_against_oracle(got, b, T, R, "general")
    packed, ragged, _ = _packed_preps(b, T, R)
    for what, mk in (("packed", packed), ("ragged", ragged)):
        p = mk()
        assert p.packed and int(p.status_word().item()) == 0, what
        other = _prep_arrays(p)
        for k in got:
            assert np.array_equal(other[k], got[k]), f"{what} {k}"


@pytest.mark.gpu
def test_graph_prep_refuses_past_16_bit_combos_and_the_module_stays_correct(monkeypatch):
    """(1, 65536), C = 65537: the packed and ragged preps refuse with status -5, a ragged batch gets a ValueError naming the
    combo count, and the module still computes the layer and the message passing through the general prep and basic kernels."""
    from qagnn_b200.modeling_qagnn import graph_prep
    for name in ("QAGNN_MP_PATH", "QAGNN_GEMM", "QAGNN_MP_FASTPROJ", "QAGNN_MP_WARPS"):
        monkeypatch.delenv(name, raising=False)
    T, R = PREP_REFUSED
    H, D = 4, 32
    b = batch(T, R, D, seed=65536, B=3, n=30, e=200)
    packed, ragged, rg = _packed_preps(b, T, R)
    for what, mk in (("packed", packed), ("ragged", ragged)):
        with pytest.raises(_lib.QagnnError) as e:
            mk()
        assert e.value.status == -5, what
    with pytest.raises(ValueError, match=f"{combos(T, R)} edge-feature combos"):
        graph_prep(rg, b["node_type"].reshape(-1).to(DEV), b["n"], T, R, True)

    sd = O.random_state_dict(1, D, T, R, "peaky", seed=5)
    prep = _prep(b, T, R, 0)
    assert_extreme_combos(prep, T, R, "general")
    _check_prep_against_oracle(_prep_arrays(prep), b, T, R, "general", per_graph=False)
    assert mp_path(prep, H, D, T, R) == PATHS["basic"]
    layer = layer_module(H, D, T, R, sd)
    got, names = _profiled(lambda: _layer_call(layer, b, prep))
    assert_path_ran(names, "basic", "layer")
    r = Row(H, D, T, R, "basic")
    _check_layer(got, _layer_refs(r, b, sd), "layer at C = 65537")
    mod = mp_module(H, D, 1, T, R, sd).eval()
    out, names = _profiled(lambda: _mp_call(mod, b))
    assert_path_ran(names, "basic", "message passing")
    assert not mod._last_prep.packed
    ref = mp_ref(sd, b["H"], b["edge_index"], b["edge_type"], b["node_type"], b["node_score"], 1, T, R, H)
    Hh.assert_close(out, ref, "message passing at C = 65537")
    with pytest.raises(ValueError, match=f"{combos(T, R)} edge-feature combos"):
        with torch.no_grad():
            mod(torch.zeros(rg.node_capacity, D, device=DEV), rg, b["node_type"].reshape(-1).to(DEV),
                torch.zeros(rg.node_capacity, 1, device=DEV))


# ---------------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------------
def _mp_train_ref(sd, H_in, ei, et, nt, score, k, T, R):
    """QAGNN_Message_Passing.train() without dropout, fp64 and differentiable: BatchNorm batch statistics (the oracle's
    train=True), the shared edge encoder read from its own keys."""
    D = H_in.size(-1)
    extra = O.node_feature_extra(sd, nt, score, T, D, F64)
    X = H_in.reshape(-1, D)
    for l_ in range(k):
        X = O.gelu_tanh(O.gatconve_forward(sd, f"gnn_layers.{l_}", X, ei, et, nt.reshape(-1), extra, T, R, 4, F64,
                                           edge_encoder_prefix="edge_encoder", train=True)[0])
    return O.gelu_tanh(O.linear(H_in.reshape(-1, D), sd, "Vh") + O.linear(X, sd, "Vx"))


def _train_run(mod, b, G):
    mod.zero_grad(set_to_none=True)
    H = b["H"].to(DEV).requires_grad_(True)
    sc = b["node_score"].to(DEV).requires_grad_(True)
    out = mod(H, (b["edge_index"].to(DEV), b["edge_type"].to(DEV)), b["node_type"].to(DEV), sc)
    (out * G.to(DEV)).sum().backward()
    return [out.detach().cpu(), H.grad.cpu(), sc.grad.cpu()] + [p.grad.cpu() for p in mod.parameters()]


TRAIN_CASES = [(7, 3), (16, 23)]


@pytest.mark.gpu
@pytest.mark.parametrize("T,R", TRAIN_CASES)
def test_training_forward_and_backward_at_other_type_counts(T, R, monkeypatch):
    """.train() forward and backward against fp64 autograd of the oracle; the edge-encoder BatchNorm takes its batch
    statistics over every edge, which the kernels form from the combo table weighted by combo_count.  Under
    torch.use_deterministic_algorithms(True) two runs give the same bits."""
    from tests.test_gpu_eval_grad import _grad_close
    from tests.test_gpu_train_deterministic import _flag
    D, k = 64, 2
    b = batch(T, R, D, seed=T * 31 + R, B=3, n=30, e=90)
    sd = O.random_state_dict(k, D, T, R, "peaky", seed=T + R)
    s64 = {kk: v.double().requires_grad_(True) if v.is_floating_point() else v for kk, v in sd.items()}
    H64, sc64 = b["H"].double().requires_grad_(True), b["node_score"].double().requires_grad_(True)
    ref = _mp_train_ref(s64, H64, b["edge_index"], b["edge_type"], b["node_type"], sc64, k, T, R)
    G = torch.randn(ref.shape, generator=torch.Generator().manual_seed(3), dtype=F64)
    (ref * G).sum().backward()

    mod = mp_module(4, D, k, T, R, sd, dropout=0.0).train()
    got = _train_run(mod, b, G.float().reshape(b["H"].shape))
    assert_extreme_combos(mod._last_prep, T, R, "train")
    Hh.assert_close(got[0].reshape(-1, D), ref, "train-mode out")
    _grad_close(got[1], H64.grad, "dL/dH")
    _grad_close(got[2], sc64.grad, "dL/dnode_score")
    names = [kk for kk, _ in mod.named_parameters()]
    gmax = max(float(s64[kk].grad.abs().max()) for kk in names if s64[kk].grad is not None)
    for kk, g_ in zip(names, got[3:]):
        _grad_close(g_, s64[kk].grad, f"dL/d{kk}", floor=1e-2 * gmax)

    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    with _flag(True):
        runs = [_train_run(mod, b, G.float().reshape(b["H"].shape)) for _ in range(2)]
    for i, (a, c) in enumerate(zip(*runs)):
        assert torch.equal(a, c), f"tensor {i} differs between two deterministic runs"


@pytest.mark.gpu
@pytest.mark.parametrize("T,R", TRAIN_CASES)
def test_core_backward_writes_every_combo_row(T, R):
    """dKe / dMe over all C rows through the CUDA core against fp64 autograd: the rows of combos without edges are exact
    zeros, the others within the core's bar (tests/test_gpu_heads.py)."""
    from qagnn_b200 import training as TR
    H, D = 4, 64
    b = batch(T, R, D, seed=T * 17 + R, B=3, n=30, e=90)
    ei, et, nt = b["edge_index"], b["edge_type"], b["node_type"].reshape(-1)
    N, C_ = nt.numel(), combos(T, R)
    g = torch.Generator().manual_seed(T + R)
    qkm = torch.randn(N, 3 * D, generator=g)
    qkm[:, :D] /= (D // H) ** 0.5
    ke, me, G = torch.randn(C_, D, generator=g), torch.randn(C_, D, generator=g), torch.randn(N, D, generator=g)
    prep = _prep(b, T, R, 0)
    leaves = [t.to(DEV).requires_grad_(True) for t in (qkm, ke, me)]
    aggr, alpha = TR._MPCore.apply(*leaves, prep, (N, ei.size(1), D, H, T, R), True)
    grads = torch.autograd.grad(aggr, leaves, G.to(DEV), retain_graph=True)
    grads2 = torch.autograd.grad(aggr, leaves, G.to(DEV))
    ref_leaves = [t.double().requires_grad_(True) for t in (qkm, ke, me)]
    raggr, ralpha = mp_core_ref(*ref_leaves, *_edges(ei, et, nt, T, R), H)
    rgrads = torch.autograd.grad(raggr, ref_leaves, G.double())
    cpu = lambda ts: [t.detach().cpu() for t in ts]  # noqa: E731
    _check_core(dict(got=cpu([aggr, alpha, *grads]), again=cpu(grads2), ref=[raggr.detach(), ralpha.detach(), *rgrads]),
                D, "random")
    used = torch.zeros(C_, dtype=torch.bool)
    used[_edges(ei, et, nt, T, R)[2]] = True
    assert not bool(used.all()), "every combo has an edge: nothing to check"
    for name, g_ in (("dKe", grads[1]), ("dMe", grads[2])):
        assert bool((g_.cpu()[~used] == 0).all()), f"{name}: a combo without edges has a non-zero row"


@pytest.mark.gpu
@pytest.mark.parametrize("TR_,accepted", COMBO_SORT_CASES, ids=["c6144", "c6145"])
def test_combo_sort_at_its_limit(TR_, accepted):
    """C = 6144 sorts every edge like a stable numpy argsort of the by-source combos; C = 6145 raises QagnnError."""
    T, R = TR_
    b = batch(T, R, 8, seed=6144, B=4, n=100, e=6000)
    prep = _prep(b, T, R, 0)
    assert_extreme_combos(prep, T, R, "combo sort")
    if not accepted:
        with pytest.raises(_lib.QagnnError):
            prep.combo_sort()
        return
    count, order = prep.combo_sort()
    by_src = prep.array("csr_src_combo").cpu().numpy().astype(np.int64)
    Ep = prep.N + prep.E
    assert np.array_equal(order[:Ep].cpu().numpy(), np.argsort(by_src, kind="stable"))
    assert np.array_equal(count.cpu().numpy(), np.bincount(by_src, minlength=combos(T, R)))
