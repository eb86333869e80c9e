"""The eval forward under bf16 autocast (include/qagnn_b200.h, qagnn_mp_forward_typed / qagnn_gatconve_forward_typed).

Contract: every GEMM of the fp32 tensor-core path takes bf16_rn of the operands that path feeds it (the folded weights
included) and accumulates in fp32; everything that is not a GEMM operand (the folds, Ke / Me, Q|Kx|Mx, logits, softmax,
aggr) stays fp32.  The tests check
  * the single-pass GEMM against the split-bf16 GEMM on bf16-representable operands (every lo plane is zero, so the two
    must agree bit for bit), and the fused single-pass MLP against its two-launch form;
  * layers and whole forwards against an fp64 emulation of the contract that follows the path that runs, with bars in
    bf16 units that the test shows to reject the fp32 forward, unrounded weights, rounded Ke / Me and swapped heads;
  * shapes without the wgmma GEMM (D % 8 != 0, QAGNN_GEMM=ffma): the fp32 path rounded, bit for bit;
  * determinism, CUDA-graph replay and DecoderStep capture;
  * the decoder head / tail kernels under autocast (they read fp32 operands; failed before this mode existed).
"""
import ctypes
import math

import pytest
import torch

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200 import _lib, ops
from qagnn_b200.data import PackedAdj
from tests import helpers as Hh

DEV = "cuda:0"
BF = torch.bfloat16
U = 2.0 ** -8  # one bf16 unit (relative spacing of the 8-bit significand)


def _autocast():
    return torch.autocast("cuda", dtype=BF)


def bf(t):
    """bf16_rn of an fp32 (or fp64) tensor, as fp64"""
    return t.float().to(BF).double()


# ------------------------------------------------------------------------------------------------------------------------
# 1. the single-pass GEMM against the split GEMM on bf16-representable operands
# ------------------------------------------------------------------------------------------------------------------------
def _bf16_operands(M, N, K1, K2, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a1 = (torch.randn(M, K1, device=DEV, generator=g) * 0.5).to(BF)
    a2 = (torch.randn(M, K2, device=DEV, generator=g) * 0.5).to(BF) if K2 else None
    w = (torch.randn(N, K1 + K2, device=DEV, generator=g) / (K1 + K2) ** 0.5).to(BF)
    b = torch.randn(N, device=DEV, generator=g) * 0.1
    return a1, a2, w, b


def _gemm_pair(monkeypatch, M, N, K1, K2, act, ctas, store, seed=0):
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    monkeypatch.setenv("QAGNN_TC_STORE", store)
    a1, a2, w, b = _bf16_operands(M, N, K1, K2, seed)
    single = ops.linear_bf16(a1, w, b, a2, act)
    plane = ops.linear_bf16(a1, w, b, a2, act, out_dtype=BF)
    split = ops.linear_bf16x3(a1.float(), w.float(), b, a2.float() if a2 is not None else None, act)
    torch.cuda.synchronize()
    return single, plane, split


@pytest.mark.gpu
@pytest.mark.parametrize("store", ["tma", "direct"])
@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("act", ["none", "relu", "gelu"])
@pytest.mark.parametrize("N", [40, 120, 200, 256])  # wgmma widths 64, 128, 208, 256
def test_single_pass_equals_split_on_bf16_operands(monkeypatch, N, act, ctas, store):
    """hi*lo and lo*hi products of zero lo planes add exact zeros: the single pass must give the split GEMM's bits."""
    single, plane, split = _gemm_pair(monkeypatch, 300, N, 200, 104, act, ctas, store)
    assert torch.equal(single, split)
    assert torch.equal(plane, single.to(BF)), "the bf16 plane output is not RNE of the fp32 output"


@pytest.mark.gpu
@pytest.mark.parametrize("K2", [0, 104])
@pytest.mark.parametrize("K1", [8, 72, 200, 296])
def test_single_pass_k_tails(monkeypatch, K1, K2):
    """K off the k-block and k16 grids, one and two A segments."""
    for ctas in ("1", "0"):
        single, plane, split = _gemm_pair(monkeypatch, 257, 208, K1, K2, "gelu", ctas, "tma", seed=K1 + K2)
        assert torch.equal(single, split), f"K={K1}+{K2} CTAS={ctas}"
        assert torch.equal(plane, single.to(BF))


# ------------------------------------------------------------------------------------------------------------------------
# helpers: modules from the goldens' inputs and weights
# ------------------------------------------------------------------------------------------------------------------------
def _mp_case(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    mod = qagnn_b200.QAGNN_Message_Passing(None, c["k"], fx["n_ntype"], fx["n_etype"], c["D"], c["D"], c["D"]).eval()
    mod.load_state_dict(sd, strict=True)
    mod = mod.to(DEV)
    d = {k: v.to(DEV) for k, v in inp.items()}
    return fx, inp, sd, mod, d


def _run_mp(mod, d, **kw):
    with torch.no_grad(), _autocast():
        return mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], **kw)


def _layer_case(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    x, extra, node_type, ei, et, sd = Hh.regen_layer_inputs(fx)
    D = c["D"]
    enc = torch.nn.Sequential(torch.nn.Linear(fx["n_etype"] + 1 + fx["n_ntype"] * 2, D), torch.nn.BatchNorm1d(D),
                              torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, fx["n_ntype"], fx["n_etype"], enc, head_count=c["H"]).eval()
    layer.load_state_dict({k[len("gnn_layers.0."):]: v for k, v in sd.items() if k.startswith("gnn_layers.0.")}, strict=True)
    return fx, (x, extra, node_type, ei, et), sd, layer.to(DEV)


# ------------------------------------------------------------------------------------------------------------------------
# 3. fp64 emulation of the contract
# ------------------------------------------------------------------------------------------------------------------------
class Variant:
    """What the emulation does; the defaults are the contract, the others are what the bars must reject."""

    def __init__(self, round_weights=True, round_tables=False, swap_heads=False):
        self.round_weights, self.round_tables, self.swap_heads = round_weights, round_tables, swap_heads


def _w(t, v):
    return bf(t) if v.round_weights else t.double()


def _emulate_layer(sd, prefix, ee, x_b, ex_b, ei, et, nt, n_ntype, n_etype, H, v, type_bias=None):
    """One GATConvE layer (before mp_helper's GELU) from bf16 inputs x_b / ex_b (fp64 tensors holding bf16 values).
    type_bias: None = the general projection ([x | extra] operand); else (type_emb [N, D/2] fp64) for the fast form, where
    ex_b holds [0 | score_emb] and the type-embedding columns enter as fp32 bias rows.  Returns (out, mag, rss) with mag /
    rss = sum / root-sum-square of |hidden_j * W2[c, j]| per output element (the last GEMM's magnitude)."""
    N, D = x_b.shape
    d = D // H
    g = lambda k: sd[f"{prefix}.{k}"].double()  # noqa: E731
    inv = float(torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(d), dtype=torch.float32)))
    wq = (sd[f"{prefix}.linear_query.weight"] * inv)  # fp32, as the fold computes it
    wk, wm = sd[f"{prefix}.linear_key.weight"], sd[f"{prefix}.linear_msg.weight"]
    Wp = torch.cat([wq, wk[:, :2 * D], wm[:, :2 * D]])  # [3D, 2D] fp32
    bp = torch.cat([(sd[f"{prefix}.linear_query.bias"] * inv).double(), torch.zeros(2 * D, dtype=torch.float64)])
    if type_bias is None:
        A = torch.cat([x_b, ex_b], 1)
        qkm = A @ _w(Wp, v).t() + bp
    else:  # fast form: [x | score_emb] rounded, the type columns [D, D + D/2) exact in fp32 bias rows
        Dh = D // 2
        A = torch.cat([x_b, ex_b[:, Dh:]], 1)
        Wx = torch.cat([Wp[:, :D], Wp[:, D + Dh:]], 1)
        qkm = A @ _w(Wx, v).t() + bp + type_bias @ Wp[:, D:D + Dh].double().t()
    Q, Kx, Mx = qkm[:, :D], qkm[:, D:2 * D], qkm[:, 2 * D:]
    # edge table part (exact fp32 folds; rounded only in the variant the bars must reject)
    f64 = torch.float64
    edge_vec = torch.cat([O.make_one_hot(et, n_etype + 1, f64), torch.zeros(N, n_etype + 1, dtype=f64).index_fill_(1, torch.tensor([n_etype]), 1.0)])
    hv = torch.cat([O.make_one_hot(nt[ei[0]], n_ntype, f64), O.make_one_hot(nt[ei[1]], n_ntype, f64)], 1)
    sv = O.make_one_hot(nt, n_ntype, f64)
    headtail = torch.cat([hv, torch.cat([sv, sv], 1)])
    emb = O.mlp_lin_bn_relu_lin(torch.cat([edge_vec, headtail], 1), {k: t.double() for k, t in sd.items()}, ee)
    Ke = emb @ wk[:, 2 * D:].double().t() + g("linear_key.bias")
    Me = emb @ wm[:, 2 * D:].double().t() + g("linear_msg.bias")
    if v.round_tables:
        Ke, Me = bf(Ke), bf(Me)
    loop = torch.arange(N).unsqueeze(0).repeat(2, 1)
    src, tgt = torch.cat([ei, loop], 1)
    key = (Kx[tgt] + Ke).view(-1, H, d)
    msg = (Mx[src] + Me).view(-1, H, d)
    query = Q[src].view(-1, H, d)
    alpha = O.segment_softmax((query * key).sum(2), src)
    if v.swap_heads and H > 1:
        alpha = alpha[:, [1, 0] + list(range(2, H))]
    cnt = O.scatter_sum(torch.ones(src.numel(), dtype=f64), src, N)[src]
    aggr = O.scatter_sum((msg * (alpha * cnt.unsqueeze(1)).unsqueeze(2)).view(-1, D), tgt, N)
    # node MLP with the BatchNorm folded into mlp.0 (fp32 fold), hidden layer rounded (the GEMM2 A operand)
    gm, bt = sd[f"{prefix}.mlp.1.weight"], sd[f"{prefix}.mlp.1.bias"]
    mu, var = sd[f"{prefix}.mlp.1.running_mean"], sd[f"{prefix}.mlp.1.running_var"]
    sc = gm / torch.sqrt(var + 1e-5)
    w1 = sd[f"{prefix}.mlp.0.weight"] * sc.unsqueeze(1)
    b1 = ((sd[f"{prefix}.mlp.0.bias"] - mu) * sc + bt).double()
    h = bf(torch.relu(bf(aggr) @ _w(w1, v).t() + b1))
    w2 = _w(sd[f"{prefix}.mlp.3.weight"], v)
    out = h @ w2.t() + g("mlp.3.bias")
    prod = h.abs() @ w2.abs().t()
    rss = ((h * h) @ (w2 * w2).t()).sqrt()
    return out, prod, rss


def _bars_hold(got, emu, mag, rss, ulp_out=False):
    """(ok, fraction over the tight bar, worst ratio to the loose bar).  Tight: fp32 accumulation (2^-18 of the
    magnitude) - all but a few elements, those where an fp32 difference flipped a rounding to bf16 upstream (at most 5%).
    Loose: such flips, a few bf16 units of the root-sum-square magnitude.  ulp_out (a bf16-rounded output): plus one unit
    of the output, and up to 15% of the elements may differ - an fp32 difference far below one unit still crosses a
    rounding boundary now and then (7% at D = 1024, where each output sums 1024 hidden products)."""
    got, emu = got.detach().double().cpu(), emu.double().cpu()
    err = (got - emu).abs()
    tight = 2.0 ** -18 * mag + 2.0 ** -14 * emu.abs()
    loose = 4 * U * rss + 2.0 ** -18 * mag + (U * emu.abs() if ulp_out else 0)
    frac = (err > tight).double().mean().item() if err.numel() else 0.0
    worst = (err / loose).max().item() if err.numel() else 0.0
    return frac <= (0.15 if ulp_out else 0.05) and worst <= 1.0, frac, worst


def _gelu_bars(out, mag, rss):
    return O.gelu_tanh(out), 1.13 * mag, 1.13 * rss  # GELU's slope stays below 1.13


def _layer_emulation(fx, tensors, sd, v):
    c = fx["case"]
    x, extra, node_type, ei, et = tensors
    ee = "gnn_layers.0.edge_encoder" if "gnn_layers.0.edge_encoder.0.weight" in sd else "edge_encoder"
    return _emulate_layer(sd, "gnn_layers.0", ee, bf(x), bf(extra), ei, et, node_type, fx["n_ntype"], fx["n_etype"],
                          c["H"], v)


LAYER_GOLDENS = ["layer_h8_d1024", "layer_hub", "layer_single_node", "layer_multi_dup", "layer_h4_d200_prod",
                 "layer_src_only_tgt_only"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["auto", "csr", "basic"])
@pytest.mark.parametrize("name", LAYER_GOLDENS)
def test_layer_matches_emulation(monkeypatch, name, path):
    if path != "auto":
        monkeypatch.setenv("QAGNN_MP_PATH", path)
    fx, tensors, sd, layer = _layer_case(name)
    x, extra, node_type, ei, et = tensors
    with torch.no_grad(), _autocast():
        out, (_, alpha) = layer(x.to(DEV), ei.to(DEV), et.to(DEV), node_type.to(DEV), extra.to(DEV),
                                return_attention_weights=True)
    assert out.dtype == BF and alpha.dtype == torch.float32
    emu, mag, rss = _layer_emulation(fx, tensors, sd, Variant())
    ok, frac, worst = _bars_hold(out, bf(emu), mag, rss, ulp_out=True)
    assert ok, f"{name}/{path}: {frac:.3f} of the elements over the tight bar, worst {worst:.2f} of the loose bar"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["layer_h4_d200_prod", "layer_h8_d1024"])
def test_layer_bars_reject(name):
    """The bars see the fp32 forward, unrounded weights, rounded Ke / Me and two swapped heads."""
    fx, tensors, sd, layer = _layer_case(name)
    x, extra, node_type, ei, et = tensors
    args = (x.to(DEV), ei.to(DEV), et.to(DEV), node_type.to(DEV), extra.to(DEV))
    with torch.no_grad():
        out32 = layer(*args)
        with _autocast():
            out16 = layer(*args)
    emu, mag, rss = _layer_emulation(fx, tensors, sd, Variant())
    assert not _bars_hold(out32.to(BF), bf(emu), mag, rss, ulp_out=True)[0], "the fp32 forward passes the bf16 bars"
    for v in (Variant(round_weights=False), Variant(round_tables=True), Variant(swap_heads=True)):
        e, m, r = _layer_emulation(fx, tensors, sd, v)
        assert not _bars_hold(out16, bf(e), m, r, ulp_out=True)[0], vars(v)


def _emulate_mp(fx, inp, sd, fast, teacher_layers=None, v=None, H=4, k=None):
    """QAGNN_Message_Passing under the contract; teacher_layers: the kernel's fp32 layer outputs, each layer then starts
    from the previous kernel layer rounded.  H: the layers' head count (the module builds them with GATConvE's default, 4);
    k: the layer count (default the case's); at k = 0 the output is GELU(Vh(H) + Vx(H)).  Returns (out, mag, rss, layers)
    with per-layer (x, mag, rss)."""
    v = v or Variant()
    c = fx["case"]
    D, k = c["D"], c["k"] if k is None else k
    n_ntype, n_etype = fx["n_ntype"], fx["n_etype"]
    sdd = {kk: t.double() for kk, t in sd.items()}
    nt = inp["node_type"].reshape(-1)
    H0 = bf(inp["H"].reshape(-1, D))
    type_emb = O.gelu_tanh(O.make_one_hot(nt, n_ntype, torch.float64) @ sdd["emb_node_type.weight"].t() + sdd["emb_node_type.bias"])
    js = torch.pow(1.1, torch.arange(D // 2).float())
    sinb = torch.sin((js * inp["node_score"].reshape(-1, 1).float()).double())
    if fast:  # emb_score on the single-pass GEMM: rounded sin basis and weight
        score_emb = bf(O.gelu_tanh(bf(sinb) @ _w(sd["emb_score.weight"], v).t() + sdd["emb_score.bias"]))
        ex_b = torch.cat([torch.zeros_like(type_emb), score_emb], 1)
    else:
        ex_b = bf(torch.cat([type_emb, O.gelu_tanh(sinb @ sdd["emb_score.weight"].t() + sdd["emb_score.bias"])], 1))
    x_b, layers = H0, []
    for l in range(k):
        out, mag, rss = _emulate_layer(sd, f"gnn_layers.{l}", "edge_encoder", x_b, ex_b, inp["edge_index"], inp["edge_type"], nt,
                                       n_ntype, n_etype, H, v, type_bias=type_emb if fast else None)
        X, mag, rss = _gelu_bars(out, mag, rss)
        layers.append((X, mag, rss))
        x_b = bf(teacher_layers[l].cpu()) if teacher_layers is not None else bf(X)
    wv = torch.cat([_w(sd["Vh.weight"], v), _w(sd["Vx.weight"], v)], 1)
    A = torch.cat([H0, x_b], 1)
    out, mag, rss = _gelu_bars(A @ wv.t() + sdd["Vh.bias"] + sdd["Vx.bias"], A.abs() @ wv.abs().t(), ((A * A) @ (wv * wv).t()).sqrt())
    return out, mag, rss, layers


def _whole_forward_holds(got, emu, mag, rss):
    """The whole forward without teacher forcing: layer differences compound, so a few units more on the output."""
    err = (got.detach().double().cpu() - bf(emu)).abs()
    return bool((err <= 16 * U * rss + U * bf(emu).abs() + 2.0 ** -18 * mag).all())


MP_GOLDENS = ["cfg2small_prod", "cfg2small_realistic", "cfg1_peaky_k2", "no_edges", "cfg1_prod"]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fast", "fastproj0", "csr", "basic"])
@pytest.mark.parametrize("name", MP_GOLDENS)
def test_forward_matches_emulation(monkeypatch, name, mode):
    """Teacher-forced per layer, and the whole forward: the fast form (default on the tiled path) with the type embedding
    in fp32 bias rows, the general [x | extra] projection (QAGNN_MP_FASTPROJ=0) and the sliced / basic CSR paths."""
    if mode == "fastproj0":
        monkeypatch.setenv("QAGNN_MP_FASTPROJ", "0")
    elif mode in ("csr", "basic"):
        monkeypatch.setenv("QAGNN_MP_PATH", mode)
    fx, inp, sd, mod, d = _mp_case(name)
    out, layers = _run_mp(mod, d, return_layers=True)
    # the fast form runs on the tiled path (QAGNN_MP_PATH_TILED = 0) when D/2 is a multiple of 4
    prep = mod._last_prep
    tiled = _lib.load().qagnn_mp_path(ctypes.byref(mod._shape(prep.N, prep.E, prep.n_per_graph))) == 0
    fast = mode == "fast" and tiled and (fx["case"]["D"] // 2) % 4 == 0
    assert out.dtype == BF and layers.dtype == torch.float32
    emu, mag, rss, emu_layers = _emulate_mp(fx, inp, sd, fast, teacher_layers=layers)
    D = fx["case"]["D"]
    for l, (X, m, r) in enumerate(emu_layers):
        ok, frac, worst = _bars_hold(layers[l].view(-1, D), X, m, r)
        assert ok, f"{name}/{mode} layer {l}: {frac:.3f} over the tight bar, worst {worst:.2f} of the loose bar"
    ok, frac, worst = _bars_hold(out.view(-1, D), bf(emu), mag, rss, ulp_out=True)
    assert ok, f"{name}/{mode} out: {frac:.3f} over the tight bar, worst {worst:.2f} of the loose bar"
    emu2, mag2, rss2, _ = _emulate_mp(fx, inp, sd, fast)
    assert _whole_forward_holds(out.view(-1, D), emu2, mag2, rss2), f"{name}/{mode}: the whole forward"
    # and the fp32 forward is not within the bars
    with torch.no_grad():
        _, layers32 = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    assert not _bars_hold(layers32[0].view(-1, D), *emu_layers[0])[0]


# ------------------------------------------------------------------------------------------------------------------------
# 2. fused MLP, 4. shapes without the wgmma GEMM, 5. replay and determinism
# ------------------------------------------------------------------------------------------------------------------------
def _synth_layer(D, N=300, E=1500, seed=3):
    """a GATConvE layer (4 heads) with seeded weights and BatchNorm statistics, and a random graph"""
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    enc = torch.nn.Sequential(torch.nn.Linear(38 + 1 + 8, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, 4, 38, enc, head_count=4).eval()
    bn = layer.mlp[1]
    bn.running_mean.uniform_(-0.2, 0.2, generator=g)
    bn.running_var.uniform_(0.5, 2.0, generator=g)
    layer = layer.to(DEV)
    x = torch.randn(N, D, generator=g) * 0.5
    extra = torch.randn(N, D, generator=g) * 0.5
    nt = torch.randint(0, 4, (N,), generator=g)
    ei = torch.randint(0, N, (2, E), generator=g)
    et = torch.randint(0, 38, (E,), generator=g)
    return layer, [t.to(DEV) for t in (x, ei, et, nt, extra)]


@pytest.mark.gpu
@pytest.mark.parametrize("D", [8, 64, 200, 208])
def test_fused_mlp_equals_two_launches(monkeypatch, D):
    """The single-pass fused node MLP (hidden layer as one bf16 fragment in registers) gives the bits of mlp.0 writing the
    hidden hi plane and mlp.3 reading it (QAGNN_MLP_FUSED=0), with CTA pairs and single CTAs."""
    layer, args = _synth_layer(D)
    outs = {}
    for ctas in ("1", "0"):
        monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
        for fused in ("1", "0"):
            monkeypatch.setenv("QAGNN_MLP_FUSED", fused)
            with torch.no_grad(), _autocast():
                outs[ctas, fused] = layer(*args)
    ref = outs["1", "1"]
    assert ref.dtype == BF
    for key, o in outs.items():
        assert torch.equal(o, ref), key


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["d100", "ffma"])
def test_shapes_without_wgmma_round_the_fp32_path(monkeypatch, case):
    name = "tiny_realistic_d100" if case == "d100" else "cfg2small_prod"
    if case == "ffma":
        monkeypatch.setenv("QAGNN_GEMM", "ffma")
    fx, inp, sd, mod, d = _mp_case(name)
    Hb = d["H"].to(BF)
    adj = (d["edge_index"], d["edge_type"])
    with torch.no_grad():
        ref, ref_layers = mod(Hb.float(), adj, d["node_type"], d["node_score"], return_layers=True)
        with _autocast():
            out, layers = mod(Hb, adj, d["node_type"], d["node_score"], return_layers=True)
            out_f32_in = mod(d["H"], adj, d["node_type"], d["node_score"])
    assert out.dtype == BF
    assert torch.equal(out, ref.to(BF))
    assert torch.equal(layers, ref_layers)
    assert torch.equal(out_f32_in, out), "an fp32 H is rounded once on entry"


@pytest.mark.gpu
def test_reruns_replay_and_edge_capacity_are_bit_identical():
    fx, inp, sd, mod, d = _mp_case("cfg2small_prod")
    adj = (d["edge_index"], d["edge_type"])
    a = _run_mp(mod, d)
    b = _run_mp(mod, d)
    assert torch.equal(a, b)
    mod.use_cuda_graph = True
    with torch.no_grad():
        with _autocast():
            g16 = mod(d["H"], adj, d["node_type"], d["node_score"]).clone()
            g16b = mod(d["H"], adj, d["node_type"], d["node_score"]).clone()
        g32 = mod(d["H"], adj, d["node_type"], d["node_score"]).clone()
        with _autocast():
            g16c = mod(d["H"], adj, d["node_type"], d["node_score"]).clone()
    mod.use_cuda_graph = False
    with torch.no_grad():
        e32 = mod(d["H"], adj, d["node_type"], d["node_score"])
    assert g16.dtype == BF and g32.dtype == torch.float32
    assert torch.equal(g16, a) and torch.equal(g16b, a) and torch.equal(g16c, a)
    assert torch.equal(g32, e32)
    # the same batch packed at an edge capacity (spare edge columns) and packed exactly
    n, B = fx["case"]["n"], fx["case"]["B"]
    cnt = torch.bincount(inp["edge_index"][0] // n, minlength=B)
    gp = torch.zeros(B + 1, dtype=torch.long)
    gp[1:] = torch.cumsum(cnt, 0)
    E = inp["edge_index"].size(1)
    cap = E + 37
    ei = torch.zeros(2, cap, dtype=torch.long)
    et = torch.zeros(cap, dtype=torch.long)
    ei[:, :E], et[:E] = inp["edge_index"], inp["edge_type"]
    me = int(cnt.max())
    pa_cap = PackedAdj(ei.to(DEV), et.to(DEV), None, n, None, gp.to(DEV), me, -1, cap)
    pa_exact = PackedAdj(d["edge_index"], d["edge_type"], None, n, None, gp.to(DEV), me, -1, E)
    with torch.no_grad(), _autocast():
        o_cap = mod(d["H"], pa_cap, d["node_type"], d["node_score"])
        o_exact = mod(d["H"], pa_exact, d["node_type"], d["node_score"])
    assert torch.equal(o_cap, o_exact)
    assert torch.equal(o_exact, a)


def _decoder(name="decoder_small"):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    dec = qagnn_b200.QAGNN(None, c["k"], fx["n_ntype"], fx["n_etype"], c["sent_dim"], c["n_concept"], c["D"],
                           c["concept_in_dim"], c["n_head"], c["D"], c["n_fc_layer"], 0.2, 0.2, 0.2).eval()
    dec.load_state_dict(fx["state_dict"], strict=True)
    dec = dec.to(DEV)
    d = {k: v.to(DEV) for k, v in inp.items()}
    args = (sent_vecs.to(DEV), concept_ids.to(DEV), d["node_type"], d["node_score"], d["adj_lengths"],
            (d["edge_index"], d["edge_type"]))
    return fx, dec, args, d


@pytest.mark.gpu
def test_decoder_step_capture_equals_eager_under_autocast():
    from qagnn_b200.pipeline import DecoderStep
    fx, dec, args, d = _decoder()
    sent, cids, nt, ns, al, adj = args
    with torch.no_grad(), _autocast():
        H, s = _head_input(dec, args)
    inputs = {"H": H.contiguous(), "edge_index": d["edge_index"], "edge_type": d["edge_type"], "node_type": nt,
              "node_score": s.contiguous(), "sent_vecs": sent, "adj_lengths": al}
    step = DecoderStep(dec.gnn, dec.pooler, dec.fc, inputs, autocast_dtype=BF)
    logits, attn, gnn_out = [t.clone() for t in step.run()]
    eager = DecoderStep(dec.gnn, dec.pooler, dec.fc, inputs, use_cuda_graph=False, autocast_dtype=BF)
    le, ae, ge = eager.run()
    assert gnn_out.dtype == BF
    assert torch.equal(logits, le) and torch.equal(attn, ae) and torch.equal(gnn_out, ge)
    ref32 = DecoderStep(dec.gnn, dec.pooler, dec.fc, inputs)
    l32, _, g32 = [t.clone() for t in ref32.run()]
    assert g32.dtype == torch.float32
    logits2, _, gnn_out2 = step.run()
    assert torch.equal(gnn_out2, gnn_out) and torch.equal(logits2, logits), "an fp32 capture disturbed the bf16 one"


# ------------------------------------------------------------------------------------------------------------------------
# 6. the decoder head / tail kernels under autocast
# ------------------------------------------------------------------------------------------------------------------------
def _head_input(dec, args):
    """(gnn_input, s) of the fused head: what QAGNN.pooled_features hands the message passing"""
    seen = {}
    orig = dec.gnn.forward

    def spy(H, A, node_type, node_score, *a, **kw):
        seen["H"], seen["s"] = H, node_score
        return orig(H, A, node_type, node_score, *a, **kw)

    dec.gnn.forward = spy
    try:
        dec(*args)
    finally:
        dec.gnn.forward = orig
    return seen["H"], seen["s"]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fused_head_under_autocast(dtype):
    fx, dec, args, d = _decoder()
    sent, cids, nt, ns, al, adj = args
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
        H, _ = _head_input(dec, args)
        # the PyTorch head (modeling_qagnn.py:153-160) under the same autocast: torch.cat promotes to fp32
        g0 = dec.activation(dec.svec2nvec(sent)).unsqueeze(1)
        g1 = dec.concept_emb(cids[:, 1:] - 1, None)
        ref = torch.cat([g0, g1], 1)
    assert H.dtype == torch.float32 and ref.dtype == torch.float32
    assert torch.equal(H, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("xdtype", [torch.float32, torch.bfloat16])
def test_fused_tail_under_autocast(xdtype):
    """concat and attention of the one-kernel tail (and the fused pooling) under bf16 autocast, with fp32 or bf16 node
    features, against the einsum path in fp64 on the same operands (qs rounded by autocast, X widened)."""
    fx, dec, args, d = _decoder()
    sent, cids, nt, ns, al, adj = args
    pool = dec.pooler
    g = torch.Generator(device=DEV).manual_seed(5)
    B, n, D = sent.size(0), nt.size(1), dec.concept_dim
    X = torch.randn(B, n, D, device=DEV, generator=g).to(xdtype)
    with torch.no_grad(), _autocast():
        concat, attn = pool.pool_concat(sent, X, nt, al)
        qs = pool.w_qs(sent)
    pos = torch.arange(n, device=DEV)
    mask = (pos >= al.unsqueeze(1)) | (nt == 3)
    mask[:, 0] = mask[:, 0] & ~mask.all(1)
    with torch.no_grad(), _autocast():
        pooled, attn2 = pool(sent, X, mask)
    nh, dk = pool.n_head, pool.d_k
    Xd, qd = X.double(), qs.double().view(B, nh, dk)
    ks = (Xd @ pool.w_ks.weight.double().t() + pool.w_ks.bias.double()).view(B, n, nh, dk)
    vs = (Xd @ pool.w_vs.weight.double().t() + pool.w_vs.bias.double()).view(B, n, nh, dk)
    logits = torch.einsum("bhd,blhd->hbl", qd, ks) / math.sqrt(dk)
    a = torch.softmax(logits.masked_fill(mask.unsqueeze(0), float("-inf")), 2)
    ref_pooled = torch.einsum("hbl,blhd->bhd", a, vs).reshape(B, nh * dk)
    ref_concat = torch.cat([ref_pooled, sent.double(), Xd[:, 0]], 1)
    Hh.assert_close(attn, a.reshape(nh * B, n), "attn")
    Hh.assert_close(concat, ref_concat, "concat")
    Hh.assert_close(attn2, a.reshape(nh * B, n), "attn (fused pooling)")
    Hh.assert_close(pooled, ref_pooled, "pooled (fused pooling)")


@pytest.mark.gpu
def test_fp32_eval_after_autocast_eval_is_unchanged():
    """The concept table is built and cached in fp32 whatever autocast the first call runs under; concept_in_dim = 30
    takes the plain PyTorch projection (the split GEMM wants K % 8 == 0), which autocast would run in half precision."""
    fx = Hh.load_golden("decoder_small")
    c = dict(fx["case"], concept_in_dim=30)
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    torch.manual_seed(0)
    dec = qagnn_b200.QAGNN(None, c["k"], fx["n_ntype"], fx["n_etype"], c["sent_dim"], c["n_concept"], c["D"], 30,
                           c["n_head"], c["D"], c["n_fc_layer"], 0.2, 0.2, 0.2).eval().to(DEV)
    d = {k: v.to(DEV) for k, v in inp.items()}
    args = (sent_vecs.to(DEV), concept_ids.to(DEV), d["node_type"], d["node_score"], d["adj_lengths"],
            (d["edge_index"], d["edge_type"]))
    with torch.no_grad():
        before = dec(*args)[0].clone()
        for dtype in (torch.float16, torch.bfloat16):
            dec.concept_emb.invalidate_table()
            with torch.autocast("cuda", dtype=dtype):
                dec(*args)
            after = dec(*args)[0]
            assert torch.equal(after, before), dtype
