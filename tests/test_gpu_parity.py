"""Parity of the CUDA path (through the C ABI) against the goldens minted from the reference and
against the CPU oracle.  Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200.modeling_qagnn import GraphPrep
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mp_module(c, fx, sd):
    mod = qagnn_b200.QAGNN_Message_Passing(None, c["k"], fx["n_ntype"], fx["n_etype"], c["D"], c["D"], c["D"]).eval()
    mod.load_state_dict(sd, strict=True)
    return mod.to(DEV)


def _dev(inp):
    return {k: v.to(DEV) for k, v in inp.items()}


def _graph_ptr(edge_index, n, B):
    """first edge of every sub-graph of a batch whose edges are laid out graph by graph"""
    cnt = torch.bincount(edge_index[0] // n, minlength=B)
    gp = torch.zeros(B + 1, dtype=torch.long)
    gp[1:] = torch.cumsum(cnt, 0)
    return gp


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_graph_prep_bit_exact(name, packed):
    """packed=True: the one-launch per-sub-graph kernel (qagnn_graph_prep_packed) must give the same arrays, bit for bit."""
    fx = Hh.load_golden(name)
    inp, _ = Hh.regen_mp_inputs(fx)
    d = _dev(inp)
    kw = {}
    if packed:
        gp = _graph_ptr(inp["edge_index"], fx["case"]["n"], fx["case"]["B"])
        kw = dict(graph_ptr=gp.to(DEV), max_edges=int((gp[1:] - gp[:-1]).max()) if gp.numel() > 1 else 0)
    prep = GraphPrep(d["edge_index"], d["edge_type"], d["node_type"], fx["n_ntype"], fx["n_etype"], fx["case"]["n"], **kw)
    ref = O.graph_prep_oracle(inp["edge_index"], inp["edge_type"], inp["node_type"], fx["n_ntype"], fx["n_etype"])
    got = {k: prep.array(k).cpu().numpy().astype(np.int64) for k in
           ("src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt", "csr_src_tgt", "csr_src_combo",
            "csr_tgt_src", "csr_tgt_combo", "csr_tgt_apos", "csr_src_tpos", "pk_src", "pk_tgt")}
    for key in ("src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt"):
        assert np.array_equal(got[key], ref[key]), key
    assert np.array_equal(got["csr_src_tgt"], ref["tgt"][ref["perm_src"]])
    assert np.array_equal(got["csr_src_combo"], ref["combo"][ref["perm_src"]])
    assert np.array_equal(got["csr_tgt_src"], ref["src"][ref["perm_tgt"]])
    assert np.array_equal(got["csr_tgt_combo"], ref["combo"][ref["perm_tgt"]])
    inv = np.empty_like(ref["perm_src"]); inv[ref["perm_src"]] = np.arange(len(inv))
    assert np.array_equal(got["csr_tgt_apos"], inv[ref["perm_tgt"]])
    inv_t = np.empty_like(ref["perm_tgt"]); inv_t[ref["perm_tgt"]] = np.arange(len(inv_t))
    assert np.array_equal(got["csr_src_tpos"], inv_t[ref["perm_src"]])
    n = fx["case"]["n"]  # packed (local endpoint << 16 | combo) used by the shared-memory-tiled kernel
    assert np.array_equal(got["pk_src"], ((ref["tgt"] % n) << 16 | ref["combo"])[ref["perm_src"]])
    assert np.array_equal(got["pk_tgt"], ((ref["src"] % n) << 16 | ref["combo"])[ref["perm_tgt"]])
    assert torch.equal(prep.edge_index_prime().cpu(), fx["edge_index_prime"])
    # degree-sorted schedule of the tiled kernel: a permutation of each graph's nodes, degrees non-increasing
    N = inp["node_type"].numel()
    for name_o, deg in (("order_src", ref["outdeg"]), ("order_tgt", ref["indeg"])):
        order = prep.buf[getattr(prep.layout, name_o):getattr(prep.layout, name_o) + 4 * N].view(torch.int32).cpu().numpy()
        for g in range(N // n):
            o = order[g * n:(g + 1) * n]
            assert sorted(o.tolist()) == list(range(n)), name_o
            dg = np.minimum(deg[g * n + o], 255)
            assert (np.diff(dg) <= 0).all(), name_o


@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_message_passing_matches_reference_golden(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    d = _dev(inp)
    mod = _mp_module(c, fx, sd)
    extra = mod.node_feature_extra(d["node_type"], d["node_score"])
    Hh.assert_close(extra, fx["extra"], "node_feature_extra")
    out, layers = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    for l, ref_l in fx["layers"].items():
        Hh.assert_close(layers[l], ref_l["x"], f"x[{l}]")
    Hh.assert_close(out, fx["out"], "out")


@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_layerwise_api_matches_fused_forward(name):
    """mp_helper-style use (one GATConvE.forward per layer + GELU) equals the fused qagnn_mp_forward."""
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    d = _dev(inp)
    mod = _mp_module(c, fx, sd)
    extra = mod.node_feature_extra(d["node_type"], d["node_score"])
    X = d["H"].view(-1, c["D"]).contiguous()
    nt = d["node_type"].view(-1)
    for l in range(c["k"]):
        X, (ei2, alpha) = mod.gnn_layers[l](X, d["edge_index"], d["edge_type"], nt, extra, return_attention_weights=True)
        X = mod.activation(X)
        if l in fx["layers"]:
            Hh.assert_close(alpha, fx["layers"][l]["alpha"], f"alpha[{l}]")
            Hh.assert_close(X, fx["layers"][l]["x"], f"x[{l}]")
            assert torch.equal(ei2.cpu(), fx["edge_index_prime"])
    _, layers = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    Hh.assert_close(X, layers[-1].cpu(), "layerwise vs fused", atol=2e-5, rtol=2e-5)


@pytest.mark.parametrize("name", Hh.golden_names("layer"))
def test_gatconve_matches_reference_golden(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    x, extra, node_type, ei, et, sd = Hh.regen_layer_inputs(fx)
    D = c["D"]
    enc = torch.nn.Sequential(torch.nn.Linear(fx["n_etype"] + 1 + fx["n_ntype"] * 2, D), torch.nn.BatchNorm1d(D),
                              torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, fx["n_ntype"], fx["n_etype"], enc, head_count=c["H"]).eval()
    layer.load_state_dict({k[len("gnn_layers.0."):]: v for k, v in sd.items() if k.startswith("gnn_layers.0.")}, strict=True)
    layer = layer.to(DEV)
    out, (ei2, alpha) = layer(x.to(DEV), ei.to(DEV), et.to(DEV), node_type.to(DEV), extra.to(DEV),
                              return_attention_weights=True)
    assert torch.equal(ei2.cpu(), fx["edge_index_prime"])
    Hh.assert_close(alpha, fx["alpha"], "alpha")
    Hh.assert_close(out, fx["out"], "out")
    # softmax groups by SOURCE: alpha sums to one over the out-edges of every source node
    sums = torch.zeros(x.size(0), c["H"], device=DEV).index_add_(0, ei2[0].to(DEV), alpha)
    assert torch.allclose(sums, torch.ones_like(sums), atol=1e-5)


@pytest.mark.parametrize("name", Hh.golden_names("decoder"))
def test_decoder_matches_reference_golden(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    dec = qagnn_b200.QAGNN(None, c["k"], fx["n_ntype"], fx["n_etype"], c["sent_dim"], c["n_concept"], c["D"],
                           c["concept_in_dim"], c["n_head"], c["D"], c["n_fc_layer"], 0.2, 0.2, 0.2).eval()
    dec.load_state_dict(fx["state_dict"], strict=True)
    dec = dec.to(DEV)
    d = _dev(inp)
    args = (sent_vecs.to(DEV), concept_ids.to(DEV), d["node_type"], d["node_score"], d["adj_lengths"],
            (d["edge_index"], d["edge_type"]))
    logits, pool_attn = dec(*args)                 # autograd on: plain-PyTorch concept projection
    with torch.no_grad():
        logits_ng, pool_attn_ng = dec(*args)       # inference mode: concept projection on the tensor-core GEMM
    for lg, pa in ((logits, pool_attn), (logits_ng, pool_attn_ng)):
        Hh.assert_close(pa, fx["pool_attn"], "pool_attn")
        Hh.assert_close(lg, fx["logits"], "logits")


def test_out_of_range_indices_raise():
    inp = O.synth_graph_batch(2, 10, 20, 64, 38, 0)
    sd = O.random_state_dict(1, 64)
    mod = qagnn_b200.QAGNN_Message_Passing(None, 1, 4, 38, 64, 64, 64).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = _dev(inp)
    bad = d["edge_index"].clone(); bad[0, 3] = 20  # == N
    with pytest.raises(IndexError):
        mod(d["H"], (bad, d["edge_type"]), d["node_type"], d["node_score"])
    bad_t = d["edge_type"].clone(); bad_t[0] = 38
    with pytest.raises(IndexError):
        mod(d["H"], (d["edge_index"], bad_t), d["node_type"], d["node_score"])


# ---- full-size (BASELINE.json configs[1]) properties -----------------------------------------
@pytest.fixture(scope="module")
def cfg2():
    B, n, e, D, k = 320, 200, 1000, 200, 5
    inp = O.synth_graph_batch(B, n, e, D, 38, seed=0, realistic=True)
    sd = O.random_state_dict(k, D, 4, 38, "peaky", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
    mod.load_state_dict(sd)
    return inp, sd, mod.to(DEV)


def test_cfg2_deterministic_and_oracle_on_a_slice(cfg2):
    inp, sd, mod = cfg2
    d = _dev(inp)
    a = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
    b = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
    assert torch.equal(a, b), "two runs on the same inputs must be bit-identical (no atomics in the data path)"
    # graphs are independent: the first 12 graphs evaluated alone by the CPU oracle
    g, n = 12, 200
    sel = inp["edge_index"][0] < g * n
    ref = O.message_passing_forward(sd, inp["H"][:g], inp["edge_index"][:, sel], inp["edge_type"][sel],
                                    inp["node_type"][:g], inp["node_score"][:g], 5, 4, 38)
    Hh.assert_close(a[:g], ref, "cfg2 slice vs oracle")


def test_cfg2_batch_independence_and_edge_permutation(cfg2):
    inp, sd, mod = cfg2
    d = _dev(inp)
    full = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
    # (1) a sub-batch gives the same rows as the full batch
    g, n = 40, 200
    sel = d["edge_index"][0] < g * n
    sub = mod(d["H"][:g], (d["edge_index"][:, sel], d["edge_type"][sel]), d["node_type"][:g], d["node_score"][:g])
    Hh.assert_close(sub, full[:g].cpu(), "sub-batch vs full batch", atol=1e-6, rtol=1e-6)
    # (2) the order of the edge list is irrelevant up to summation order
    perm = torch.randperm(d["edge_index"].size(1), device=DEV, generator=torch.Generator(DEV).manual_seed(0))
    shuf = mod(d["H"], (d["edge_index"][:, perm], d["edge_type"][perm]), d["node_type"], d["node_score"])
    Hh.assert_close(shuf, full.cpu(), "edge permutation", atol=2e-5, rtol=1e-4)


@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_tiled_and_csr_kernels_agree_and_match_golden(name):
    """The shared-memory-tiled kernel (n_per_graph known) and the general CSR kernels compute the same layer;
    both match the reference's alpha / x of layer 0."""
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    d = _dev(inp)
    mod = _mp_module(c, fx, sd)
    extra = mod.node_feature_extra(d["node_type"], d["node_score"])
    X = d["H"].view(-1, c["D"]).contiguous()
    nt = d["node_type"].view(-1)
    layer = mod.gnn_layers[0]
    prep_t = GraphPrep(d["edge_index"], d["edge_type"], nt, fx["n_ntype"], fx["n_etype"], n_per_graph=c["n"])
    prep_c = GraphPrep(d["edge_index"], d["edge_type"], nt, fx["n_ntype"], fx["n_etype"], n_per_graph=0)
    (out_t, (ei_t, al_t)), ag_t = layer(X, None, None, nt, extra, return_attention_weights=True, prep=prep_t, return_aggr=True)
    (out_c, (ei_c, al_c)), ag_c = layer(X, None, None, nt, extra, return_attention_weights=True, prep=prep_c, return_aggr=True)
    assert torch.equal(ei_t, ei_c)
    Hh.assert_close(al_t, al_c.cpu(), "alpha tiled vs csr", atol=2e-6, rtol=2e-5)
    Hh.assert_close(ag_t, ag_c.cpu(), "aggr tiled vs csr", atol=2e-5, rtol=2e-5)
    Hh.assert_close(al_t, fx["layers"][0]["alpha"], "alpha tiled vs golden")
    Hh.assert_close(mod.activation(out_t), fx["layers"][0]["x"], "x tiled vs golden")


def test_cross_graph_edge_is_rejected_when_n_per_graph_is_given():
    inp = O.synth_graph_batch(2, 10, 20, 64, 38, 0)
    d = _dev(inp)
    bad = d["edge_index"].clone(); bad[0, 0] = 0; bad[1, 0] = 15  # graph 0 -> graph 1
    GraphPrep(bad, d["edge_type"], d["node_type"], 4, 38, n_per_graph=0)  # legal for a general graph
    with pytest.raises(IndexError):
        GraphPrep(bad, d["edge_type"], d["node_type"], 4, 38, n_per_graph=10)


def test_packed_batch_through_the_module_matches_the_unpacked_call_and_rejects_bad_graph_ptr():
    """A qagnn_b200.data.PackedAdj (graph_ptr + max_edges) in place of the (edge_index, edge_type) pair: same output bits; a
    graph_ptr that disagrees with the edges is an IndexError, a cross-graph edge falls back to the general prep."""
    from qagnn_b200.data import PackedAdj
    B, n, D, k = 5, 30, 64, 2
    inp = O.synth_graph_batch(B, n, 70, D, 38, 4, realistic=True)
    sd = O.random_state_dict(k, D, 4, 38, "peaky", 4)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = _dev(inp)
    gp = _graph_ptr(inp["edge_index"], n, B)
    plain = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
    pk = PackedAdj(d["edge_index"], d["edge_type"], gp, n, None, gp.to(DEV), int((gp[1:] - gp[:-1]).max()))
    packed = mod(d["H"], pk, d["node_type"], d["node_score"])
    assert torch.equal(plain, packed)
    assert mod._last_prep.n_per_graph == n
    mod.use_cuda_graph = True  # and through the module's own CUDA-graph cache
    assert torch.equal(mod(d["H"], pk, d["node_type"], d["node_score"]), plain)
    mod.use_cuda_graph = False
    bad_gp = gp.clone(); bad_gp[2] += 3  # sub-graph 1 claims 3 edges of sub-graph 2
    with pytest.raises(IndexError):
        GraphPrep(d["edge_index"], d["edge_type"], d["node_type"].view(-1), 4, 38, n, graph_ptr=bad_gp.to(DEV),
                  max_edges=int((bad_gp[1:] - bad_gp[:-1]).max()))
    short = PackedAdj(d["edge_index"], d["edge_type"], gp, n, None, gp.to(DEV), 3)  # max_edges too small: refused, not overrun
    with pytest.raises(IndexError):
        mod(d["H"], short, d["node_type"], d["node_score"])


def test_cross_graph_edges_fall_back_to_the_general_kernels_in_the_module_api():
    """n_per_graph is a layout hint: QAGNN_Message_Passing.forward accepts any batched edge_index like the reference
    (ADVICE r1): an edge that crosses a sub-graph boundary routes the batch to the general CSR kernels."""
    B, n, D, k = 3, 20, 64, 2
    inp = O.synth_graph_batch(B, n, 50, D, 38, 9)
    sd = O.random_state_dict(k, D, 4, 38, "peaky", 9)
    ei = inp["edge_index"].clone()
    ei[0, 0], ei[1, 0] = 1, n + 3            # graph 0 -> graph 1
    ei[0, 1], ei[1, 1] = 2 * n + 5, 7        # graph 2 -> graph 0
    ref = O.message_passing_forward(sd, inp["H"], ei, inp["edge_type"], inp["node_type"], inp["node_score"], k, 4, 38)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = _dev(inp)
    out = mod(d["H"], (ei.to(DEV), d["edge_type"]), d["node_type"], d["node_score"])
    assert mod._last_prep.n_per_graph == 0
    Hh.assert_close(out, ref, "cross-graph batch vs oracle")


# ---- the exact workload bench.py times (uniform synthetic batch, production-init weights, seed 100 + rank) ----------
def test_bench_workload_matches_oracle_on_first_middle_and_last_graphs():
    import bench
    B, n, e, D, k = (bench.CFG[x] for x in ("graphs", "n", "e", "D", "k"))
    inp = O.synth_graph_batch(B, n, e, D, bench.CFG["R"], seed=100)
    sd = O.random_state_dict(k, D, bench.CFG["T"], bench.CFG["R"], "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, bench.CFG["T"], bench.CFG["R"], D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = _dev(inp)
    out = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"]).cpu()
    # 36 graphs: the first 12, 12 from the middle, and the last 12 (the tail of the persistent kernel's last slot)
    for g0 in (0, B // 2 - 6, B - 12):
        ref = bench.oracle_slice(inp, sd, g0, 12)
        Hh.assert_close(out[g0:g0 + 12], ref, f"bench workload graphs {g0}..{g0 + 11} vs oracle")
    # the CUDA-graph replay bench.py times gives the same bits
    mod.use_cuda_graph = True
    rep = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"]).cpu()
    assert torch.equal(rep, out)


# ---- every launch-time switch the shipped library keeps (read at each call) has GPU coverage ------------------------
@pytest.mark.parametrize("env", [{"QAGNN_MP_PATH": "csr"}, {"QAGNN_MP_PATH": "basic"}, {"QAGNN_TC_2CTA": "0"}, {"QAGNN_GEMM": "ffma"},
                                 {"QAGNN_MP_WARPS": "24"}, {"QAGNN_MP_WARPS": "31"}, {"QAGNN_MP_WARPS": "7"},
                                 {"QAGNN_MP_FASTPROJ": "0"}])
@pytest.mark.parametrize("name", ["cfg2small_peaky", "cfg2small_realistic", "tiny_realistic_d100", "no_edges", "cfg1_peaky_k2"])
def test_goldens_under_every_kept_switch(name, env, monkeypatch):
    for k_, v in env.items():
        monkeypatch.setenv(k_, v)
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    d = _dev(inp)
    mod = _mp_module(c, fx, sd)
    out, layers = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    for l, ref_l in fx["layers"].items():
        Hh.assert_close(layers[l], ref_l["x"], f"x[{l}] under {env}")
    Hh.assert_close(out, fx["out"], f"out under {env}")


def test_large_graph_general_path_matches_oracle():
    """Stress-shaped input (BASELINE.json configs[4] scaled down): one big graph per batch entry, H=8 — too large for
    the shared-memory tiles, so this exercises the general CSR kernels + tensor-core GEMMs end to end."""
    n, e, D, Hh_, k = 600, 6000, 256, 8, 2
    inp = O.synth_graph_batch(2, n, e, D, 38, seed=21)
    sd = O.random_state_dict(1, D, 4, 38, "peaky", seed=21)
    x = inp["H"].view(-1, D).contiguous()
    extra = torch.randn(x.shape, generator=torch.Generator().manual_seed(5)) * 0.5
    nt = inp["node_type"].view(-1)
    ref_out, ei2, ref_alpha, _ = O.gatconve_forward(sd, "gnn_layers.0", x, inp["edge_index"], inp["edge_type"], nt, extra,
                                                    4, 38, head_count=Hh_)
    enc = torch.nn.Sequential(torch.nn.Linear(38 + 1 + 8, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, 4, 38, enc, head_count=Hh_).eval()
    layer.load_state_dict({k_[len("gnn_layers.0."):]: v for k_, v in sd.items() if k_.startswith("gnn_layers.0.")})
    layer = layer.to(DEV)
    out, (ei_g, alpha) = layer(x.to(DEV), inp["edge_index"].to(DEV), inp["edge_type"].to(DEV), nt.to(DEV), extra.to(DEV),
                               return_attention_weights=True)
    assert torch.equal(ei_g.cpu(), ei2)
    Hh.assert_close(alpha, ref_alpha, "alpha")
    Hh.assert_close(out, ref_out, "out")


@pytest.mark.parametrize("path", ["auto", "basic"])
def test_stress_shape_full_size_graph_matches_oracle(path, monkeypatch):
    """BASELINE.json configs[4] at FULL per-graph size (2000 nodes / 20000 edges, hidden 1024, 8 heads): one GATConvE layer on
    one such graph against the CPU oracle, through the column-sliced kernels (auto) and the basic CSR kernels."""
    if path == "basic":
        monkeypatch.setenv("QAGNN_MP_PATH", "basic")
    n, e, D, Hh_ = 2000, 20000, 1024, 8
    inp = O.synth_graph_batch(1, n, e, D, 38, seed=55)
    sd = O.random_state_dict(1, D, 4, 38, "peaky", seed=55)
    x = inp["H"].view(-1, D).contiguous()
    extra = torch.randn(x.shape, generator=torch.Generator().manual_seed(6)) * 0.5
    nt = inp["node_type"].view(-1)
    torch.set_num_threads(min(32, torch.get_num_threads() if torch.get_num_threads() > 0 else 8))
    ref_out, ei2, ref_alpha, ref_aggr = O.gatconve_forward(sd, "gnn_layers.0", x, inp["edge_index"], inp["edge_type"], nt, extra,
                                                           4, 38, head_count=Hh_)
    enc = torch.nn.Sequential(torch.nn.Linear(38 + 1 + 8, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, 4, 38, enc, head_count=Hh_).eval()
    layer.load_state_dict({k_[len("gnn_layers.0."):]: v for k_, v in sd.items() if k_.startswith("gnn_layers.0.")})
    layer = layer.to(DEV)
    (out, (ei_g, alpha)), aggr = layer(x.to(DEV), inp["edge_index"].to(DEV), inp["edge_type"].to(DEV), nt.to(DEV), extra.to(DEV),
                                       return_attention_weights=True, return_aggr=True)
    assert torch.equal(ei_g.cpu(), ei2)
    Hh.assert_close(alpha, ref_alpha, f"alpha ({path})")
    Hh.assert_close(aggr, ref_aggr, f"aggr ({path})")
    Hh.assert_close(out, ref_out, f"out ({path})")
    again = layer(x.to(DEV), inp["edge_index"].to(DEV), inp["edge_type"].to(DEV), nt.to(DEV), extra.to(DEV))
    assert torch.equal(again, out), "the large-graph path must be run-to-run bit-identical"


def test_lm_qagnn_forward_api_with_packed_and_nested_adjacency():
    """LM_QAGNN.forward keeps the reference's positional-input API (modeling_qagnn.py:207-251): nested
    [batch][choice] adjacency lists and the packed form give identical logits; the decoder part matches the oracle."""
    from transformers import RobertaConfig
    from qagnn_b200.data import pack_adj
    torch.manual_seed(0)
    cfg = RobertaConfig(vocab_size=100, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128,
                        max_position_embeddings=40)
    bs, nc, n, D, k = 3, 5, 20, 64, 2
    model = qagnn_b200.LM_QAGNN(None, "roberta-tiny", k, 4, 38, n_concept=200, concept_dim=D, concept_in_dim=D,
                                n_attention_head=2, fc_dim=D, n_fc_layer=0, p_emb=0.2, p_gnn=0.2, p_fc=0.2,
                                init_range=0.02, encoder_config={"config": cfg}).eval().to(DEV)
    g = torch.Generator().manual_seed(1)
    input_ids = torch.randint(3, 100, (bs, nc, 16), generator=g)
    attn = torch.ones(bs, nc, 16, dtype=torch.long)
    ttype = torch.zeros(bs, nc, 16, dtype=torch.long)
    omask = torch.zeros(bs, nc, 16, dtype=torch.long)
    inp = O.synth_graph_batch(bs * nc, n, 50, D, 38, seed=3, realistic=True)
    concept_ids = torch.randint(1, 201, (bs, nc, n), generator=g); concept_ids[:, :, 0] = 0
    ei_nested, et_nested = [], []
    for b in range(bs):
        ei_row, et_row = [], []
        for c in range(nc):
            gi = b * nc + c
            sel = (inp["edge_index"][0] >= gi * n) & (inp["edge_index"][0] < (gi + 1) * n)
            ei_row.append((inp["edge_index"][:, sel] - gi * n).to(DEV)); et_row.append(inp["edge_type"][sel].to(DEV))
        ei_nested.append(ei_row); et_nested.append(et_row)
    dec_in = (concept_ids.to(DEV), inp["node_type"].view(bs, nc, n).to(DEV), inp["node_score"].view(bs, nc, n, 1).to(DEV),
              inp["adj_lengths"].view(bs, nc).to(DEV))
    lm_in = (input_ids.to(DEV), attn.to(DEV), ttype.to(DEV), omask.to(DEV))
    with torch.no_grad():
        logits, pool_attn = model(*lm_in, *dec_in, ei_nested, et_nested)
        packed = pack_adj([[e.cpu() for e in r] for r in ei_nested], [[e.cpu() for e in r] for r in et_nested], n)
        logits_p, _ = model(*lm_in, *dec_in, packed.to(DEV), None)
        sent_vecs, _ = model.encoder(*[x.view(bs * nc, -1) for x in lm_in])
    assert logits.shape == (bs, nc) and pool_attn.shape == (2 * bs * nc, n)
    assert torch.equal(logits, logits_p)
    sd = {k_: v.cpu() for k_, v in model.decoder.state_dict().items()}
    ref_logits, _, _ = O.qagnn_decoder_forward(sd, sent_vecs.cpu(), concept_ids.view(bs * nc, n), inp["node_type"],
                                               inp["node_score"], inp["adj_lengths"], inp["edge_index"], inp["edge_type"],
                                               k, 4, 38, 2, 0)
    Hh.assert_close(logits.view(-1, 1), ref_logits, "LM_QAGNN logits vs oracle decoder")


def test_tiled_kernel_hub_nodes_and_unstaged_graphs():
    """Tiled-path corner cases against the oracle and the CSR kernels: a degree-199 hub (logits beyond the 8th edge go
    through the L2 scratch), a graph with more edges than the shared-memory CSR staging holds (global fallback inside
    the kernel), a graph with no edges at all, in one batch."""
    n, D, k = 200, 200, 1
    g = torch.Generator().manual_seed(11)
    def rnd(e, lo=0):
        return torch.randint(lo, n, (2, e), generator=g)
    hub = torch.cat([torch.stack([torch.zeros(n - 1, dtype=torch.long), torch.arange(1, n)]),
                     torch.stack([torch.arange(1, n), torch.zeros(n - 1, dtype=torch.long)])], dim=1)
    graphs = [rnd(1000), rnd(3600), hub, torch.zeros(2, 0, dtype=torch.long), rnd(900)]
    ei = torch.cat([e + i * n for i, e in enumerate(graphs)], dim=1)
    et = torch.randint(0, 38, (ei.size(1),), generator=g)
    B = len(graphs)
    nt = torch.randint(0, 3, (B, n), generator=g); nt[:, 0] = 3
    x = torch.randn(B * n, D, generator=g) * 0.5
    extra = torch.randn(B * n, D, generator=g) * 0.5
    sd = O.random_state_dict(k, D, 4, 38, "peaky", seed=11)
    ref_out, ei2, ref_alpha, ref_aggr = O.gatconve_forward(sd, "gnn_layers.0", x, ei, et, nt.view(-1), extra, 4, 38)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    layer = mod.gnn_layers[0]
    xd, ed, ntd = x.to(DEV), extra.to(DEV), nt.view(-1).to(DEV)
    prep_t = GraphPrep(ei.to(DEV), et.to(DEV), ntd, 4, 38, n_per_graph=n)
    prep_c = GraphPrep(ei.to(DEV), et.to(DEV), ntd, 4, 38, n_per_graph=0)
    (out_t, (_, al_t)), ag_t = layer(xd, None, None, ntd, ed, return_attention_weights=True, prep=prep_t, return_aggr=True)
    (out_c, (_, al_c)), ag_c = layer(xd, None, None, ntd, ed, return_attention_weights=True, prep=prep_c, return_aggr=True)
    Hh.assert_close(al_t, ref_alpha, "alpha tiled vs oracle")
    Hh.assert_close(al_c, ref_alpha, "alpha csr vs oracle")
    Hh.assert_close(ag_t, ref_aggr, "aggr tiled vs oracle", atol=1e-4, rtol=2e-4)
    Hh.assert_close(ag_c, ref_aggr, "aggr csr vs oracle", atol=1e-4, rtol=2e-4)
    Hh.assert_close(out_t, ref_out, "out tiled vs oracle")
    Hh.assert_close(out_c, ref_out, "out csr vs oracle")


def test_fused_attention_pool_matches_oracle():
    """qagnn_attention_pool (keys/values folded into the query / out of the sum, one pass over the node tile) against
    the oracle's restatement of MultiheadAttPoolLayer (utils/layers.py:324-371)."""
    from qagnn_b200.layers import MultiheadAttPoolLayer
    torch.manual_seed(3)
    for (b, n, D, S, nh) in [(7, 200, 200, 1024, 2), (3, 33, 64, 48, 4)]:
        pool = MultiheadAttPoolLayer(nh, S, D).eval()
        q, k = torch.randn(b, S), torch.randn(b, n, D) * 0.7
        mask = torch.rand(b, n) < 0.4
        mask[:, 0] = False
        sd = {"pooler." + k_: v for k_, v in pool.state_dict().items()}
        ref_out, ref_attn = O.multihead_att_pool(sd, "pooler", q, k, mask, nh)
        with torch.no_grad():
            got_out, got_attn = pool.to(DEV)(q.to(DEV), k.to(DEV), mask.to(DEV))  # CUDA: fused kernel
        Hh.assert_close(got_attn, ref_attn, "pool attn", atol=2e-6, rtol=1e-4)
        Hh.assert_close(got_out, ref_out, "pooled", atol=2e-5, rtol=1e-4)


def test_cuda_graph_replay_and_streamed_runner_match_plain_forward():
    """use_cuda_graph replays and the double-buffered StreamedRunner (copies on their own streams) give bit-identical
    results to the plain forward, batch after batch."""
    from qagnn_b200.pipeline import StreamedRunner
    B, n, e, D, k = 6, 50, 200, 64, 2
    sd = O.random_state_dict(k, D, 4, 38, "peaky", seed=4)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    batches = [O.synth_graph_batch(B, n, e, D, 38, seed=40 + i) for i in range(5)]
    plain = []
    for bt in batches:
        d = _dev(bt)
        plain.append(mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"]).cpu())
    mod.use_cuda_graph = True
    host = [{k_: v.pin_memory() for k_, v in bt.items() if k_ != "adj_lengths"} for bt in batches]
    runner = StreamedRunner(mod, host[0], torch.device(DEV), depth=2)
    got = []
    for i, hb in enumerate(host):
        slot = runner.submit(hb)
        if i >= 1:  # consume the previous result while this batch is in flight
            prev = (i - 1) % 2
            runner.ev_down[prev].synchronize()
            got.append(runner.host_out[prev][0].clone())
    runner.drain()
    torch.cuda.synchronize()
    got.append(runner.host_out[(len(host) - 1) % 2][0].clone())
    for a, b in zip(got, plain):
        assert torch.equal(a, b)
    assert len(mod._graphs) == 2  # one captured graph per buffer set


def test_decoder_step_graph_matches_module_composition():
    """qagnn_b200.pipeline.DecoderStep (MP forward + pool mask + fused pooling + answer MLP as ONE CUDA graph) gives the
    same logits / attention as calling the decoder's modules one by one, and replays follow new contents of its buffers."""
    from qagnn_b200.layers import MLP, MultiheadAttPoolLayer
    from qagnn_b200.pipeline import DecoderStep
    B, n, e, D, k, S = 10, 40, 120, 64, 2, 96
    sd = O.random_state_dict(k, D, 4, 38, "peaky", 3)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, 4, 38, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    torch.manual_seed(4)
    pooler = MultiheadAttPoolLayer(2, S, D).eval().to(DEV)
    fc = MLP(D + S + D, D, 1, 0, 0.2, layer_norm=True).eval().to(DEV)
    # the reference's answer MLP is a CPU copy: moving `fc` itself would free the weights the captured graph reads
    fc_ref = copy.deepcopy(fc).cpu()

    def batch(seed):
        inp = O.synth_graph_batch(B, n, e, D, 38, seed, realistic=True)
        inp["sent_vecs"] = torch.randn(B, S, generator=torch.Generator().manual_seed(seed)) * 0.5
        return {k_: inp[k_].to(DEV) for k_ in DecoderStep.FIELDS}, inp

    d, inp = batch(11)
    step = DecoderStep(mod, pooler, fc, d, 1, None, use_cuda_graph=True)
    assert step.graph is not None
    for seed in (11, 12):
        nd, ninp = batch(seed)
        if seed != 11:  # same adjacency buffers (their length is part of the captured graph), new features / scores / sentences
            for k_ in ("edge_index", "edge_type", "node_type", "adj_lengths"):
                nd[k_], ninp[k_] = d[k_].clone(), inp[k_]
        for k_ in DecoderStep.FIELDS:
            d[k_].copy_(nd[k_])
        logits, attn, gout = (t.clone() for t in step.run())
        with torch.no_grad():
            ref_out = O.message_passing_forward(sd, ninp["H"], ninp["edge_index"], ninp["edge_type"], ninp["node_type"],
                                                ninp["node_score"], k, 4, 38)
            mask = (torch.arange(n) >= ninp["adj_lengths"].unsqueeze(1)) | (ninp["node_type"] == 3)
            mask[mask.all(1), 0] = 0
            psd = {"pooler." + k_: v.cpu() for k_, v in pooler.state_dict().items()}
            gv, ref_attn = O.multihead_att_pool(psd, "pooler", ninp["sent_vecs"], ref_out, mask, 2)
            ref_logits = fc_ref(torch.cat((gv, ninp["sent_vecs"], ref_out[:, 0]), 1))
        Hh.assert_close(gout, ref_out, f"gnn_out seed {seed}")
        Hh.assert_close(attn, ref_attn, f"pool_attn seed {seed}", atol=2e-5)
        Hh.assert_close(logits, ref_logits, f"logits seed {seed}")


@pytest.mark.parametrize("hub_deg", [33, 300, 5000, 9000])
def test_graph_prep_hub_segments_are_sorted_by_edge_id(hub_deg):
    """Segments longer than 32 edges go through the per-CTA sort of graph prep (bitonic in shared memory up to 8192 ids,
    rank counting beyond): perm arrays must still equal the stable sort of the oracle."""
    N, T, R = 64, 4, 38
    g = torch.Generator().manual_seed(hub_deg)
    E = hub_deg * 2 + 200
    src = torch.randint(0, N, (E,), generator=g)
    tgt = torch.randint(0, N, (E,), generator=g)
    idx = torch.randperm(E, generator=g)
    src[idx[:hub_deg]] = 5            # node 5: a source hub
    tgt[idx[hub_deg:2 * hub_deg]] = 9  # node 9: a target hub
    ei = torch.stack([src, tgt])
    et = torch.randint(0, R, (E,), generator=g)
    nt = torch.randint(0, T, (N,), generator=g)
    prep = GraphPrep(ei.to(DEV), et.to(DEV), nt.to(DEV), T, R, 0)
    ref = O.graph_prep_oracle(ei, et, nt, T, R)
    for key in ("rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt"):
        assert np.array_equal(prep.array(key).cpu().numpy().astype(np.int64), ref[key]), key
