"""Ragged eval batches on the GPU: every sub-graph keeps only its adj_lengths rows, graph g's from node_ptr[g] on.  Whatever
the decoder returns for a ragged batch is checked against the padded layout's valid rows and the committed goldens.  Needs a
GPU: run with -m gpu."""
import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200.modeling_qagnn import GraphPrep
from qagnn_b200.pipeline import DecoderStep
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R = 4, 38


def ragged_inputs(H, edge_index, edge_type, node_type, node_score, adj_lengths, n, node_capacity=None, edge_capacity=None):
    """(host ragged PackedAdj, packed H [N_cap, D], node_type [N_cap], node_score [N_cap, 1], row index of every packed row in
    the padded [B*n] layout) of a padded batch whose edges stay inside each graph's first adj_lengths nodes."""
    B = adj_lengths.numel()
    g = edge_index[0] // n
    order = torch.argsort(g, stable=True)
    ei, et, g = edge_index[:, order], edge_type[order], g[order]
    counts = torch.bincount(g, minlength=B).tolist()
    eis = list(torch.split(ei - g * n, counts, dim=1))
    ets = list(torch.split(et, counts))
    adj = Dt.pack_adj(eis, ets, n, pin=False, edge_capacity=edge_capacity, adj_lengths=adj_lengths,
                      node_capacity=node_capacity)
    rows = torch.cat([b * n + torch.arange(int(adj_lengths[b])) for b in range(B)])
    N_cap = adj.node_capacity
    Hp = torch.zeros(N_cap, H.size(-1), dtype=H.dtype)
    Hp[:rows.numel()] = H.reshape(-1, H.size(-1))[rows]
    ntp = torch.full((N_cap,), 2, dtype=torch.long)
    ntp[:rows.numel()] = node_type.reshape(-1)[rows]
    nsp = torch.zeros(N_cap, 1)
    nsp[:rows.numel()] = node_score.reshape(-1, 1)[rows]
    return adj, Hp, ntp, nsp, rows


def _dev_adj(adj):
    return adj.to(DEV)


def _module(k, D, seed=5, regime="prod", heads=None):
    sd = O.random_state_dict(k, D, T, R, regime, seed=seed)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, T, R, D, D, D).eval()
    mod.load_state_dict(sd)
    return mod.to(DEV)


def _loader_batch(n_questions=6, nc=5, n=200, D=200, seed=3):
    import os
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_questions * nc, seed=seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, n, nc)
    qs = np.arange(n_questions)
    pad = flat.pack(qs, pin=False)
    B = n_questions * nc
    gen = torch.Generator().manual_seed(seed)
    return {"H": torch.randn(B, n, D, generator=gen) * 0.5, "edge_index": pad.edge_index.clone(), "edge_type": pad.edge_type.clone(),
            "node_type": ntypes.reshape(B, n), "node_score": scores.reshape(B, n, 1), "adj_lengths": lens.reshape(-1)}, n


def _mp_cases():
    out = []
    for name in ("cfg2small_realistic", "tiny_realistic_d100"):
        fx = Hh.load_golden(name)
        inp, _ = Hh.regen_mp_inputs(fx)
        c = fx["case"]
        # the golden graphs use all n nodes: a ragged batch of full-length graphs
        inp["adj_lengths"] = torch.full((c["B"],), c["n"], dtype=torch.long)
        out.append((name, inp, c["n"], c["k"], c["D"]))
    inp, n = _loader_batch()
    out.append(("loader_shaped", inp, n, 3, 200))
    return out


@pytest.fixture(scope="module")
def mp_cases():
    return _mp_cases()


def test_ragged_prep_equals_the_general_prep(mp_cases):
    name, inp, n, k, D = mp_cases[2]
    adj, Hp, ntp, nsp, _ = ragged_inputs(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                                         inp["adj_lengths"], n, node_capacity=int(inp["adj_lengths"].sum()) + 437)
    a = _dev_adj(adj)
    nt = ntp.to(DEV)
    pr = GraphPrep(a.edge_index, a.edge_type, nt, T, R, n, graph_ptr=a.graph_ptr_dev, max_edges=a.max_edges, node_ptr=a.node_ptr_dev)
    pg = GraphPrep(a.edge_index, a.edge_type, nt, T, R, 0)
    assert pr.packed and pr.node_ptr is not None and int(pr.status_word().item()) == 0
    for key in ("src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src", "perm_tgt", "csr_src_tgt", "csr_src_combo",
                "csr_tgt_src", "csr_tgt_combo", "csr_tgt_apos", "csr_src_tpos"):
        assert torch.equal(pr.array(key), pg.array(key)), key


def _mp_both(mod, inp, n):
    """(padded output rows of the valid nodes, ragged output rows) of QAGNN_Message_Passing."""
    adj, Hp, ntp, nsp, rows = ragged_inputs(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                                            inp["adj_lengths"], n, node_capacity=int(inp["adj_lengths"].sum()) + 61)
    with torch.no_grad():
        pad = mod(inp["H"].to(DEV), (inp["edge_index"].to(DEV), inp["edge_type"].to(DEV)), inp["node_type"].to(DEV),
                  inp["node_score"].to(DEV))
        rag = mod(Hp.to(DEV), _dev_adj(adj), ntp.to(DEV), nsp.to(DEV))
    return pad.reshape(-1, pad.size(-1))[rows.to(DEV)], rag, rows.numel()


@pytest.mark.parametrize("case", [0, 1, 2])
def test_module_ragged_rows_equal_the_padded_valid_rows(mp_cases, case):
    name, inp, n, k, D = mp_cases[case]
    mod = _module(k, D)
    pad, rag, nv = _mp_both(mod, inp, n)
    assert rag.shape[0] == nv + 61 and bool(torch.isfinite(rag).all())
    Hh.assert_close(rag[:nv], pad, f"{name}: ragged rows", atol=2e-5, rtol=1e-4)


@pytest.mark.parametrize("path", ["csr", "basic"])
def test_ragged_tiled_kernel_matches_the_csr_kernels(mp_cases, monkeypatch, path):
    name, inp, n, k, D = mp_cases[2]
    mod = _module(k, D)
    layer = mod.gnn_layers[0]
    adj, Hp, ntp, nsp, _ = ragged_inputs(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                                         inp["adj_lengths"], n, node_capacity=int(inp["adj_lengths"].sum()) + 300)
    a = _dev_adj(adj)
    x, nt = Hp.to(DEV), ntp.to(DEV)
    with torch.no_grad():
        extra = mod.node_feature_extra(nt, nsp.to(DEV))
        (o1, (ei1, al1)), ag1 = layer(x, a, None, nt, extra, return_attention_weights=True, return_aggr=True)
        monkeypatch.setenv("QAGNN_MP_PATH", path)
        layer._prep_cache = (None, None)
        (o2, (ei2, al2)), ag2 = layer(x, a, None, nt, extra, return_attention_weights=True, return_aggr=True)
    assert torch.equal(ei1, ei2)
    Hh.assert_close(al1, al2, "alpha", atol=2e-6, rtol=2e-5)
    Hh.assert_close(ag1, ag2, "aggr", atol=2e-5, rtol=2e-5)


def _decoder(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    dec = qagnn_b200.QAGNN(None, c["k"], fx["n_ntype"], fx["n_etype"], c["sent_dim"], c["n_concept"], c["D"], c["concept_in_dim"],
                           c["n_head"], c["D"], c["n_fc_layer"], 0.0, 0.0, 0.0)
    dec.load_state_dict(fx["state_dict"], strict=True)
    return fx, c, inp, sent_vecs, concept_ids, dec.to(DEV).eval()


def _decoder_both(dec, c, inp, sent_vecs, concept_ids, node_capacity_extra=29):
    adj, *_ = ragged_inputs(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                            inp["adj_lengths"], c["n"], node_capacity=int(inp["adj_lengths"].sum()) + node_capacity_extra)
    args = (sent_vecs.to(DEV), concept_ids.to(DEV), inp["node_type"].to(DEV), inp["node_score"].to(DEV), inp["adj_lengths"].to(DEV))
    with torch.no_grad():
        pad = dec(*args, (inp["edge_index"].to(DEV), inp["edge_type"].to(DEV)))
        rag = dec(*args, _dev_adj(adj))
    return pad, rag


@pytest.mark.parametrize("name", ["decoder_small", "decoder_fc1"])
def test_decoder_ragged_matches_goldens_and_padded(name):
    fx, c, inp, sent_vecs, concept_ids, dec = _decoder(name)
    (lp, ap), (lr, ar) = _decoder_both(dec, c, inp, sent_vecs, concept_ids)
    Hh.assert_close(lr, fx["logits"], "logits vs golden", atol=5e-5, rtol=1e-4)
    Hh.assert_close(lr, lp, "logits vs padded", atol=5e-5, rtol=1e-4)
    Hh.assert_close(ar, ap, "pool_attn vs padded", atol=2e-5, rtol=1e-4)
    Hh.assert_close(ar, fx["pool_attn"], "pool_attn vs golden", atol=2e-5, rtol=1e-4)
    pos = torch.arange(c["n"], device=DEV)
    masked = (pos >= inp["adj_lengths"].to(DEV).unsqueeze(1)).repeat(c["n_head"], 1)
    assert bool((ar[masked] == 0).all())


def test_decoder_ragged_under_bf16_autocast_matches_padded():
    fx, c, inp, sent_vecs, concept_ids, dec = _decoder("decoder_small")
    with torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):
        (lp, ap), (lr, ar) = _decoder_both(dec, c, inp, sent_vecs, concept_ids)
    Hh.assert_close(lr.float(), lp.float(), "bf16 logits vs padded", atol=5e-5, rtol=1e-4)
    Hh.assert_close(ar, ap, "bf16 pool_attn vs padded", atol=2e-5, rtol=1e-4)


def _edge_case_batch(n=40, D=64, seed=11):
    """Graphs with adj_lengths 1, a graph with nodes and no edges, a graph with exactly n nodes, and ordinary ones."""
    gen = torch.Generator().manual_seed(seed)
    lens = torch.tensor([1, 7, n, 13, 1, 25])
    B = lens.numel()
    eis, ets = [], []
    for b in range(B):
        L = int(lens[b])
        m = 0 if b == 1 or L == 1 else 3 * L
        s, t = torch.randint(0, L, (m,), generator=gen), torch.randint(0, L, (m,), generator=gen)
        eis.append(torch.stack([s, t]) + b * n)
        ets.append(torch.randint(0, R, (m,), generator=gen))
    nt = torch.full((B, n), 2, dtype=torch.long)
    nt[:, 0] = 3
    nt[:, 1:4] = torch.randint(0, 2, (B, 3), generator=gen)
    return {"H": torch.randn(B, n, D, generator=gen), "edge_index": torch.cat(eis, 1), "edge_type": torch.cat(ets),
            "node_type": nt, "node_score": torch.randn(B, n, 1, generator=gen), "adj_lengths": lens}, n


@pytest.mark.parametrize("heads", [1, 2, 4, 8, 16])
def test_gatconve_ragged_edge_cases_every_head_count(heads):
    inp, n = _edge_case_batch()
    D = 64
    enc = torch.nn.Sequential(torch.nn.Linear(R + 1 + 2 * T, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))
    torch.manual_seed(heads)
    layer = qagnn_b200.GATConvE(None, D, T, R, enc, head_count=heads).to(DEV).eval()
    adj, Hp, ntp, nsp, rows = ragged_inputs(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                                            inp["adj_lengths"], n, node_capacity=int(inp["adj_lengths"].sum()) + 5)
    extra = torch.randn(inp["H"].shape, generator=torch.Generator().manual_seed(2))
    extra_p = torch.zeros_like(Hp)
    extra_p[:rows.numel()] = extra.reshape(-1, D)[rows]
    with torch.no_grad():
        pad = layer(inp["H"].reshape(-1, D).to(DEV), inp["edge_index"].to(DEV), inp["edge_type"].to(DEV),
                    inp["node_type"].reshape(-1).to(DEV), extra.reshape(-1, D).to(DEV))
        rag = layer(Hp.to(DEV), _dev_adj(adj), None, ntp.to(DEV), extra_p.to(DEV))
    Hh.assert_close(rag[:rows.numel()], pad[rows.to(DEV)], f"heads={heads}", atol=2e-5, rtol=1e-4)
    assert bool(torch.isfinite(rag).all())


def test_single_graph_batch():
    inp, n = _edge_case_batch()
    one = {k: v[2:3] for k, v in inp.items() if k not in ("edge_index", "edge_type")}
    sel = (inp["edge_index"][0] // n) == 2
    one["edge_index"] = inp["edge_index"][:, sel] - 2 * n
    one["edge_type"] = inp["edge_type"][sel]
    mod = _module(2, 64)
    pad, rag, nv = _mp_both(mod, one, n)
    Hh.assert_close(rag[:nv], pad, "B = 1", atol=2e-5, rtol=1e-4)


# ---- captured DecoderStep -----------------------------------------------------------------------------------------------
NQ, NC, S = 3, 5, 48


def _step_parts(D=200, k=3):
    from qagnn_b200.layers import MLP, MultiheadAttPoolLayer
    mod = _module(k, D)
    torch.manual_seed(4)
    return mod, MultiheadAttPoolLayer(2, S, D).eval().to(DEV), MLP(D + S + D, D, 1, 0, 0.2, layer_norm=True).eval().to(DEV)


def _ragged_host_batches(n_batches, seed=0, N_cap=None, K=None):
    import os
    import tempfile
    n, D = 200, 200
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_batches * NQ * NC, seed=seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, n, NC)
    N_cap = N_cap or Dt.split_node_capacity(lens, NQ)
    K = K or flat.max_batch_edges(NQ)
    gen = torch.Generator().manual_seed(seed)
    out = []
    for b in range(n_batches):
        qs = np.arange(b * NQ, (b + 1) * NQ)
        adj = flat.pack(qs, pin=False, edge_capacity=K, adj_lengths=lens[qs], node_capacity=N_cap)
        B = NQ * NC
        H = torch.randn(B, n, D, generator=gen) * 0.5
        rows = torch.cat([g * n + torch.arange(int(l)) for g, l in enumerate(lens[qs].reshape(-1))])
        Hp = torch.zeros(N_cap, D)
        Hp[:rows.numel()] = H.reshape(-1, D)[rows]
        ntp = torch.full((N_cap,), 2, dtype=torch.long)
        ntp[:rows.numel()] = ntypes[qs].reshape(-1)[rows]
        nsp = torch.zeros(N_cap, 1)
        nsp[:rows.numel()] = scores[qs].reshape(-1, 1)[rows]
        out.append({"H": Hp, "edge_index": adj.edge_index.clone(), "edge_type": adj.edge_type.clone(), "node_type": ntp,
                    "node_score": nsp, "sent_vecs": torch.randn(B, S, generator=gen) * 0.5,
                    "adj_lengths": lens[qs].reshape(-1).clone(), "graph_ptr": adj.graph_ptr.clone()})
    return out, flat.max_graph_edges(), N_cap


def _eager_step(parts, host, M):
    d = {k: v.to(DEV) for k, v in host.items()}
    return [t.clone() for t in DecoderStep(*parts, d, use_cuda_graph=False, max_edges=M, max_nodes=200).run()]


def test_one_captured_ragged_step_replays_every_batch_bit_for_bit():
    parts = _step_parts()
    hosts, M, N_cap = _ragged_host_batches(4)
    assert len({int(h["adj_lengths"].sum()) for h in hosts}) >= 3 and len({int(h["graph_ptr"][-1]) for h in hosts}) >= 3
    d = {k: v.to(DEV) for k, v in hosts[0].items()}
    step = DecoderStep(*parts, d, use_cuda_graph=True, max_edges=M, max_nodes=200)
    assert step.graph is not None and step.ragged
    for i, h in enumerate(hosts):
        for key in DecoderStep.RAGGED_FIELDS:
            d[key].copy_(h[key])
        got = [t.clone() for t in step.run()]
        again = [t.clone() for t in step.run()]
        ref = _eager_step(parts, h, M)
        for name, a, b, c in zip(("logits", "pool_attn", "gnn_out"), got, again, ref):
            assert torch.equal(a, b), f"batch {i}: {name} differs between two replays"
            assert torch.equal(a, c), f"batch {i}: {name} differs from the eager ragged call"


def test_ragged_refusals():
    parts = _step_parts()
    hosts, M, N_cap = _ragged_host_batches(2, seed=5)
    d = {k: v.to(DEV) for k, v in hosts[0].items()}
    step = DecoderStep(*parts, d, use_cuda_graph=True, max_edges=M, max_nodes=200)
    # an edge whose target lies in the next graph's rows: IndexError at the next run
    bad = {k: v.clone() for k, v in hosts[1].items()}
    e = int(bad["graph_ptr"][1]) - 1  # last edge of graph 0
    bad["edge_index"][1, e] = int(bad["adj_lengths"][0]) + 1
    for key in DecoderStep.RAGGED_FIELDS:
        d[key].copy_(bad[key])
    step.run()
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        step.run()
    # a batch over the node capacity is refused while packing
    with pytest.raises(ValueError, match="node capacity"):
        Dt.pack_adj([torch.zeros(2, 0, dtype=torch.long)] * 2, [torch.zeros(0, dtype=torch.long)] * 2, 200,
                    adj_lengths=torch.tensor([150, 150]), node_capacity=299)
    # training keeps the padded layout
    mod = parts[0]
    h = hosts[0]
    adj = Dt.PackedAdj(h["edge_index"].to(DEV), h["edge_type"].to(DEV), h["graph_ptr"], 200, None, h["graph_ptr"].to(DEV), M,
                       -1, h["edge_index"].size(1), None,
                       torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(h["adj_lengths"], 0)]).to(DEV), N_cap)
    mod.train()
    try:
        with pytest.raises(ValueError, match="eval"):
            mod(h["H"].to(DEV), adj, h["node_type"].to(DEV), h["node_score"].to(DEV))
    finally:
        mod.eval()
