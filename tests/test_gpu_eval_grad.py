"""Gradients through the decoder in .eval(): with grad mode on and inputs that require grad, GATConvE, QAGNN_Message_Passing
and QAGNN run the autograd path with the reference's eval semantics (running-statistics BatchNorm, no dropout), on padded
and ragged batches.  Checked against autograd of the fp64 oracle run in eval semantics.  Needs a GPU: run with -m gpu."""
import math
import re

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200 import training as TR
from qagnn_b200.layers import MultiheadAttPoolLayer
from tests import helpers as Hh
from tests.test_gpu_train_deterministic import _flag as _deterministic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R = 4, 38


def _grad_close(got, ref, what, floor=0.0):
    # the training bar of tests/test_gpu_training.py: 1e-4 of the tensor's scale plus 1e-4 relative
    assert got is not None, f"{what}: no gradient"
    scale = max(float(ref.abs().max()), floor, 1e-6)
    Hh.assert_close(got, ref, what, atol=1e-4 * scale, rtol=1e-4)


def _set_running_stats(sd, seed):
    """Non-trivial running statistics in every BatchNorm of a state dict (the 'prod' goldens have 0 / 1)."""
    g = torch.Generator().manual_seed(seed)
    for k in sorted(sd):
        if k.endswith("running_mean"):
            sd[k] = 0.3 * torch.randn(sd[k].shape, generator=g)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g)
    for k in sd:  # the layers' aliases of the shared edge encoder hold its values
        shared = re.sub(r"gnn_layers\.\d+\.edge_encoder", "edge_encoder", k)
        if shared != k and shared in sd:
            sd[k] = sd[shared]
    return sd


def _leaves64(sd):
    """fp64 copies of a state dict; floating parameters become leaves that take gradients, running statistics do not."""
    return {k: (v.double().requires_grad_(not ("running" in k or "num_batches" in k)) if v.dtype.is_floating_point else v)
            for k, v in sd.items()}


def _bn_buffers(mod):
    return {k: v.detach().clone() for k, v in mod.named_buffers() if "running" in k or "num_batches" in k}


def _assert_buffers_unchanged(mod, before):
    for k, v in _bn_buffers(mod).items():
        assert torch.equal(v, before[k]), f"{k} changed in an eval-mode forward + backward"


# ---- GATConvE against fp64 autograd, every head count ------------------------------------------------------------------
LAYER_CASES = [(name, h) for name in Hh.golden_names("layer") for h in (1, 2, 4, 8, 16)
               if Hh.load_golden(name)["case"]["D"] % h == 0]


@pytest.mark.parametrize("name,heads", LAYER_CASES)
def test_gatconve_eval_gradients_match_fp64_autograd(name, heads):
    fx = Hh.load_golden(name)
    x, extra, nt, ei, et, sd = Hh.regen_layer_inputs(fx)
    sd = _set_running_stats(dict(sd), seed=heads)
    D = x.size(1)
    T_, R_ = fx["n_ntype"], fx["n_etype"]
    pre = "gnn_layers.0."
    s64 = _leaves64(sd)
    x64, e64 = x.double().requires_grad_(True), extra.double().requires_grad_(True)
    ref_out, _, ref_alpha, _ = O.gatconve_forward(s64, "gnn_layers.0", x64, ei, et, nt, e64, T_, R_, head_count=heads,
                                                  dtype=torch.float64)
    G = torch.randn(ref_out.shape, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    (ref_out * G).sum().backward()

    enc = torch.nn.Sequential(torch.nn.Linear(R_ + 1 + 2 * T_, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(),
                              torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, T_, R_, enc, head_count=heads)
    layer.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
    layer = layer.to(DEV).eval()
    before = _bn_buffers(layer)
    xg, eg = x.to(DEV).requires_grad_(True), extra.to(DEV).requires_grad_(True)
    out, (ei_p, alpha) = layer(xg, ei.to(DEV), et.to(DEV), nt.to(DEV), eg, return_attention_weights=True)
    assert out.grad_fn is not None
    Hh.assert_close(out, ref_out, "eval-grad out")
    Hh.assert_close(alpha, ref_alpha, "alpha")
    (out * G.float().to(DEV)).sum().backward()
    _assert_buffers_unchanged(layer, before)
    _grad_close(xg.grad, x64.grad, "dL/dx")
    _grad_close(eg.grad, e64.grad, "dL/dextra")
    got = dict(layer.named_parameters())
    gmax = max(float(s64[pre + k].grad.abs().max()) for k in got)
    for k, p in got.items():
        _grad_close(p.grad, s64[pre + k].grad, f"dL/d{k}", floor=1e-2 * gmax)


# ---- QAGNN_Message_Passing against fp64 autograd ------------------------------------------------------------------------
def _mp_module(fx, sd, dropout=0.2):
    c = fx["case"]
    mod = qagnn_b200.QAGNN_Message_Passing(None, c["k"], fx["n_ntype"], fx["n_etype"], c["D"], c["D"], c["D"], dropout=dropout)
    mod.load_state_dict(sd, strict=True)
    return mod.to(DEV).eval()


@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_message_passing_eval_gradients_match_fp64_autograd(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    sd = _set_running_stats(dict(sd), seed=c["seed"] + 100)
    s64 = _leaves64(sd)
    H64 = inp["H"].double().requires_grad_(True)
    sc64 = inp["node_score"].double().requires_grad_(True)
    ref = O.message_passing_forward(s64, H64, inp["edge_index"], inp["edge_type"], inp["node_type"], sc64, c["k"],
                                    fx["n_ntype"], fx["n_etype"], dtype=torch.float64)
    G = torch.randn(ref.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    (ref * G).sum().backward()

    mod = _mp_module(fx, sd, dropout=0.5)  # dropout would show at this rate: eval semantics must switch it off
    before = _bn_buffers(mod)
    H = inp["H"].to(DEV).requires_grad_(True)
    sc = inp["node_score"].to(DEV).requires_grad_(True)
    out = mod(H, (inp["edge_index"].to(DEV), inp["edge_type"].to(DEV)), inp["node_type"].to(DEV), sc)
    Hh.assert_close(out, ref, "eval-grad out")
    (out * G.float().to(DEV)).sum().backward()
    _assert_buffers_unchanged(mod, before)
    _grad_close(H.grad, H64.grad, "dL/dH")
    _grad_close(sc.grad, sc64.grad, "dL/dnode_score")
    got = dict(mod.named_parameters())
    gmax = max(float(s64[k].grad.abs().max()) for k in got)
    for k, p in got.items():
        _grad_close(p.grad, s64[k].grad, f"dL/d{k}", floor=1e-2 * gmax)


def test_eval_gradients_are_deterministic_and_match_the_fused_forward(monkeypatch):
    """Two eval-mode forward + backward runs under deterministic algorithms give the same bits (dropout 0.5 is off), and
    the output equals the fused no-grad eval output within the parity bar."""
    fx = Hh.load_golden("cfg2small_realistic")
    inp, sd = Hh.regen_mp_inputs(fx)
    mod = _mp_module(fx, sd, dropout=0.5)
    d = {k: v.to(DEV) for k, v in inp.items()}
    adj = (d["edge_index"], d["edge_type"])
    with torch.no_grad():
        fused = mod(d["H"], adj, d["node_type"], d["node_score"])
    before = _bn_buffers(mod)
    runs = []
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # cuBLAS needs a fixed workspace in deterministic mode
    with _deterministic(True):
        for seed in (0, 1):  # a different RNG state each run: a live dropout would draw different masks
            torch.manual_seed(seed)
            mod.zero_grad(set_to_none=True)
            H = d["H"].clone().requires_grad_(True)
            sc = d["node_score"].clone().requires_grad_(True)
            out = mod(H, adj, d["node_type"], sc)
            out.square().sum().backward()
            runs.append([out.detach(), H.grad, sc.grad] + [p.grad.clone() for p in mod.parameters()])
    _assert_buffers_unchanged(mod, before)
    for i, (a, b) in enumerate(zip(*runs)):
        assert torch.equal(a, b), f"tensor {i} differs between two deterministic eval-mode runs"
    Hh.assert_close(runs[0][0], fused, "autograd path vs fused eval forward")


def test_no_grad_and_frozen_inputs_keep_the_fused_forward():
    """An eval call whose inputs do not require grad returns the fused output (no grad_fn), bit for bit, whatever grad mode."""
    fx = Hh.load_golden("cfg1_peaky_k2")
    inp, sd = Hh.regen_mp_inputs(fx)
    mod = _mp_module(fx, sd)
    d = {k: v.to(DEV) for k, v in inp.items()}
    args = (d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
    with torch.no_grad():
        a = mod(*args)
    b = mod(*args)
    assert b.grad_fn is None and torch.equal(a, b)
    with torch.no_grad():
        c = mod(d["H"].requires_grad_(True), *args[1:])
    assert c.grad_fn is None and torch.equal(a, c)


# ---- the decoder end to end ---------------------------------------------------------------------------------------------
def _decoder(name):
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    dec = qagnn_b200.QAGNN(None, c["k"], fx["n_ntype"], fx["n_etype"], c["sent_dim"], c["n_concept"], c["D"], c["concept_in_dim"], c["n_head"], c["D"],
                           c["n_fc_layer"], 0.3, 0.3, 0.3)
    sd = _set_running_stats({k: v.clone() for k, v in fx["state_dict"].items()}, seed=c["seed"])
    dec.load_state_dict(sd, strict=True)
    return c, sd, inp, sent_vecs, concept_ids, dec.to(DEV).eval()


@pytest.mark.parametrize("name", ["decoder_small", "decoder_fc1"])
def test_decoder_eval_gradients_match_fp64_autograd(name):
    c, sd, inp, sent_vecs, concept_ids, dec = _decoder(name)
    s64 = _leaves64(sd)
    s64["concept_emb.emb.weight"].requires_grad_(False)  # freeze_ent_emb=True
    sv64 = sent_vecs.double().requires_grad_(True)
    ns64 = inp["node_score"].double().requires_grad_(True)
    logits64, attn64, _ = O.qagnn_decoder_forward(s64, sv64, concept_ids, inp["node_type"], ns64, inp["adj_lengths"],
                                                  inp["edge_index"], inp["edge_type"], c["k"], T, R, c["n_head"], c["n_fc_layer"],
                                                  dtype=torch.float64)
    W = torch.randn(logits64.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    (logits64 * W).sum().backward()

    before = _bn_buffers(dec)
    sv = sent_vecs.to(DEV).requires_grad_(True)
    ns = inp["node_score"].to(DEV).requires_grad_(True)
    logits, attn = dec(sv, concept_ids.to(DEV), inp["node_type"].to(DEV), ns, inp["adj_lengths"].to(DEV),
                       (inp["edge_index"].to(DEV), inp["edge_type"].to(DEV)))
    Hh.assert_close(logits, logits64, "logits")
    Hh.assert_close(attn, attn64, "pool_attn")
    (logits * W.float().to(DEV)).sum().backward()
    _assert_buffers_unchanged(dec, before)
    _grad_close(sv.grad, sv64.grad, "dL/dsent_vecs")
    _grad_close(ns.grad, ns64.grad, "dL/dnode_scores")
    got = dict(dec.named_parameters())
    gmax = max(float(s64[k].grad.abs().max()) for k, p in got.items() if p.requires_grad)
    for k, p in got.items():
        if not p.requires_grad:
            assert p.grad is None, k
            continue
        _grad_close(p.grad, s64[k].grad, f"dL/d{k}", floor=1e-2 * gmax)
    for k in ("gnn.gnn_layers.0.linear_key.weight", "gnn.edge_encoder.0.weight", "gnn.emb_score.weight", "svec2nvec.weight",
              "concept_emb.cpt_transform.weight"):
        if k in got:
            assert got[k].grad is not None and bool(got[k].grad.abs().max() > 0), f"{k} got no gradient"


# ---- ragged equals padded -----------------------------------------------------------------------------------------------
def _split_graphs(edge_index, edge_type, B, n):
    g = edge_index[0] // n
    order = torch.argsort(g, stable=True)
    ei, et, g = edge_index[:, order], edge_type[order], g[order]
    counts = torch.bincount(g, minlength=B).tolist()
    return list(torch.split(ei - g * n, counts, dim=1)), list(torch.split(et, counts))


def _ragged_adj(edge_index, edge_type, adj_lengths, n, extra_rows):
    """A ragged device PackedAdj of a padded batch whose edges stay in each graph's first adj_lengths nodes, with
    `extra_rows` tail rows past the batch."""
    B = adj_lengths.numel()
    eis, ets = _split_graphs(edge_index, edge_type, B, n)
    return Dt.pack_adj(eis, ets, n, pin=False, adj_lengths=adj_lengths,
                       node_capacity=int(adj_lengths.sum()) + extra_rows).to(DEV)


def _loader_decoder_batch(n_questions=4, nc=5, n=200, D=200, seed=3, sent_dim=64, n_concept=400):
    import os
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_questions * nc, seed=seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, n, nc)
    pad = flat.pack(np.arange(n_questions), pin=False)
    B = n_questions * nc
    g = torch.Generator().manual_seed(seed)
    concept_ids = torch.randint(1, n_concept + 1, (B, n), generator=g)
    concept_ids[:, 0] = 0
    return {"edge_index": pad.edge_index.clone(), "edge_type": pad.edge_type.clone(), "node_type": ntypes.reshape(B, n),
            "node_score": scores.reshape(B, n, 1).float(), "adj_lengths": lens.reshape(-1), "concept_ids": concept_ids,
            "sent_vecs": torch.randn(B, sent_dim, generator=g) * 0.5, "n": n, "D": D, "n_concept": n_concept}


def _edge_case_decoder_batch(n=40, seed=11, sent_dim=48, n_concept=300):
    """Graphs of length 1 (one whose only node is a context node, so every position is masked), a graph of length n, a
    graph with nodes and no edges, and ordinary ones."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor([1, 7, n, 13, 1, 25])
    B = lens.numel()
    eis = []
    ets = []
    for b in range(B):
        L = int(lens[b])
        m = 0 if b == 1 or L == 1 else 3 * L
        eis.append(torch.stack([torch.randint(0, L, (m,), generator=g), torch.randint(0, L, (m,), generator=g)]) + b * n)
        ets.append(torch.randint(0, R, (m,), generator=g))
    nt = torch.full((B, n), 2, dtype=torch.long)
    nt[:, 0] = 3
    nt[:, 1:4] = torch.randint(0, 2, (B, 3), generator=g)
    concept_ids = torch.randint(1, n_concept + 1, (B, n), generator=g)
    concept_ids[:, 0] = 0
    return {"edge_index": torch.cat(eis, 1), "edge_type": torch.cat(ets), "node_type": nt,
            "node_score": torch.randn(B, n, 1, generator=g), "adj_lengths": lens, "concept_ids": concept_ids,
            "sent_vecs": torch.randn(B, sent_dim, generator=g) * 0.5, "n": n, "D": 64, "n_concept": n_concept}


def _fresh_decoder(bt, k=2, n_head=2, concept_in_dim=32, seed=0):
    torch.manual_seed(seed)
    D = bt["D"]
    dec = qagnn_b200.QAGNN(None, k, T, R, bt["sent_vecs"].size(1), bt["n_concept"], D, concept_in_dim, n_head, D, 1, 0.3, 0.3,
                           0.3)
    sd = _set_running_stats(dict(dec.state_dict()), seed=seed + 1)
    dec.load_state_dict(sd)
    return dec.to(DEV).eval()


def _decoder_grads(dec, bt, adj):
    dec.zero_grad(set_to_none=True)
    sv = bt["sent_vecs"].to(DEV).requires_grad_(True)
    ns = bt["node_score"].to(DEV).requires_grad_(True)
    logits, attn = dec(sv, bt["concept_ids"].to(DEV), bt["node_type"].to(DEV), ns, bt["adj_lengths"].to(DEV), adj)
    W = torch.randn(logits.shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    (logits * W).sum().backward()
    grads = {"sent_vecs": sv.grad, "node_scores": ns.grad}
    grads.update({k: p.grad for k, p in dec.named_parameters() if p.requires_grad})
    return logits.detach(), attn.detach(), grads


@pytest.mark.parametrize("batch", ["edge_cases", "loader_shaped"])
def test_ragged_decoder_gradients_equal_the_padded_ones(batch, monkeypatch):
    bt = _edge_case_decoder_batch() if batch == "edge_cases" else _loader_decoder_batch()
    dec = _fresh_decoder(bt)
    before = _bn_buffers(dec)
    padded = (bt["edge_index"].to(DEV), bt["edge_type"].to(DEV))
    ragged = _ragged_adj(bt["edge_index"], bt["edge_type"], bt["adj_lengths"], bt["n"], extra_rows=37)
    lp, ap, gp = _decoder_grads(dec, bt, padded)
    lr, ar, gr = _decoder_grads(dec, bt, ragged)
    _assert_buffers_unchanged(dec, before)
    Hh.assert_close(lr, lp, "logits")
    Hh.assert_close(ar, ap, "pool_attn", atol=2e-5)
    gmax = max(float(g.abs().max()) for g in gp.values())
    assert gp.keys() == gr.keys()
    for k in gp:
        assert gr[k] is not None, k
        _grad_close(gr[k], gp[k], f"ragged dL/d{k}", floor=1e-2 * gmax)
    # and a second ragged run gives the same bits (deterministic sums in the pooling backward and the edge table)
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    with _deterministic(True):
        _, _, g1 = _decoder_grads(dec, bt, ragged)
        _, _, g2 = _decoder_grads(dec, bt, ragged)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), f"ragged dL/d{k} differs between two deterministic runs"


def test_ragged_message_passing_gradients_equal_the_padded_valid_rows():
    """dL/dH on the valid rows, dL/dnode_score and every parameter gradient of QAGNN_Message_Passing on a ragged batch with
    tail rows equal the padded batch's; the tail rows get exactly zero gradient."""
    bt = _loader_decoder_batch()
    fx = Hh.load_golden("cfg2small_realistic")
    _, sd = Hh.regen_mp_inputs(fx)
    mod = _mp_module(fx, _set_running_stats(dict(sd), seed=8), dropout=0.5)
    n, D = bt["n"], 200
    B = bt["adj_lengths"].numel()
    H = torch.randn(B, n, D, generator=torch.Generator().manual_seed(1)) * 0.5
    rows = torch.cat([b * n + torch.arange(int(bt["adj_lengths"][b])) for b in range(B)])
    adj = _ragged_adj(bt["edge_index"], bt["edge_type"], bt["adj_lengths"], n, extra_rows=50)
    N_cap = adj.node_capacity
    Hp = torch.zeros(N_cap, D)
    Hp[:rows.numel()] = H.reshape(-1, D)[rows]
    ntp = torch.full((N_cap,), 2, dtype=torch.long)
    ntp[:rows.numel()] = bt["node_type"].reshape(-1)[rows]
    nsp = torch.zeros(N_cap, 1)
    nsp[:rows.numel()] = bt["node_score"].reshape(-1, 1)[rows]
    G = torch.randn(B * n, D, generator=torch.Generator().manual_seed(2))

    def run(Hin, A, nt, ns, Gin):
        mod.zero_grad(set_to_none=True)
        Hg, sg = Hin.to(DEV).requires_grad_(True), ns.to(DEV).requires_grad_(True)
        out = mod(Hg, A, nt.to(DEV), sg)
        (out.reshape(-1, D) * Gin.to(DEV)).sum().backward()
        return out.detach().reshape(-1, D), Hg.grad.reshape(-1, D), sg.grad.reshape(-1), {k: p.grad for k, p in mod.named_parameters()}

    Gp, Gr = torch.zeros(B * n, D), torch.zeros(N_cap, D)  # no gradient from the padding or tail rows' outputs
    Gp[rows] = G[rows]
    Gr[:rows.numel()] = G[rows]
    op, hp, sp, pp = run(H, (bt["edge_index"].to(DEV), bt["edge_type"].to(DEV)), bt["node_type"], bt["node_score"], Gp)
    orr, hr, sr, pr = run(Hp, adj, ntp, nsp, Gr)
    nv = rows.numel()
    r = rows.to(DEV)
    Hh.assert_close(orr[:nv], op[r], "ragged out rows")
    _grad_close(hr[:nv], hp[r], "ragged dL/dH valid rows")
    _grad_close(sr[:nv], sp[r], "ragged dL/dnode_score valid rows")
    assert bool((hr[nv:] == 0).all()) and bool((sr[nv:] == 0).all()), "tail rows got a gradient"
    gmax = max(float(g.abs().max()) for g in pp.values())
    for k in pp:
        _grad_close(pr[k], pp[k], f"ragged dL/d{k}", floor=1e-2 * gmax)


def test_ragged_core_kernels_match_the_general_prep(monkeypatch):
    """The message-passing core forward and its backward kernels (atomic and deterministic, fp32 and bf16) on a ragged
    GraphPrep give what they give on the general prep of the same edges: they walk CSR row pointers only.  The tail rows
    carry a self loop and nothing else."""
    from qagnn_b200.modeling_qagnn import GraphPrep
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    bt = _loader_decoder_batch()
    adj = _ragged_adj(bt["edge_index"], bt["edge_type"], bt["adj_lengths"], bt["n"], extra_rows=41)
    N_cap, D, Hh_ = adj.node_capacity, 64, 4
    B = bt["adj_lengths"].numel()
    rows = torch.cat([b * bt["n"] + torch.arange(int(bt["adj_lengths"][b])) for b in range(B)])
    nt = torch.full((N_cap,), 2, dtype=torch.long)
    nt[:rows.numel()] = bt["node_type"].reshape(-1)[rows]
    nt = nt.to(DEV)
    pr = GraphPrep(adj.edge_index, adj.edge_type, nt, T, R, bt["n"], graph_ptr=adj.graph_ptr_dev, max_edges=adj.max_edges,
                   node_ptr=adj.node_ptr_dev)
    pg = GraphPrep(adj.edge_index, adj.edge_type, nt, T, R, 0)
    assert pr.node_ptr is not None and int(pr.status_word().item()) == 0
    tail = torch.arange(N_cap, device=DEV) >= rows.numel()
    for key in ("rowptr_src", "rowptr_tgt"):
        assert bool((pr.array(key).diff()[tail] == 1).all()), f"{key}: a tail row has an edge besides its self loop"
    g = torch.Generator().manual_seed(4)
    C_ = R * T * T + T
    qkm = torch.randn(N_cap, 3 * D, generator=g).to(DEV)
    ke, me = torch.randn(C_, D, generator=g).to(DEV), torch.randn(C_, D, generator=g).to(DEV)
    G = torch.randn(N_cap, D, generator=g).to(DEV)
    for dt in (torch.float32, torch.bfloat16):
        for det in (False, True):
            res = []
            for prep in (pr, pg):
                q, k_, m = (t.to(dt).clone().requires_grad_(True) for t in (qkm, ke, me))
                with _deterministic(det):
                    aggr, alpha = TR._MPCore.apply(q, k_, m, prep, (N_cap, prep.E, D, Hh_, T, R), True)
                    (aggr.float() * G).sum().backward()
                res.append([aggr.detach().float(), alpha, q.grad.float(), k_.grad.float(), m.grad.float()])
            tol = 1e-4 if dt == torch.float32 else 2.0 ** -7
            for name, a, b in zip(("aggr", "alpha", "d_qkm", "d_ke", "d_me"), *res):
                if det or name in ("aggr", "alpha"):
                    assert torch.equal(a, b), f"{dt} det={det}: {name} differs between the ragged and the general prep"
                else:  # float atomics: the order of the sums may differ
                    Hh.assert_close(a, b, f"{dt}: {name}", atol=tol * float(b.abs().max()), rtol=tol)
            if dt == torch.float32:  # and both are the graph part of the layer, computed in fp64 on the ragged prep's edges
                from tests.test_gpu_train_bf16 import _mp_core_ref64
                Ep = pr.E + N_cap
                src, tgt, combo = (pr.array(k)[:Ep].long() for k in ("src", "tgt", "combo"))
                ref, _ = _mp_core_ref64(qkm.double(), ke.double(), me.double(), src, tgt, combo, Hh_)
                Hh.assert_close(res[0][0], ref, "ragged aggr vs fp64")


def test_ragged_training_is_still_refused():
    bt = _edge_case_decoder_batch()
    dec = _fresh_decoder(bt).train()
    adj = _ragged_adj(bt["edge_index"], bt["edge_type"], bt["adj_lengths"], bt["n"], extra_rows=3)
    with pytest.raises(ValueError, match="eval"):
        dec(bt["sent_vecs"].to(DEV), bt["concept_ids"].to(DEV), bt["node_type"].to(DEV), bt["node_score"].to(DEV),
            bt["adj_lengths"].to(DEV), adj)


# ---- the ragged pooling backward against the PyTorch pooler ------------------------------------------------------------
@pytest.mark.parametrize("heads", range(1, 9))
def test_ragged_pooling_backward_matches_the_pytorch_pooler(heads):
    """pool_concat_ragged's gradients (qagnn_attention_pool_backward_ragged) against the PyTorch pooler in fp64 on the
    re-padded batch, at graph lengths 1 to 200, a graph whose every node is masked, and tail rows; bit-identical twice."""
    n, S = 200, 40
    D = 24 * heads
    lens = torch.tensor([1, 2, 7, 31, 64, 113, 199, 200, 1])
    B = lens.numel()
    g = torch.Generator().manual_seed(heads)
    nt = torch.randint(0, 4, (B, n), generator=g)
    nt[-1, 0] = 3  # a graph of one context node: every position masked, node 0 kept
    X = torch.randn(B, n, D, generator=g)
    q = torch.randn(B, S, generator=g)
    torch.manual_seed(heads)
    pool = MultiheadAttPoolLayer(heads, S, D).to(DEV).eval()
    for p in pool.parameters():
        p.data.normal_(0, 0.3, generator=None)
    rows = torch.cat([b * n + torch.arange(int(lens[b])) for b in range(B)])
    N_cap = rows.numel() + 13
    Xp = torch.zeros(N_cap, D)
    Xp[:rows.numel()] = X.reshape(-1, D)[rows]
    ntp = torch.full((N_cap,), 2, dtype=torch.long)
    ntp[:rows.numel()] = nt.reshape(-1)[rows]
    node_ptr = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)]).to(DEV)
    Gc = torch.randn(B, 2 * D + S, generator=g).to(DEV)

    def ragged():
        pool.zero_grad(set_to_none=True)
        qg, xg = q.to(DEV).requires_grad_(True), Xp.to(DEV).requires_grad_(True)
        concat, attn = pool.pool_concat_ragged(qg, xg, node_ptr, ntp.to(DEV), lens.to(DEV), n)
        (concat * Gc).sum().backward()
        return [concat.detach(), attn, qg.grad, xg.grad] + [p.grad.clone() for p in pool.parameters()]

    got, again = ragged(), ragged()
    for i, (a, b) in enumerate(zip(got, again)):
        assert torch.equal(a, b), f"tensor {i} differs between two runs"
    ref_pool = MultiheadAttPoolLayer(heads, S, D).eval()
    ref_pool.load_state_dict({k: v.cpu() for k, v in pool.state_dict().items()})
    ref_pool = ref_pool.double()
    q64, x64 = q.double().requires_grad_(True), X.double().requires_grad_(True)
    mask = O.decoder_pool_mask(lens, nt)
    pooled, attn64 = ref_pool(q64, x64, mask)
    concat64 = torch.cat([pooled, q64, x64[:, 0]], 1)
    (concat64 * Gc.double().cpu()).sum().backward()
    Hh.assert_close(got[0], concat64, "concat")
    Hh.assert_close(got[1], attn64, "attn", atol=2e-5)
    _grad_close(got[2], q64.grad, "dL/dq")
    dX = torch.zeros(B * n, D, dtype=torch.float64)
    dX[rows] = got[3][:rows.numel()].cpu().double()
    _grad_close(dX.view(B, n, D), x64.grad, "dL/dX")
    assert bool((got[3][rows.numel():] == 0).all()), "tail rows got a gradient"
    # dL/dw_ks.bias is mathematically zero (softmax is shift invariant): judged on 1e-2 of the largest gradient
    gmax = max(float(p.grad.abs().max()) for p in ref_pool.parameters())
    for (k, p), gg in zip(ref_pool.named_parameters(), got[4:]):
        _grad_close(gg, p.grad, f"dL/d{k}", floor=1e-2 * gmax)


# ---- autocast -----------------------------------------------------------------------------------------------------------
MANT = {torch.float16: 10, torch.bfloat16: 7}


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_eval_gradients_under_autocast_stay_within_the_dtype(dt, monkeypatch):
    """Eval-mode gradients under autocast against the same model with the message-passing core replaced by an fp64 one
    (tests/test_gpu_train_bf16.py's approach): the CUDA core may not cost more than autocast already costs against fp32,
    plus one ulp of the dtype at the tensor's scale."""
    from tests.test_gpu_train_bf16 import _Fp64Core
    fx = Hh.load_golden("train_tiny_realistic_d100")
    inp, sd = Hh.regen_mp_inputs(fx)
    mod = _mp_module(fx, _set_running_stats(dict(sd), seed=12))
    d = {k: v.to(DEV) for k, v in inp.items()}
    W = MG.train_loss_weights(fx["case"]).to(DEV)

    def step(amp):
        mod.zero_grad(set_to_none=True)
        H = d["H"].clone().requires_grad_(True)
        sc = d["node_score"].clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=amp or torch.float32, enabled=amp is not None):
            out = mod(H, (d["edge_index"], d["edge_type"]), d["node_type"], sc)
            loss = (out.float() * W).sum()
        loss.backward()
        grads = {"H": H.grad, "node_score": sc.grad}
        grads.update({k: p.grad for k, p in mod.named_parameters()})
        return out.detach().float(), grads

    before = _bn_buffers(mod)
    out, grads = step(dt)
    f32_out, f32_grads = step(None)
    monkeypatch.setattr(TR, "_MPCore", _Fp64Core)
    ref_out, ref_grads = step(dt)
    monkeypatch.undo()
    _assert_buffers_unchanged(mod, before)
    ulp = 2.0 ** -(MANT[dt] + 1)
    err, auto = float((out - ref_out).abs().max()), float((ref_out - f32_out).abs().max())
    assert err <= auto + ulp * float(ref_out.abs().max()), f"{dt} output: {err:.3e} vs autocast's {auto:.3e}"
    gmax = max(float(g.abs().max()) for g in ref_grads.values())
    for k, g in grads.items():
        assert g is not None and bool(torch.isfinite(g).all()), f"dL/d{k} is missing or not finite"
        scale = max(float(ref_grads[k].abs().max()), 1e-2 * gmax)
        err = float((g.float() - ref_grads[k].float()).abs().max())
        auto = float((ref_grads[k].float() - f32_grads[k].float()).abs().max())
        assert err <= auto + ulp * scale, f"{dt} dL/d{k}: max|err| {err:.3e}, autocast's {auto:.3e}, scale {scale:.3e}"
    assert math.isfinite(float(out.abs().max()))
