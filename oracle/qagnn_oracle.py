"""TEST INFRASTRUCTURE — CPU oracle for the QA-GNN message-passing hot path.  NOT product code.

A plain CPU restatement (torch CPU tensors used as an ndarray library; no autograd, no
nn.Module, no CUDA) of the reference algorithm, op for op and in the reference's own
(un-factorised) form: per-edge one-hot features, per-edge edge-encoder MLP, per-edge K/M/Q
linears on gathered `[x_i ‖ e]`, `[x_j ‖ e]`, per-SOURCE softmax, out-degree rescale, per-TARGET
scatter-add.  Each function cites the reference file:line it follows (paths relative to
/root/reference).  Third-party arithmetic that is absent from /root/reference
(torch-geometric==1.7.0 `MessagePassing.propagate` / `utils.softmax`, torch-scatter==2.0.7
`scatter`; pinned in README.md:33-35) is restated from its published semantics and anchored on
the reference's call sites `modeling/modeling_qagnn.py:388,442,472,479`.

Pinning: the reference ships no tests or golden vectors for this path (SURVEY.md §4), so the
oracle is pinned against outputs of the reference's *own modules run in the build container*
(`oracle/ref_shim.py` + `oracle/make_goldens.py` → `tests/golden/*.pt`);
`tests/test_oracle_golden.py` checks this file against every one of those vectors.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs may import this module.  Weights are passed as a flat dict with the reference's
`state_dict` key names (SURVEY.md §8b "Parameter / checkpoint contract").
"""
import math

import numpy as np
import torch

BN_EPS = 1e-5  # torch.nn.BatchNorm1d default, used by modeling_qagnn.py:30,408


# ----------------------------------------------------------------------------------------------
# small pieces
# ----------------------------------------------------------------------------------------------
def gelu_tanh(x):
    """utils/layers.py:10-14 — tanh-approximation GELU."""
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * torch.pow(x, 3))))


def make_one_hot(labels, C, dtype):
    """modeling/modeling_qagnn.py:352-367."""
    out = torch.zeros(labels.numel(), C, dtype=dtype)
    out[torch.arange(labels.numel()), labels] = 1
    return out


def linear(x, sd, prefix):
    return x @ sd[prefix + ".weight"].to(x.dtype).t() + sd[prefix + ".bias"].to(x.dtype)


def batchnorm_eval(x, sd, prefix):
    """torch.nn.BatchNorm1d in eval mode (running statistics)."""
    dt = x.dtype
    mean, var = sd[prefix + ".running_mean"].to(dt), sd[prefix + ".running_var"].to(dt)
    return (x - mean) / torch.sqrt(var + BN_EPS) * sd[prefix + ".weight"].to(dt) + sd[prefix + ".bias"].to(dt)


def batchnorm_train(x, sd, prefix):
    """torch.nn.BatchNorm1d in training mode: normalises with the biased statistics of the rows of `x`
    (the running-statistics side effect is not modelled here)."""
    dt = x.dtype
    mean, var = x.mean(0), x.var(0, unbiased=False)
    return (x - mean) / torch.sqrt(var + BN_EPS) * sd[prefix + ".weight"].to(dt) + sd[prefix + ".bias"].to(dt)


def mlp_lin_bn_relu_lin(x, sd, prefix, train=False):
    """Sequential(Linear, BatchNorm1d, ReLU, Linear) — modeling_qagnn.py:30 and :408."""
    h = linear(x, sd, prefix + ".0")
    h = torch.relu(batchnorm_train(h, sd, prefix + ".1") if train else batchnorm_eval(h, sd, prefix + ".1"))
    return linear(h, sd, prefix + ".3")


def scatter_sum(src, index, dim_size):
    """torch_scatter.scatter(..., reduce='sum') along dim 0 [3P, torch-scatter 2.0.7]."""
    out = torch.zeros((dim_size,) + tuple(src.shape[1:]), dtype=src.dtype)
    return out.index_add_(0, index, src)


def scatter_max(src, index, dim_size):
    """torch_scatter.scatter(..., reduce='max') along dim 0; empty groups -> 0."""
    out = torch.full((dim_size,) + tuple(src.shape[1:]), float("-inf"), dtype=src.dtype)
    idx = index.view(-1, *([1] * (src.dim() - 1))).expand_as(src)
    out = out.scatter_reduce(0, idx, src, reduce="amax", include_self=True)
    return torch.where(torch.isinf(out), torch.zeros_like(out), out)


def segment_softmax(src, index):
    """torch_geometric.utils.softmax (1.7.0) as called at modeling_qagnn.py:472."""
    n = int(index.max()) + 1
    out = (src - scatter_max(src, index, n)[index]).exp()
    return out / (scatter_sum(out, index, n)[index] + 1e-16)


# ----------------------------------------------------------------------------------------------
# GATConvE  (modeling/modeling_qagnn.py:380-484)
# ----------------------------------------------------------------------------------------------
def gatconve_forward(sd, prefix, x, edge_index, edge_type, node_type, node_feature_extra,
                     n_ntype, n_etype, head_count=4, dtype=torch.float32, edge_encoder_prefix=None, train=False):
    """GATConvE.forward + GATConvE.message.

    Returns (out [N,D], edge_index' [2,E+N], alpha [E+N,H] (softmax BEFORE the out-degree
    rescale, modeling_qagnn.py:473), aggr [N,D] (propagate output before the node MLP)).
    `prefix` addresses the layer (e.g. 'gnn_layers.0'); the shared edge encoder is read from
    `edge_encoder_prefix` (default f'{prefix}.edge_encoder', an alias of the shared module).
    train=True: both BatchNorms use batch statistics (the module in .train(), qagnn.py:249); every op is a torch op, so
    autograd through this function gives the reference's gradients.
    """
    ee = edge_encoder_prefix if edge_encoder_prefix is not None else prefix + ".edge_encoder"
    x = x.to(dtype)
    extra = node_feature_extra.to(dtype)
    N, D = x.shape
    H = head_count
    d = D // H
    # :419-421  edge-type one-hots, self loops get their own type index n_etype
    edge_vec = make_one_hot(edge_type, n_etype + 1, dtype)
    self_edge_vec = torch.zeros(N, n_etype + 1, dtype=dtype)
    self_edge_vec[:, n_etype] = 1
    # :423-429  head (=src) / tail (=tgt) node-type one-hots
    head_vec = make_one_hot(node_type[edge_index[0]], n_ntype, dtype)
    tail_vec = make_one_hot(node_type[edge_index[1]], n_ntype, dtype)
    headtail_vec = torch.cat([head_vec, tail_vec], dim=1)
    self_head_vec = make_one_hot(node_type, n_ntype, dtype)
    self_headtail_vec = torch.cat([self_head_vec, self_head_vec], dim=1)
    # :431-433
    edge_vec = torch.cat([edge_vec, self_edge_vec], dim=0)
    headtail_vec = torch.cat([headtail_vec, self_headtail_vec], dim=0)
    edge_emb = mlp_lin_bn_relu_lin(torch.cat([edge_vec, headtail_vec], dim=1), sd, ee, train)
    # :436-438  self loops appended AFTER the real edges
    loop = torch.arange(N, dtype=torch.long).unsqueeze(0).repeat(2, 1)
    ei = torch.cat([edge_index, loop], dim=1)
    # :440-442 + [3P] propagate: x_j = x[src], x_i = x[tgt]
    x2 = torch.cat([x, extra], dim=1)
    src, tgt = ei[0], ei[1]
    x_j, x_i = x2[src], x2[tgt]
    # message  :464-470
    key = linear(torch.cat([x_i, edge_emb], dim=1), sd, prefix + ".linear_key").view(-1, H, d)
    msg = linear(torch.cat([x_j, edge_emb], dim=1), sd, prefix + ".linear_msg").view(-1, H, d)
    query = linear(x_j, sd, prefix + ".linear_query").view(-1, H, d)
    query = query / math.sqrt(d)
    scores = (query * key).sum(dim=2)
    # :471-473  softmax grouped by SOURCE node
    alpha = segment_softmax(scores, src)
    # :476-481  rescale by out-degree of the source (self loop included)
    Nn = int(src.max()) + 1
    cnt = scatter_sum(torch.ones(ei.size(1), dtype=dtype), src, Nn)[src]
    alpha_scaled = alpha * cnt.unsqueeze(1)
    out_msg = (msg * alpha_scaled.view(-1, H, 1)).view(-1, H * d)
    # [3P] aggregate: scatter-add by TARGET, dim_size = N
    aggr = scatter_sum(out_msg, tgt, N)
    # :443
    out = mlp_lin_bn_relu_lin(aggr, sd, prefix + ".mlp", train)
    return out, ei, alpha, aggr


# ----------------------------------------------------------------------------------------------
# QAGNN_Message_Passing  (modeling/modeling_qagnn.py:7-95)
# ----------------------------------------------------------------------------------------------
def node_feature_extra(sd, node_type, node_score, n_ntype, D, dtype=torch.float32, prefix=""):
    """modeling_qagnn.py:62-73,86: type embedding ‖ sin-basis score embedding -> [B*n, D]."""
    B, n = node_type.shape
    T = make_one_hot(node_type.reshape(-1), n_ntype, dtype).view(B, n, n_ntype)
    node_type_emb = gelu_tanh(linear(T, sd, prefix + "emb_node_type"))
    js = torch.arange(D // 2).unsqueeze(0).unsqueeze(0).float()
    js = torch.pow(1.1, js)  # fp32 on purpose, exactly as :70-71
    # the sine argument is formed in fp32 whatever `dtype` is: 1.1^j reaches 1.25e4, so the fp32
    # rounding of js*score is part of the function the reference defines (ill-conditioned otherwise)
    Bm = torch.sin((js * node_score.float()).to(dtype))
    node_score_emb = gelu_tanh(linear(Bm, sd, prefix + "emb_score"))
    return torch.cat([node_type_emb, node_score_emb], dim=2).view(B * n, -1)


def message_passing_forward(sd, H_in, edge_index, edge_type, node_type, node_score, k, n_ntype, n_etype,
                            head_count=4, dtype=torch.float32, prefix="", return_layers=False):
    """QAGNN_Message_Passing.forward in eval mode (dropout = identity), :53-95 with mp_helper :45-50."""
    B, n, D = H_in.shape
    Hd = H_in.to(dtype)
    extra = node_feature_extra(sd, node_type, node_score, n_ntype, D, dtype, prefix)
    X = Hd.reshape(-1, D)
    nt = node_type.reshape(-1)
    layers = []
    for l in range(k):
        X, _, alpha, aggr = gatconve_forward(sd, f"{prefix}gnn_layers.{l}", X, edge_index, edge_type, nt, extra,
                                             n_ntype, n_etype, head_count, dtype,
                                             edge_encoder_prefix=prefix + "edge_encoder")
        X = gelu_tanh(X)
        if return_layers:
            layers.append({"x": X.clone(), "alpha": alpha, "aggr": aggr})
    Xv = X.view(B, n, D)
    out = gelu_tanh(linear(Hd, sd, prefix + "Vh") + linear(Xv, sd, prefix + "Vx"))
    if return_layers:
        return out, extra, layers
    return out


# ----------------------------------------------------------------------------------------------
# QAGNN decoder  (modeling/modeling_qagnn.py:141-189) — the step either side of the hot path
# ----------------------------------------------------------------------------------------------
def batch_graph(edge_index_list, edge_type_list, n_nodes):
    """LM_QAGNN.batch_graph, modeling_qagnn.py:244-251."""
    ei = [edge_index_list[i] + i * n_nodes for i in range(len(edge_index_list))]
    return torch.cat(ei, dim=1), torch.cat(edge_type_list, dim=0)


def multihead_att_pool(sd, prefix, q, k, mask, n_head):
    """utils/layers.py:324-371 + 276-299 (eval: dropout = identity)."""
    bs, len_k, dk_orig = k.shape
    d_k = dk_orig // n_head
    qs = linear(q, sd, prefix + ".w_qs").view(bs, n_head, d_k)
    ks = linear(k, sd, prefix + ".w_ks").view(bs, len_k, n_head, d_k)
    vs = linear(k, sd, prefix + ".w_vs").view(bs, len_k, n_head, d_k)
    qs = qs.permute(1, 0, 2).contiguous().view(n_head * bs, d_k)
    ks = ks.permute(2, 0, 1, 3).contiguous().view(n_head * bs, len_k, d_k)
    vs = vs.permute(2, 0, 1, 3).contiguous().view(n_head * bs, len_k, d_k)
    m = mask.repeat(n_head, 1)
    attn = (qs.unsqueeze(1) * ks).sum(2) / np.power(d_k, 0.5)
    attn = attn.masked_fill(m, -np.inf)
    attn = torch.softmax(attn, dim=1)
    out = (attn.unsqueeze(2) * vs).sum(1)
    out = out.view(n_head, bs, d_k).permute(1, 0, 2).contiguous().view(bs, n_head * d_k)
    return out, attn


def decoder_head(sd, sv, concept_ids, node_scores, adj_lengths, dtype=torch.float32):
    """modeling_qagnn.py:153-167: the GNN input (context node GELU(svec2nvec(sv)), then the concept rows) and the
    normalised node scores.  Returns (gnn_input [B, n, D], node_scores [B, n, 1]); adj_lengths = 0 gives NaN scores."""
    gnn_input0 = gelu_tanh(linear(sv, sd, "svec2nvec")).unsqueeze(1)
    emb = sd["concept_emb.emb.weight"].to(dtype)[concept_ids[:, 1:] - 1]
    if "concept_emb.cpt_transform.weight" in sd:  # utils/layers.py:600-603
        emb = gelu_tanh(linear(emb, sd, "concept_emb.cpt_transform"))
    gnn_input = torch.cat([gnn_input0, emb], dim=1)
    n = node_scores.size(1)
    _mask = (torch.arange(n) < adj_lengths.unsqueeze(1)).to(dtype)
    ns = -node_scores.to(dtype)
    ns = ns - ns[:, 0:1, :]
    ns = ns.squeeze(2) * _mask
    mean_norm = ns.abs().sum(dim=1) / adj_lengths
    ns = (ns / (mean_norm.unsqueeze(1) + 1e-05)).unsqueeze(2)
    return gnn_input, ns


def decoder_pool_mask(adj_lengths, node_type_ids):
    """modeling_qagnn.py:174-176: the pooler's mask [B, n] (True = excluded): nodes past the length and context nodes
    (type 3); a row with every node masked keeps node 0."""
    n = node_type_ids.size(1)
    mask = torch.arange(n) >= adj_lengths.unsqueeze(1)
    mask = mask | (node_type_ids == 3)
    mask[mask.all(1), 0] = 0
    return mask


def qagnn_decoder_forward(sd, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, edge_index,
                          edge_type, k, n_ntype, n_etype, n_attention_head, n_fc_layer, head_count=4,
                          dtype=torch.float32):
    """QAGNN.forward (eval), modeling_qagnn.py:141-189.  `sd` holds the decoder's state_dict
    (keys 'svec2nvec.*', 'concept_emb.*', 'gnn.*', 'pooler.*', 'fc.layers.*')."""
    sv = sent_vecs.to(dtype)
    gnn_input, ns = decoder_head(sd, sv, concept_ids, node_scores, adj_lengths, dtype)
    gnn_output = message_passing_forward(sd, gnn_input, edge_index, edge_type, node_type_ids, ns, k, n_ntype,
                                         n_etype, head_count, dtype, prefix="gnn.")
    Z = gnn_output[:, 0]
    mask = decoder_pool_mask(adj_lengths, node_type_ids)
    graph_vecs, pool_attn = multihead_att_pool(sd, "pooler", sv, gnn_output, mask, n_attention_head)
    concat = torch.cat((graph_vecs, sv, Z), 1)
    h = concat
    for i in range(n_fc_layer + 1):  # utils/layers.py:47-87 with layer_norm=True, gelu
        h = linear(h, sd, f"fc.layers.{i}-Linear")
        if i < n_fc_layer:
            w, b = sd[f"fc.layers.{i}-LayerNorm.weight"].to(dtype), sd[f"fc.layers.{i}-LayerNorm.bias"].to(dtype)
            h = torch.nn.functional.layer_norm(h, (h.size(-1),), w, b, 1e-5)
            h = gelu_tanh(h)
    return h, pool_attn, gnn_output


# ----------------------------------------------------------------------------------------------
# Integer side: what graph-prep must reproduce bit-exactly (numpy, int64)
# ----------------------------------------------------------------------------------------------
def graph_prep_oracle(edge_index, edge_type, node_type, n_ntype, n_etype):
    """Index bookkeeping implied by modeling_qagnn.py:419-438,476-479:
    edge_index' (self loops appended), edge-feature index
    combo = (etype*T + type[src])*T + type[tgt] (self loop of v: R*T*T + type[v]), out-degree by
    source, and the stable CSR orders by source / by target."""
    ei = edge_index.numpy().astype(np.int64)
    et = edge_type.numpy().astype(np.int64)
    nt = node_type.numpy().astype(np.int64).reshape(-1)
    N = nt.shape[0]
    loop = np.arange(N, dtype=np.int64)
    src = np.concatenate([ei[0], loop])
    tgt = np.concatenate([ei[1], loop])
    etp = np.concatenate([et, np.full(N, n_etype, dtype=np.int64)])
    # index of the distinct one-hot edge feature: real edges (et, type[src], type[tgt]); self loops (type[v])
    E_real = ei.shape[1]
    combo = (etp * n_ntype + nt[src]) * n_ntype + nt[tgt]
    combo[E_real:] = n_etype * n_ntype * n_ntype + nt[src[E_real:]]
    outdeg = np.bincount(src, minlength=N).astype(np.int64)
    indeg = np.bincount(tgt, minlength=N).astype(np.int64)
    perm_src = np.argsort(src, kind="stable")
    perm_tgt = np.argsort(tgt, kind="stable")
    rowptr_src = np.concatenate([[0], np.cumsum(outdeg)])
    rowptr_tgt = np.concatenate([[0], np.cumsum(indeg)])
    return {"src": src, "tgt": tgt, "combo": combo, "outdeg": outdeg, "indeg": indeg,
            "perm_src": perm_src, "perm_tgt": perm_tgt, "rowptr_src": rowptr_src, "rowptr_tgt": rowptr_tgt}


# ----------------------------------------------------------------------------------------------
# Deterministic synthetic inputs (SURVEY.md §8d); shared by tests, goldens and bench
# ----------------------------------------------------------------------------------------------
def synth_graph_batch(B, n, e_per_graph, D, n_etype=38, seed=0, realistic=False, n_ntype=4):
    """cfg-1/cfg-2 style batch: x, extra-free inputs for QAGNN_Message_Passing.

    Plain variant: edge endpoints ~ U{0..n-1}^2 (+g*n), duplicates and i->i allowed; edge_type
    ~ U{0..R-1}; node_type ~ U{0..T-2} with node 0 of each graph = T-1 (T = n_ntype; every node is
    type 0 at T = 1); H ~ N(0,1)*0.5; scores N(0,1).
    Realistic variant (T >= 4: it uses the loader's types 0, 1, 2 and 3): adj_lengths ~ U{8..n},
    min(e/2, 2.5*len) forward edges among the valid nodes + the exact inverse half with type + R/2,
    context node 0 linked to the q/a nodes with types 0/1, padded nodes isolated (self loop only).
    At the default T = 4 the draws are those of the loader's four types.
    """
    if n_ntype < 1 or (realistic and n_ntype < 4):
        raise ValueError(f"synth_graph_batch: n_ntype = {n_ntype} (the realistic variant needs at least 4 node types)")
    g = torch.Generator().manual_seed(seed)
    H = torch.randn(B, n, D, generator=g) * 0.5
    node_score = torch.randn(B, n, 1, generator=g)
    node_type = torch.randint(0, max(n_ntype - 1, 1), (B, n), generator=g)
    node_type[:, 0] = n_ntype - 1
    if not realistic:
        ei = torch.randint(0, n, (B, 2, e_per_graph), generator=g)
        ei = ei + (torch.arange(B) * n).view(B, 1, 1)
        edge_index = ei.permute(1, 0, 2).reshape(2, B * e_per_graph).contiguous()
        edge_type = torch.randint(0, n_etype, (B * e_per_graph,), generator=g)
        adj_lengths = torch.full((B,), n, dtype=torch.long)
    else:
        half = n_etype // 2
        adj_lengths = torch.randint(min(8, n), n + 1, (B,), generator=g)
        eis, ets = [], []
        for b in range(B):
            L = int(adj_lengths[b])
            # loader layout (data_utils.py:107-136): context node, then q entities, then a entities, then others
            nq = min(int(torch.randint(1, 9, (1,), generator=g)), max(L - 2, 0))
            na = min(int(torch.randint(1, 4, (1,), generator=g)), max(L - 1 - nq, 0))
            node_type[b, 1:] = 2
            node_type[b, 1:1 + nq] = 0
            node_type[b, 1 + nq:1 + nq + na] = 1
            ef = min(e_per_graph // 2, int(2.5 * L))  # ~2.5 forward edges per node (SURVEY.md §8d cfg 3)
            nctx = min(nq + na, ef)
            s = torch.randint(1, max(L, 2), (ef,), generator=g).clamp_(max=L - 1)
            t = torch.randint(1, max(L, 2), (ef,), generator=g).clamp_(max=L - 1)
            r = torch.randint(2, half, (ef,), generator=g)
            if nctx > 0:  # context -> q/a links use relation ids 0/1 (data_utils.py:147-169)
                qa = torch.arange(1, 1 + nctx)
                s[:nctx] = 0
                t[:nctx] = qa
                r[:nctx] = node_type[b, qa]
            eis.append(torch.stack([torch.cat([s, t]), torch.cat([t, s])]) + b * n)
            ets.append(torch.cat([r, r + half]))
        edge_index = torch.cat(eis, dim=1).contiguous()
        edge_type = torch.cat(ets)
    return {"H": H, "edge_index": edge_index, "edge_type": edge_type, "node_type": node_type,
            "node_score": node_score, "adj_lengths": adj_lengths}


# per-module weight gains of the 'peaky' regime: large query/key gains make the per-source softmax
# sharp, small msg / mlp.0 gains keep activations O(1) over k layers despite the out-degree rescale
PEAKY_GAIN = {"linear_key": 2.0, "linear_query": 2.0, "linear_msg": 0.15, "mlp.0": 0.4, "mlp.3": 1.0,
              "edge_encoder.0": 1.5, "edge_encoder.3": 1.0}


def random_state_dict(k, D, n_ntype=4, n_etype=38, regime="prod", seed=0):
    """Random weights for QAGNN_Message_Passing with the reference's state_dict key names.

    'prod'  — N(0, 0.02) weights, zero biases (QAGNN._init_weights, modeling_qagnn.py:131-138):
              near-uniform attention.
    'peaky' — N(0, gain/sqrt(fan_in)) weights (gains in PEAKY_GAIN), random biases and non-trivial
              BatchNorm running statistics / affine terms: sharp attention, exercises the softmax.
    """
    g = torch.Generator().manual_seed(1000 + seed)
    sd = {}

    def lin(name, fo, fi):
        if regime == "prod":
            sd[name + ".weight"] = torch.randn(fo, fi, generator=g) * 0.02
            sd[name + ".bias"] = torch.zeros(fo)
        else:
            gain = PEAKY_GAIN.get(name.split(".")[-1] if not name[-1].isdigit() else ".".join(name.split(".")[-2:]), 1.0)
            sd[name + ".weight"] = torch.randn(fo, fi, generator=g) * (gain / math.sqrt(fi))
            sd[name + ".bias"] = torch.randn(fo, generator=g) * 0.1

    def bn(name, f):
        if regime == "prod":
            sd[name + ".weight"], sd[name + ".bias"] = torch.ones(f), torch.zeros(f)
            sd[name + ".running_mean"], sd[name + ".running_var"] = torch.zeros(f), torch.ones(f)
        else:
            sd[name + ".weight"] = 1 + 0.3 * torch.randn(f, generator=g)
            sd[name + ".bias"] = 0.2 * torch.randn(f, generator=g)
            sd[name + ".running_mean"] = 0.3 * torch.randn(f, generator=g)
            sd[name + ".running_var"] = 0.5 + torch.rand(f, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(0)

    lin("emb_node_type", D // 2, n_ntype)
    lin("emb_score", D // 2, D // 2)
    lin("edge_encoder.0", D, n_etype + 1 + 2 * n_ntype)
    bn("edge_encoder.1", D)
    lin("edge_encoder.3", D, D)
    for l in range(k):
        p = f"gnn_layers.{l}"
        for suffix in ("0.weight", "0.bias", "1.weight", "1.bias", "1.running_mean", "1.running_var",
                       "1.num_batches_tracked", "3.weight", "3.bias"):
            sd[f"{p}.edge_encoder.{suffix}"] = sd[f"edge_encoder.{suffix}"]  # aliases of the shared module
        lin(p + ".linear_key", D, 3 * D)
        lin(p + ".linear_msg", D, 3 * D)
        lin(p + ".linear_query", D, 2 * D)
        lin(p + ".mlp.0", D, D)
        bn(p + ".mlp.1", D)
        lin(p + ".mlp.3", D, D)
    lin("Vh", D, D)
    lin("Vx", D, D)
    return sd
