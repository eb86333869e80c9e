"""The training micro-step without host synchronisation and as CUDA graphs: the device-side combo sort against
argsort(stable=True) / bincount, an eager training step under torch.cuda.set_sync_debug_mode("error"), and
pipeline.TrainStep (the QAGNN decoder's forward and backward replayed as two CUDA graphs) against eager training.
Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200.data import PackedAdj
from qagnn_b200.modeling_qagnn import GraphPrep
from qagnn_b200.pipeline import TrainStep
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R = 4, 38
CMB = R * T * T + T


def _grad_close(got, ref, what, floor=0.0):
    scale = max(float(ref.abs().max()), floor, 1e-6)  # the training bar of test_gpu_training.py
    Hh.assert_close(got, ref, what, atol=1e-4 * scale, rtol=1e-4)


def _packed(ei, et, B, n, capacity=None):
    """Device PackedAdj of a batch whose edges are laid out graph by graph, in an edge buffer of width `capacity`."""
    g = ei[0] // n
    assert bool((g[1:] >= g[:-1]).all())
    gp = torch.zeros(B + 1, dtype=torch.long)
    gp[1:] = torch.cumsum(torch.bincount(g, minlength=B), 0)
    E = ei.size(1)
    K = E if capacity is None else int(capacity)
    buf = torch.zeros(3, K, dtype=torch.long)
    buf[:2, :E], buf[2, :E] = ei, et
    return PackedAdj(buf[:2], buf[2], gp, n, buf, n_edges=E, edge_capacity=K).to(DEV)


# ---- combo sort ---------------------------------------------------------------------------------------------------------
def _reference_sort(prep, n_real):
    Ep = n_real + prep.N
    order = torch.argsort(prep.array("csr_src_combo")[:Ep].long(), stable=True).to(torch.int32)
    combo = prep.array("combo")
    count = torch.bincount(torch.cat([combo[:n_real], combo[prep.E:]]).long(), minlength=CMB)
    return count, order


def _check_sort(prep, n_real):
    ref_count, ref_order = _reference_sort(prep, n_real)
    count, order = prep.combo_sort()
    Ep = n_real + prep.N
    assert count.dtype == torch.int64 and order.dtype == torch.int32 and order.numel() == prep.E + prep.N
    assert torch.equal(count, ref_count) and int(count.sum()) == Ep
    assert torch.equal(order[:Ep], ref_order)
    assert torch.equal(prep.combo_count(), ref_count) and torch.equal(prep.combo_order(), ref_order)
    first = (count.clone(), order[:Ep].clone())
    prep._combo = None
    count2, order2 = prep.combo_sort()
    assert torch.equal(count2, first[0]) and torch.equal(order2[:Ep], first[1]), "two runs differ"


@pytest.mark.parametrize("name", Hh.golden_names("train"))
def test_combo_sort_on_training_goldens(name):
    fx = Hh.load_golden(name)
    inp, _ = Hh.regen_mp_inputs(fx)
    prep = GraphPrep(inp["edge_index"].to(DEV), inp["edge_type"].to(DEV), inp["node_type"].reshape(-1).to(DEV), T, R)
    _check_sort(prep, prep.E)


@pytest.mark.parametrize("case", ["cfg2", "no_edges", "single_node", "single_node_self_edge"])
def test_combo_sort_shapes(case):
    if case == "cfg2":  # 320 graphs x 200 nodes x 1000 edges: E' = 384 k, 94 tiles
        inp = O.synth_graph_batch(320, 200, 1000, 2, R, seed=3)
        ei, et, nt = inp["edge_index"], inp["edge_type"], inp["node_type"].reshape(-1)
    elif case == "no_edges":
        ei, et = torch.zeros(2, 0, dtype=torch.long), torch.zeros(0, dtype=torch.long)
        nt = torch.randint(0, T, (5000,), generator=torch.Generator().manual_seed(1))
    else:
        ei = torch.zeros(2, int(case.endswith("edge")), dtype=torch.long)
        et = torch.full((ei.size(1),), 7, dtype=torch.long)
        nt = torch.tensor([2])
    prep = GraphPrep(ei.to(DEV), et.to(DEV), nt.to(DEV), T, R)
    _check_sort(prep, prep.E)


@pytest.mark.parametrize("fill", [0.3, 0.6, 0.9])
def test_combo_sort_at_an_edge_capacity(fill):
    B, n = 40, 200
    inp = O.synth_graph_batch(B, n, 1200, 2, R, seed=11, realistic=True)
    E = inp["edge_index"].size(1)
    adj = _packed(inp["edge_index"], inp["edge_type"], B, n, capacity=int(E / fill))
    nt = inp["node_type"].reshape(-1).to(DEV)
    prep = GraphPrep(adj.edge_index, adj.edge_type, nt, T, R, n, graph_ptr=adj.graph_ptr_dev, max_edges=adj.max_edges)
    assert prep.packed and prep.E == adj.edge_capacity > E
    _check_sort(prep, E)
    exact = _packed(inp["edge_index"], inp["edge_type"], B, n)
    pe = GraphPrep(exact.edge_index, exact.edge_type, nt, T, R, n, graph_ptr=exact.graph_ptr_dev, max_edges=exact.max_edges)
    assert torch.equal(pe.combo_count(), prep.combo_count()) and torch.equal(pe.combo_order(), prep.combo_order())


# ---- decoders and batches -----------------------------------------------------------------------------------------------
def _mp_golden_decoder(name, dropout=0.0):
    """A QAGNN decoder around the message passing of an MP training golden, with the golden's graph batch."""
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    torch.manual_seed(c["seed"])
    dec = qagnn_b200.QAGNN(None, c["k"], T, R, 48, 300, c["D"], 32, 2, c["D"], 1, dropout, dropout, dropout)
    dec.gnn.load_state_dict(sd)
    g = torch.Generator().manual_seed(c["seed"] + 1)
    B, n = c["B"], c["n"]
    cid = torch.randint(1, 301, (B, n), generator=g)
    cid[:, 0] = 0
    batch = {"sent_vecs": torch.randn(B, 48, generator=g), "concept_ids": cid, "node_type_ids": inp["node_type"],
             "node_scores": inp["node_score"], "adj_lengths": inp["adj_lengths"]}
    return dec.to(DEV).train(), {k: v.to(DEV) for k, v in batch.items()}, inp["edge_index"], inp["edge_type"], n


def _decoder_golden():
    fx = Hh.load_golden("train_decoder_small")
    c = fx["case"]
    inp, sent_vecs, concept_ids = MG.build_decoder_inputs(c, fx["n_etype"])
    dec = qagnn_b200.QAGNN(None, c["k"], fx["n_ntype"], fx["n_etype"], c["sent_dim"], c["n_concept"], c["D"], c["concept_in_dim"],
                           c["n_head"], c["D"], c["n_fc_layer"], 0.0, 0.0, 0.0)
    dec.load_state_dict(fx["state_dict"], strict=True)
    batch = {"sent_vecs": sent_vecs, "concept_ids": concept_ids, "node_type_ids": inp["node_type"],
             "node_scores": inp["node_score"], "adj_lengths": inp["adj_lengths"]}
    return dec.to(DEV).train(), {k: v.to(DEV) for k, v in batch.items()}, inp["edge_index"], inp["edge_type"], c["n"]


def _zero_dropout(dec):
    for m in dec.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    dec.gnn.dropout_rate = 0.0


def _leaves(batch):
    sv = batch["sent_vecs"].clone().requires_grad_(True)
    ns = batch["node_scores"].clone().requires_grad_(True)
    return sv, ns


def _args(batch, sv, ns, adj):
    return sv, batch["concept_ids"], batch["node_type_ids"], ns, batch["adj_lengths"], adj


def _bn_buffers(dec):
    return {k: v.detach().clone() for k, v in dec.named_buffers() if "running" in k or "num_batches" in k}


def _assert_buffers(got, ref, what):
    for k in ref:
        if "num_batches" in k:
            assert int(got[k]) == int(ref[k]), f"{what}: {k}"
        else:
            Hh.assert_close(got[k], ref[k], f"{what}: {k}", atol=1e-5, rtol=1e-4)


# ---- eager training without host synchronisation ------------------------------------------------------------------------
@pytest.mark.parametrize("autocast", [None, torch.float16])
def test_eager_training_step_does_not_synchronise(autocast):
    dec, batch, ei, et, n = _mp_golden_decoder("train_cfg2tiny_prod", dropout=0.2)
    B = batch["concept_ids"].size(0)
    adj = _packed(ei, et, B, n, capacity=ei.size(1) + 500)
    dec.gnn.check_batch(adj, batch["node_type_ids"])  # index validation: once, eagerly
    dec.gnn.check_indices = False
    w = torch.randn(B, 1, device=DEV)
    ctx = (lambda: torch.autocast("cuda", dtype=autocast)) if autocast else torch.enable_grad

    def step():
        sv, ns = _leaves(batch)
        with ctx():
            logits, _ = dec(*_args(batch, sv, ns, adj))
            loss = (logits.float() * w).sum()
        loss.backward()
        return sv

    step()  # first step: builds the constant one-hot table
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sv = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert sv.grad is not None and bool(torch.isfinite(sv.grad).all())


# ---- TrainStep against eager training -----------------------------------------------------------------------------------
def _compare(step_dec, eager_dec, step_sv, step_ns, eager_sv, eager_ns):
    _grad_close(step_sv.grad, eager_sv.grad, "dL/dsent_vecs")
    _grad_close(step_ns.grad, eager_ns.grad, "dL/dnode_scores")
    ref = {k: p.grad for k, p in eager_dec.named_parameters() if p.grad is not None}
    got = {k: p.grad for k, p in step_dec.named_parameters() if p.grad is not None}
    assert got.keys() == ref.keys() and len(ref) > 10
    gmax = max(float(g.abs().max()) for g in ref.values())
    for k in ref:
        _grad_close(got[k], ref[k], f"dL/d{k}", floor=1e-2 * gmax)


@pytest.mark.parametrize("name", Hh.golden_names("train") + ["train_decoder_small"])
def test_train_step_matches_eager_training(name):
    dec, batch, ei, et, n = _decoder_golden() if name == "train_decoder_small" else _mp_golden_decoder(name)
    _zero_dropout(dec)
    B = batch["concept_ids"].size(0)
    exact, cap = _packed(ei, et, B, n), _packed(ei, et, B, n, capacity=ei.size(1) + 777)
    eager_dec, step_dec = copy.deepcopy(dec), copy.deepcopy(dec)
    step = TrainStep(step_dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=cap.max_edges)
    assert step.mode.startswith("two CUDA graphs")
    w = torch.randn(B, 1, device=DEV)
    es, en = _leaves(batch)
    ss, sn = _leaves(batch)
    for it in range(3):
        logits_e, attn_e = eager_dec(*_args(batch, es, en, exact))
        logits_s, attn_s = step(*_args(batch, ss, sn, cap))
        Hh.assert_close(logits_s, logits_e, f"step {it}: logits")
        Hh.assert_close(attn_s, attn_e, f"step {it}: pool_attn")
        loss_e, loss_s = (logits_e * w).sum(), (logits_s * w).sum()
        assert abs(float(loss_s.detach()) - float(loss_e.detach())) <= 1e-4 * (1 + abs(float(loss_e.detach())))
        loss_e.backward()
        loss_s.backward()
        _assert_buffers(_bn_buffers(step_dec), _bn_buffers(eager_dec), f"step {it}")
        if it == 0:
            _compare(step_dec, eager_dec, ss, sn, es, en)
    _compare(step_dec, eager_dec, ss, sn, es, en)  # accumulated over three micro-steps


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("split") / "train.graph.adj.pk")
    Dt.synth_adj_pickle(path, 24 * 5, seed=31)
    cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, 200, 5)
    return ntypes, scores, lens, flat


def _split_batch(split, qs, capacity, seed, sent_dim=48, n_concept=300):
    ntypes, scores, lens, flat = split
    adj = flat.pack(np.asarray(qs), pin=False, edge_capacity=capacity).to(DEV)
    B = len(qs) * 5
    g = torch.Generator().manual_seed(seed)
    cid = torch.randint(1, n_concept + 1, (B, 200), generator=g)
    cid[:, 0] = 0
    batch = {"sent_vecs": torch.randn(B, sent_dim, generator=g), "concept_ids": cid, "node_type_ids": ntypes[qs].reshape(B, 200),
             "node_scores": scores[qs].reshape(B, 200, 1), "adj_lengths": lens[qs].reshape(B)}
    return {k: v.to(DEV) for k, v in batch.items()}, adj


def _split_decoder(dropout=0.0, D=64):
    torch.manual_seed(8)
    dec = qagnn_b200.QAGNN(None, 2, T, R, 48, 300, D, 32, 2, D, 1, dropout, dropout, dropout)
    dec.gnn.load_state_dict(O.random_state_dict(2, D, T, R, "prod", seed=8))
    return dec.to(DEV).train()


def test_four_edge_counts_replay_one_capture(split):
    ntypes, scores, lens, flat = split
    BS = 2
    K, M = flat.max_batch_edges(BS), flat.max_graph_edges()
    dec = _split_decoder()
    _zero_dropout(dec)
    eager_dec, step_dec = copy.deepcopy(dec), copy.deepcopy(dec)
    qsets = [[0, 1], [5, 9], [12, 20], [3, 17]]
    batches = [_split_batch(split, qs, K, 40 + i) for i, qs in enumerate(qsets)]
    assert len({b[1].n_edges for b in batches}) == 4 and all(b[1].n_edges < K for b in batches)
    step = TrainStep(step_dec, *_args(batches[0][0], batches[0][0]["sent_vecs"], batches[0][0]["node_scores"], batches[0][1]),
                     max_edges=M)
    w = torch.randn(BS * 5, 1, device=DEV)
    for i, ((batch, cap), qs) in enumerate(zip(batches, qsets)):
        exact = _split_batch(split, qs, None, 40 + i)[1]
        es, en = _leaves(batch)
        ss, sn = _leaves(batch)
        (eager_dec(*_args(batch, es, en, exact))[0] * w).sum().backward()
        (step(*_args(batch, ss, sn, cap))[0] * w).sum().backward()
        _grad_close(ss.grad, es.grad, f"batch {i}: dL/dsent_vecs")
    ref = {k: p.grad for k, p in eager_dec.named_parameters() if p.grad is not None}
    gmax = max(float(g.abs().max()) for g in ref.values())
    for k, p in step_dec.named_parameters():
        if k in ref:
            _grad_close(p.grad, ref[k], f"accumulated dL/d{k}", floor=1e-2 * gmax)
    _assert_buffers(_bn_buffers(step_dec), _bn_buffers(eager_dec), "after four micro-steps")


def test_dropout_draws_a_new_mask_on_every_replay(split):
    dec = _split_decoder(dropout=0.5)
    dec.pooler.attn_dropout.p = 0.5
    batch, cap = _split_batch(split, [2, 6], split[3].max_batch_edges(2), 3)
    step = TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=split[3].max_graph_edges())
    a_logits, a_attn = (t.clone() for t in step(*_args(batch, batch["sent_vecs"], batch["node_scores"], cap)))
    b_logits, b_attn = (t.clone() for t in step(*_args(batch, batch["sent_vecs"], batch["node_scores"], cap)))
    B, n = batch["node_type_ids"].shape
    pos = torch.arange(n, device=DEV)
    live = ~((pos >= batch["adj_lengths"].unsqueeze(1)) | (batch["node_type_ids"] == 3))  # nodes the pooling attends to
    live = live.repeat(a_attn.size(0) // B, 1)
    zero_frac = float((a_attn[live] == 0).float().mean())
    assert 0.4 < zero_frac < 0.6, f"attention dropout 0.5 zeroed {zero_frac:.3f} of the weights"
    assert not torch.equal(a_attn, b_attn) and not torch.equal(a_logits, b_logits), "two replays drew the same masks"


def test_fp16_autocast_grad_scaler_step_refreshes_the_eval_path(split):
    dec = _split_decoder(dropout=0.1)
    batch, cap = _split_batch(split, [4, 8], split[3].max_batch_edges(2), 5)
    exact = _split_batch(split, [4, 8], None, 5)[1]
    with torch.no_grad():
        before = dec.eval()(*_args(batch, batch["sent_vecs"], batch["node_scores"], exact))[0].clone()
    dec.train()
    step = TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=split[3].max_graph_edges(),
                     autocast_dtype=torch.float16)
    opt = torch.optim.SGD([p for p in dec.parameters() if p.requires_grad], lr=0.05)
    scaler = torch.amp.GradScaler("cuda")
    sv, ns = _leaves(batch)
    logits, _ = step(*_args(batch, sv, ns, cap))
    loss = torch.nn.functional.cross_entropy(logits.float().view(2, 5), torch.tensor([1, 3], device=DEV))
    scaler.scale(loss).backward()
    scaler.step(opt)
    scaler.update()
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(sv.grad).all())
    assert all(p.grad is None or bool(torch.isfinite(p.grad).all()) for p in dec.parameters())
    with torch.no_grad():
        after = dec.eval()(*_args(batch, batch["sent_vecs"], batch["node_scores"], exact))[0]
    assert not torch.allclose(before, after, atol=1e-5), "eval output did not change after the optimiser step"
    # the running statistics the replay advanced reach the eval path's folded weights
    fresh = copy.deepcopy(dec)
    fresh.gnn.invalidate()
    for layer in fresh.gnn.gnn_layers:
        layer._folded.invalidate()
    with torch.no_grad():
        Hh.assert_close(after, fresh(*_args(batch, batch["sent_vecs"], batch["node_scores"], exact))[0], "eval vs fresh fold",
                        atol=1e-6, rtol=1e-6)


def test_construction_leaves_the_model_state_as_it_was(split):
    dec = _split_decoder(dropout=0.3)
    batch, cap = _split_batch(split, [1, 7], split[3].max_batch_edges(2), 6)
    for i, p in enumerate(dec.parameters()):
        if i % 3 == 0 and p.requires_grad:
            p.grad = torch.full_like(p, 0.25 * i)
    params = {k: v.detach().clone() for k, v in dec.named_parameters()}
    buffers = {k: v.detach().clone() for k, v in dec.named_buffers()}
    grads = {k: None if v.grad is None else v.grad.clone() for k, v in dec.named_parameters()}
    torch.cuda.manual_seed(123)
    rng = torch.cuda.get_rng_state()
    TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=split[3].max_graph_edges())
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    for k, v in dec.named_parameters():
        assert torch.equal(v.detach(), params[k]), k
        assert (v.grad is None) == (grads[k] is None) and (v.grad is None or torch.equal(v.grad, grads[k])), k
    for k, v in dec.named_buffers():
        assert torch.equal(v, buffers[k]), k


def test_bad_index_in_a_later_batch_raises_at_a_later_call(split):
    dec = _split_decoder()
    K, M = split[3].max_batch_edges(2), split[3].max_graph_edges()
    batch, cap = _split_batch(split, [0, 11], K, 7)
    step = TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=M)
    step(*_args(batch, batch["sent_vecs"], batch["node_scores"], cap))[0].sum().backward()
    bad, bad_adj = _split_batch(split, [13, 14], K, 8)
    bad_adj.edge_type[bad_adj.n_edges // 2] = 10 ** 6
    step(*_args(bad, bad["sent_vecs"], bad["node_scores"], bad_adj))  # enqueued without a check that blocks
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        step(*_args(batch, batch["sent_vecs"], batch["node_scores"], cap))


def test_batch_over_capacity_and_moved_parameters_are_refused(split):
    dec = _split_decoder()
    M = split[3].max_graph_edges()
    a, b = _split_batch(split, [0, 1], None, 9), _split_batch(split, [2, 3], None, 10)
    (batch, small), (other, big) = sorted([a, b], key=lambda x: x[1].n_edges)
    assert big.n_edges > small.n_edges
    with pytest.raises(ValueError, match="max_edges"):
        TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], small), max_edges=small.max_edges - 1)
    step = TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], small), max_edges=M)
    assert step.edge_capacity == small.n_edges
    with pytest.raises(ValueError, match="edge capacity"):
        step(*_args(other, other["sent_vecs"], other["node_scores"], big))
    step(*_args(batch, batch["sent_vecs"], batch["node_scores"], small))
    dec.cpu()
    with pytest.raises(RuntimeError, match="moved"):
        step(*_args(batch, batch["sent_vecs"], batch["node_scores"], small))
