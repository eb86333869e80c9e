"""A split held on the GPU: DeviceSplit.batch against FlatAdjCache.pack, and SplitEvalStep against the eager decoder on
host-packed batches.  Every comparison is bit for bit.  Needs a GPU: run with -m gpu."""
import os
import tempfile

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200.pipeline import SplitEvalStep

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R, N = 4, 38, 200
N_CONCEPT, SENT_DIM, D = 300, 48, 64


def _load(n_questions, nc, seed):
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_questions * nc, seed=seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N, nc)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), nc, N)
    # concept ids inside the decoder's table; the context node keeps id 0
    cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)
    return cids, ntypes, scores, lens, flat


def _drop_edges(flat, graphs):
    """flat with every edge of `graphs` removed: sub-graphs with zero edges."""
    counts = np.diff(flat.graph_ptr)
    g_of = np.repeat(np.arange(flat.n_graphs()), counts)
    keep = ~np.isin(g_of, graphs)
    counts[graphs] = 0
    ptr = np.zeros_like(flat.graph_ptr)
    ptr[1:] = np.cumsum(counts)
    return Dt.FlatAdjCache(flat.src[keep], flat.tgt[keep], flat.etype[keep], ptr, flat.num_choice, flat.n_nodes)


class Split:
    def __init__(self, n_questions, nc, seed, empty=()):
        self.cids, self.ntypes, self.scores, self.lens, flat = _load(n_questions, nc, seed)
        self.flat = _drop_edges(flat, list(empty)) if empty else flat
        self.nc = nc
        self.dev = Dt.DeviceSplit(self.flat, self.cids, self.ntypes, self.scores, self.lens, DEV, T, R)

    def host(self, q, K, N_cap=None):
        """flat.pack(...).to(DEV) and the host-sliced node arrays: the reference of DeviceSplit.batch."""
        q = np.asarray(q)
        B = len(q) * self.nc
        al = self.lens[q].reshape(-1)
        adj = self.flat.pack(q, pin=False, edge_capacity=K, adj_lengths=al if N_cap is not None else None,
                             node_capacity=N_cap).to(DEV)
        return (self.cids[q].reshape(B, N).to(DEV), self.ntypes[q].reshape(B, N).to(DEV), self.scores[q].reshape(B, N, 1).to(DEV),
                al.to(DEV), adj)

    def totals(self, q):
        gids = (np.asarray(q)[:, None] * self.nc + np.arange(self.nc)).reshape(-1)
        return int(np.diff(self.flat.graph_ptr)[gids].sum()), int(self.lens.reshape(-1)[gids].sum())


@pytest.fixture(scope="module")
def s5():
    return Split(24, 5, seed=41, empty=(3, 11, 12))


@pytest.fixture(scope="module")
def s4():
    return Split(12, 4, seed=42, empty=(0,))


def _assert_same(got, ref):
    for a, b, name in zip(got[:4], ref[:4], ("concept_ids", "node_type_ids", "node_scores", "adj_lengths")):
        assert a.dtype == b.dtype and torch.equal(a, b), name
    ga, ra = got[4], ref[4]
    assert ga.buf.shape == ra.buf.shape and torch.equal(ga.buf, ra.buf), "edges"
    assert torch.equal(ga.edge_index, ra.edge_index) and torch.equal(ga.edge_type, ra.edge_type)
    assert torch.equal(ga.graph_ptr, ra.graph_ptr) and torch.equal(ga.graph_ptr_dev, ra.graph_ptr_dev)
    assert (ga.n_nodes, ga.max_edges, ga.n_edges, ga.edge_capacity, ga.node_capacity, ga.ragged) == \
           (ra.n_nodes, ra.max_edges, ra.n_edges, ra.edge_capacity, ra.node_capacity, ra.ragged)
    if ra.ragged:
        assert torch.equal(ga.node_ptr, ra.node_ptr) and torch.equal(ga.node_ptr_dev, ra.node_ptr_dev)


BATCHES = {
    "in_order": lambda s: np.arange(6),
    "shuffled": lambda s: np.random.default_rng(0).permutation(s.flat.n_questions())[:7],
    "repeated": lambda s: np.array([5, 2, 5, 0]),
    "one_question": lambda s: np.array([9]),
    "zero_edge_graphs": lambda s: np.array([2, 0, 3]),
}


@pytest.mark.parametrize("ragged", [False, True], ids=["padded", "ragged"])
@pytest.mark.parametrize("nc", [5, 4])
@pytest.mark.parametrize("case", list(BATCHES))
def test_batch_equals_host_pack(s5, s4, case, nc, ragged):
    s = s5 if nc == 5 else s4
    q = BATCHES[case](s) % s.flat.n_questions()
    e, rows = s.totals(q)
    K = e + 37  # a zero tail
    N_cap = rows + 11 if ragged else None
    _assert_same(s.dev.batch(q, K, N_cap), s.host(q, K, N_cap))


@pytest.mark.parametrize("ragged", [False, True], ids=["padded", "ragged"])
def test_batch_exactly_at_the_capacities(s5, ragged):
    q = np.array([4, 1, 7])
    e, rows = s5.totals(q)
    _assert_same(s5.dev.batch(q, e, rows if ragged else None), s5.host(q, e, rows if ragged else None))


@pytest.mark.parametrize("ragged", [False, True], ids=["padded", "ragged"])
def test_512_questions_span_several_scan_chunks(ragged):
    s = Split(512, 5, seed=43, empty=(1000, 1023, 1024))
    q = np.random.default_rng(1).permutation(512)
    K = s.flat.max_batch_edges(512)
    N_cap = Dt.split_node_capacity(s.lens, 512) if ragged else None
    got = s.dev.batch(q, K, N_cap)
    _assert_same(got, s.host(q, K, N_cap))
    assert got[4].graph_ptr.numel() == 2561


def _decoder(seed=8, k=2):
    torch.manual_seed(seed)
    dec = qagnn_b200.QAGNN(None, k, T, R, SENT_DIM, N_CONCEPT, D, 32, 2, D, 1, 0.0, 0.0, 0.0)
    dec.gnn.load_state_dict(O.random_state_dict(k, D, T, R, "prod", seed=seed))
    return dec.to(DEV).eval()


def _autocast(dt):
    return torch.autocast("cuda", dtype=dt, cache_enabled=False) if dt is not None else torch.autocast("cuda", enabled=False)


def _eager(dec, s, q, sv, K, N_cap, dt):
    with torch.no_grad(), _autocast(dt):
        logits, attn = dec(sv.float(), *s.host(q, K, N_cap))
    return logits.clone(), attn.clone()


def _order_and_bounds(s, bs, n_batches, seed):
    order = np.random.default_rng(seed).permutation(s.flat.n_questions())[:bs * n_batches]
    K, M = s.flat.max_batch_edges(bs), s.flat.max_graph_edges()
    N_cap = Dt.split_node_capacity(s.lens[torch.from_numpy(order)], bs)  # read in this fixed order
    return [order[i * bs:(i + 1) * bs] for i in range(n_batches)], K, M, N_cap


@pytest.mark.parametrize("dt", [None, torch.bfloat16], ids=["fp32", "bf16"])
def test_eight_batches_through_one_capture_equal_eager_and_ragged_equals_padded(s5, dt):
    dec = _decoder()
    bs = 3
    batches, K, M, N_cap = _order_and_bounds(s5, bs, 8, seed=2)
    g = torch.Generator(device=DEV).manual_seed(3)
    svs = [torch.randn(bs * 5, SENT_DIM, device=DEV, generator=g) for _ in batches]
    steps = {"padded": SplitEvalStep(dec, s5.dev, bs, edge_capacity=K, max_edges=M, autocast_dtype=dt),
             "ragged": SplitEvalStep(dec, s5.dev, bs, edge_capacity=K, max_edges=M, node_capacity=N_cap, autocast_dtype=dt)}
    got = {name: [] for name in steps}
    for q, sv in zip(batches, svs):
        for name, step in steps.items():
            logits, attn = step(q, sv)
            got[name].append((logits.clone(), attn.clone()))
    for name, step in steps.items():
        assert step.captures == 1 and step.graph is not None
        for (logits, attn), q, sv in zip(got[name], batches, svs):
            ref = _eager(dec, s5, q, sv, K, N_cap if name == "ragged" else None, dt)
            assert torch.equal(logits, ref[0]), name
            assert torch.equal(attn, ref[1]), name
    for (lp, ap), (lr, ar) in zip(got["padded"], got["ragged"]):
        assert torch.equal(lp, lr) and torch.equal(ap, ar)


@pytest.mark.parametrize("ragged", [False, True], ids=["padded", "ragged"])
def test_new_weights_are_captured_again_and_unchanged_ones_are_not(s5, ragged):
    dec = _decoder()
    bs = 2
    batches, K, M, N_cap = _order_and_bounds(s5, bs, 3, seed=4)
    N_cap = N_cap if ragged else None
    sv = torch.randn(bs * 5, SENT_DIM, device=DEV)
    step = SplitEvalStep(dec, s5.dev, bs, edge_capacity=K, max_edges=M, node_capacity=N_cap)
    step(batches[0], sv)
    step(batches[1], sv)
    assert step.captures == 1
    opt = torch.optim.SGD([p for p in dec.parameters() if p.requires_grad], lr=0.05)
    for p in dec.parameters():
        if p.requires_grad:
            p.grad = torch.randn_like(p)
    opt.step()
    logits, attn = step(batches[2], sv)
    assert step.captures == 2
    ref = _eager(dec, s5, batches[2], sv, K, N_cap, None)
    assert torch.equal(logits, ref[0]) and torch.equal(attn, ref[1])
    dec.load_state_dict(_decoder(seed=9).state_dict())
    logits, attn = step(batches[0], sv)
    assert step.captures == 3
    ref = _eager(dec, s5, batches[0], sv, K, N_cap, None)
    assert torch.equal(logits, ref[0]) and torch.equal(attn, ref[1])
    step(batches[1], sv)
    assert step.captures == 3


def test_bad_batches_raise_before_anything_is_enqueued(s5):
    dec = _decoder()
    bs = 2
    first = np.arange(bs)
    e, rows = s5.totals(first)
    M = s5.flat.max_graph_edges()
    sv = torch.randn(bs * 5, SENT_DIM, device=DEV)
    step = SplitEvalStep(dec, s5.dev, bs, edge_capacity=e, max_edges=M)
    logits, attn = step(first, sv)
    kept = (logits.clone(), attn.clone())
    for bad in ([0, 24], [-1, 0], [0, 10 ** 9]):
        with pytest.raises(IndexError):
            step(bad, sv)
    torch.cuda.synchronize()
    assert torch.equal(logits, kept[0]) and torch.equal(attn, kept[1])
    more_edges = next(q for q in range(24) if s5.totals([0, q])[0] > e)
    with pytest.raises(ValueError, match="edge capacity"):
        step([0, more_edges], sv)
    torch.cuda.synchronize()
    assert torch.equal(logits, kept[0]) and torch.equal(attn, kept[1])
    ragged = SplitEvalStep(dec, s5.dev, bs, edge_capacity=s5.flat.max_batch_edges(bs), max_edges=M, node_capacity=rows)
    ragged(first, sv)
    more_rows = next(q for q in range(24) if s5.totals([0, q])[1] > rows)
    with pytest.raises(ValueError, match="node capacity"):
        ragged([0, more_rows], sv)


def test_an_edge_outside_its_graphs_rows_is_refused_at_upload():
    cids, ntypes, scores, lens, flat = _load(6, 5, seed=44)
    g = 17
    src = flat.src.copy()
    src[flat.graph_ptr[g]] = int(lens.reshape(-1)[g])  # one row past the graph's last
    bad = Dt.FlatAdjCache(src, flat.tgt, flat.etype, flat.graph_ptr, 5, N)
    with pytest.raises(IndexError, match=f"question {g // 5} "):
        Dt.DeviceSplit(bad, cids, ntypes, scores, lens, DEV, T, R)


def test_a_training_decoder_is_refused(s5):
    dec = _decoder().train()
    K, M = s5.flat.max_batch_edges(2), s5.flat.max_graph_edges()
    with pytest.raises(ValueError, match="eval"):
        SplitEvalStep(dec, s5.dev, 2, edge_capacity=K, max_edges=M)
    dec.eval()
    step = SplitEvalStep(dec, s5.dev, 2, edge_capacity=K, max_edges=M)
    dec.train()
    with pytest.raises(RuntimeError, match="eval"):
        step([0, 1], torch.zeros(10, SENT_DIM, device=DEV))
