"""The CUDA-graph captures of QAGNN_Message_Passing (its use_cuda_graph cache), pipeline.DecoderStep and pipeline.TrainStep
share one capture guard: all three refuse a packed batch whose graph prep is not the packed one, and report a bad index
in a replayed batch at a later call without blocking the host.  Also the graph prep that prepare_graph() chooses.
Needs a GPU: run with -m gpu."""
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200.data import PackedAdj
from qagnn_b200.layers import MLP, MultiheadAttPoolLayer
from qagnn_b200.pipeline import DecoderStep, TrainStep
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R, D, K_LAYERS, S = 4, 38, 64, 2, 48


def _module(seed):
    mod = qagnn_b200.QAGNN_Message_Passing(None, K_LAYERS, T, R, D, D, D).eval()
    mod.load_state_dict(O.random_state_dict(K_LAYERS, D, T, R, "peaky", seed))
    return mod.to(DEV)


def _packed_prep_edge_limit(n):
    """The largest max_edges qagnn_graph_prep_packed accepts for n-node sub-graphs: one CTA holds 5n + 2 + 9 (max_edges + n)
    int32 in shared memory and keeps 4 KB of the opt-in limit free (csrc/graph_prep.cu)."""
    optin = torch.cuda.get_device_properties(DEV).shared_memory_per_block_optin
    return ((optin - 4096) // 4 - 5 * n - 2) // 9 - n


@pytest.fixture(scope="module")
def large_subgraphs():
    """Four 200-node sub-graphs of 6,500 edges each, packed at an edge capacity with 1,000 spare columns: past the
    packed prep's one-CTA limit, so graph prep falls back to the general kernels."""
    B, n, e = 4, 200, 6500
    assert e > _packed_prep_edge_limit(n)
    inp = O.synth_graph_batch(B, n, e, D, R, seed=17)
    E, K = B * e, B * e + 1000
    buf = torch.zeros(3, K, dtype=torch.long)
    buf[:2, :E], buf[2, :E] = inp["edge_index"], inp["edge_type"]
    gp = torch.arange(B + 1) * e
    adj = PackedAdj(buf[:2], buf[2], gp, n, buf, n_edges=E, edge_capacity=K).to(DEV)
    assert adj.max_edges == e
    return {k: v.to(DEV) for k, v in inp.items()}, adj


def test_module_cache_refuses_a_packed_batch_the_packed_prep_refuses(large_subgraphs):
    d, adj = large_subgraphs
    mod = _module(3)
    eager = mod(d["H"], adj, d["node_type"], d["node_score"])  # eager: the general prep on the real columns
    assert not mod._last_prep.packed and mod._last_prep.E == adj.n_edges
    assert torch.equal(eager, mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"]))
    mod.use_cuda_graph = True
    with pytest.raises(ValueError, match="packed graph prep refuses"):
        mod(d["H"], adj, d["node_type"], d["node_score"])
    assert mod.use_cuda_graph and mod.check_indices and not mod._graphs
    # the (edge_index, edge_type) pair of the same batch is captured
    assert torch.equal(mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"]), eager)


def test_decoder_step_refuses_a_packed_batch_the_packed_prep_refuses(large_subgraphs):
    d, adj = large_subgraphs
    mod = _module(3)
    torch.manual_seed(4)
    pooler = MultiheadAttPoolLayer(2, S, D).eval().to(DEV)
    fc = MLP(D + S + D, D, 1, 0, 0.2, layer_norm=True).eval().to(DEV)
    inputs = {"H": d["H"], "edge_index": adj.edge_index, "edge_type": adj.edge_type, "node_type": d["node_type"],
              "node_score": d["node_score"], "sent_vecs": torch.randn(d["H"].size(0), S, device=DEV),
              "adj_lengths": d["adj_lengths"], "graph_ptr": adj.graph_ptr_dev}
    with pytest.raises(ValueError, match="packed graph prep refuses"):
        DecoderStep(mod, pooler, fc, inputs, use_cuda_graph=True, max_edges=adj.max_edges)
    assert not mod.use_cuda_graph and mod.check_indices


def test_train_step_refuses_a_packed_batch_the_packed_prep_refuses(large_subgraphs):
    d, adj = large_subgraphs
    torch.manual_seed(8)
    dec = qagnn_b200.QAGNN(None, K_LAYERS, T, R, S, 300, D, 32, 2, D, 1, 0.0, 0.0, 0.0).to(DEV).train()
    B, n = d["node_type"].shape
    g = torch.Generator().manual_seed(8)
    cid = torch.randint(1, 301, (B, n), generator=g)
    cid[:, 0] = 0
    with pytest.raises(ValueError, match="packed graph prep refuses"):
        TrainStep(dec, torch.randn(B, S, device=DEV), cid.to(DEV), d["node_type"], d["node_score"], d["adj_lengths"], adj,
                  max_edges=adj.max_edges)
    assert dec.gnn.check_indices


@pytest.mark.parametrize("drop_graph", [False, True])
def test_module_cache_reports_a_bad_index_of_a_replay_at_a_later_call(drop_graph):
    """A replay of the module's CUDA-graph cache cannot synchronise: its status word reaches the host on its own, and the
    forward after the copy has landed raises IndexError, also when the graph was dropped (invalidate()) in between."""
    B, n = 6, 50
    inp = O.synth_graph_batch(B, n, 200, D, R, seed=23)
    d = {k: v.to(DEV) for k, v in inp.items()}
    mod = _module(5)
    mod.use_cuda_graph = True
    args = (d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"])
    good = mod(*args).clone()  # captures (after validating the batch once, eagerly) and replays
    good_type = d["edge_type"].clone()
    d["edge_type"][d["edge_type"].numel() // 2] = R  # out of range, in the buffer the graph reads
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mod(*args)  # enqueues the bad batch: nothing here may wait for the GPU
    finally:
        torch.cuda.set_sync_debug_mode(0)
    d["edge_type"].copy_(good_type)  # from here on only the bad replay's status word can raise
    if drop_graph:
        mod.invalidate()
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        mod(*args)
    assert torch.equal(mod(*args), good)
    assert len(mod._graphs) == 1


def test_prepare_graph_accepts_cross_graph_edges_with_a_2d_node_type():
    """The batch of test_gpu_parity.py::test_cross_graph_edges_fall_back_to_the_general_kernels_in_the_module_api through
    prepare_graph: n_per_graph is a layout hint, and a cross-graph edge routes the batch to the general kernels."""
    B, n, k = 3, 20, 2
    inp = O.synth_graph_batch(B, n, 50, D, R, 9)
    sd = O.random_state_dict(k, D, T, R, "peaky", 9)
    ei = inp["edge_index"].clone()
    ei[0, 0], ei[1, 0] = 1, n + 3            # graph 0 -> graph 1
    ei[0, 1], ei[1, 1] = 2 * n + 5, 7        # graph 2 -> graph 0
    ref = O.message_passing_forward(sd, inp["H"], ei, inp["edge_type"], inp["node_type"], inp["node_score"], k, T, R)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, T, R, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = {k_: v.to(DEV) for k_, v in inp.items()}
    prep = mod.prepare_graph(ei.to(DEV), d["edge_type"], d["node_type"])
    assert prep.n_per_graph == 0 and not prep.packed
    out = mod(d["H"], (ei.to(DEV), d["edge_type"]), d["node_type"], d["node_score"], prep=prep)
    Hh.assert_close(out, ref, "cross-graph batch through prepare_graph vs oracle")
