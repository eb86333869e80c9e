"""Host-side logic of pipeline.SplitTrainBatch: how an optimiser batch is cut into chunks of full micro-batches, and the
refusals raised at construction or at a call before anything reaches a device.  A DeviceSplit and a decoder on the CPU
run the same host code; no GPU needed."""
import os
import tempfile

import numpy as np
import pytest
import torch

import qagnn_b200
from qagnn_b200 import data as Dt
from qagnn_b200.pipeline import SplitTrainBatch, train_chunks

T, R, N, NC, Q, SENT_DIM = 4, 38, 200, 5, 12, 48


@pytest.mark.parametrize("mbs", [1, 2, 3])
@pytest.mark.parametrize("branches", [1, 2, 4, 8, 32])
@pytest.mark.parametrize("n", [1, 5, 6, 64, 65, 128])
def test_chunks_hold_every_full_micro_batch_in_order(n, branches, mbs):
    batch = np.arange(1000, 1000 + n)
    chunks = train_chunks(batch, mbs, branches)
    micro = [q for c in chunks for q in c]
    assert all(1 <= len(c) <= branches for c in chunks)
    assert all(len(c) == branches for c in chunks[:-1])  # only the last chunk may be short
    assert all(len(q) == mbs for q in micro)
    full = n // mbs * mbs
    assert np.array_equal(np.concatenate(micro) if micro else np.zeros(0, dtype=batch.dtype), batch[:full])
    assert len(chunks) == -(-(n // mbs) // branches)


def test_six_micro_batches_at_four_branches_split_four_and_two():
    assert [len(c) for c in train_chunks(np.arange(12), 2, 4)] == [4, 2]


@pytest.fixture(scope="module")
def split():
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, Q * NC, seed=29)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N, NC)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC, N)
    cids = torch.where(cids > 0, cids % 50 + 1, 0)
    labels = torch.arange(Q) % NC
    return flat, Dt.DeviceSplit(flat, cids, ntypes, scores, lens, "cpu", T, R, labels=labels)


def _decoder():
    torch.manual_seed(0)
    return qagnn_b200.QAGNN(None, 2, T, R, SENT_DIM, 50, 32, 32, 2, 32, 1, 0.0, 0.0, 0.0).train()


def _tb(split, dec=None, **kw):
    flat, s = split
    args = dict(branches=2, edge_capacity=flat.max_batch_edges(2), max_edges=flat.max_graph_edges())
    args.update(kw)
    return SplitTrainBatch(dec if dec is not None else _decoder(), s, 2, **args)


@pytest.mark.parametrize("branches", [0, -1])
def test_fewer_than_one_branch_is_refused(split, branches):
    with pytest.raises(ValueError, match="branches"):
        _tb(split, branches=branches)


def test_construction_refusals(split):
    with pytest.raises(ValueError, match="train"):
        _tb(split, dec=_decoder().eval())
    with pytest.raises(ValueError, match="loss"):
        _tb(split, loss="hinge")
    with pytest.raises(ValueError, match="autocast_dtype"):
        _tb(split, autocast_dtype=torch.float64)
    dec = _decoder()
    dec.gnn.edge_encoder[1].momentum = None
    with pytest.raises(ValueError, match="momentum=None"):
        _tb(split, dec=dec)
    flat, s = split
    unlabelled = Dt.DeviceSplit(flat, s.concept_ids.view(Q, NC, N), s.node_type_ids.view(Q, NC, N),
                                s.node_scores.view(Q, NC, N, 1), s.lens.view(Q, NC), "cpu", T, R)
    with pytest.raises(ValueError, match="labels"):
        _tb((flat, unlabelled))


def _sv(n_questions=2):
    return torch.zeros(n_questions * NC, SENT_DIM)


def test_call_refusals_before_anything_is_enqueued(split):
    tb = _tb(split)
    q0, q1, q2 = np.arange(0, 2), np.arange(2, 4), np.arange(4, 6)
    with pytest.raises(ValueError, match="a chunk of 3"):
        tb([q0, q1, q2], [_sv(), _sv(), _sv()])
    with pytest.raises(ValueError, match="a chunk of 0"):
        tb([], [])
    with pytest.raises(ValueError, match="a micro-batch of 1 questions"):
        tb([q0, q1[:1]], [_sv(), _sv(1)])
    with pytest.raises(ValueError, match="1 sent_vecs for 2"):
        tb([q0, q1], [_sv()])
    with pytest.raises(ValueError, match="sent_vecs is"):
        tb([q0], [torch.zeros(2 * NC, SENT_DIM + 1)])
    with pytest.raises(ValueError, match="sent_vecs is"):
        tb([q0], [torch.zeros(2 * NC, SENT_DIM, dtype=torch.int64)])
    with pytest.raises(IndexError, match="question id"):
        tb([np.array([0, Q])], [_sv()])
    tb.decoder.eval()
    with pytest.raises(RuntimeError, match="train"):
        tb([q0], [_sv()])
    assert tb.calls == 0 and tb._slots is None
