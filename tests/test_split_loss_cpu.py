"""training.answer_loss against the reference's boolean-mask compute_loss (tests/answer_oracle.py): values and gradients bit
for bit on the CPU, in fp32 and fp64, at 2 to 8 choices, every label position, tied logits, and 1 or 64 questions; the
refusals of answer_loss and SplitTrainStep; and the oracle's accuracy count against a hand count.  No GPU needed."""
import os
import tempfile

import numpy as np
import pytest
import torch

import qagnn_b200
from qagnn_b200 import data as Dt
from qagnn_b200.pipeline import SplitTrainStep
from qagnn_b200.training import answer_loss
from tests import answer_oracle as A

LOSSES = ["cross_entropy", "margin_rank"]


def _case(bs, nc, dtype, seed, tied):
    g = torch.Generator().manual_seed(seed)
    if tied:  # three values: most questions have two or more maximal choices
        logits = torch.randint(0, 3, (bs, nc), generator=g).to(dtype) * 0.5
    else:
        logits = torch.randn(bs, nc, generator=g, dtype=dtype)
    labels = torch.randint(0, nc, (bs,), generator=g)
    if bs >= 3:  # the first, a middle and the last choice appear whatever the draw
        labels[:3] = torch.tensor([0, nc // 2, nc - 1])
    return logits, labels


def _loss_and_grad(fn, logits, layout):
    x = logits.detach().clone().requires_grad_(True)
    loss = fn(x.view(-1, 1) if layout == "flat" else x)
    (loss * 0.37).backward()  # an upstream gradient other than one
    return loss.detach(), x.grad


@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("nc", range(2, 9))
@pytest.mark.parametrize("bs", [1, 64])
@pytest.mark.parametrize("tied", [False, True], ids=["distinct", "tied"])
def test_answer_loss_equals_the_reference_bit_for_bit(loss, dtype, nc, bs, tied):
    logits, labels = _case(bs, nc, dtype, seed=nc * 100 + bs, tied=tied)
    ref, ref_grad = _loss_and_grad(lambda x: A.compute_loss(x, labels, loss), logits, "square")
    for layout in ("flat", "square"):
        got, grad = _loss_and_grad(lambda x: answer_loss(x, labels, nc, loss), logits, layout)
        assert got.dtype == ref.dtype and got.shape == () and torch.equal(got, ref), layout
        assert torch.equal(grad, ref_grad), layout


@pytest.mark.parametrize("nc", [2, 5, 8])
def test_every_label_position_at_one_question(nc):
    logits, _ = _case(1, nc, torch.float32, seed=nc, tied=False)
    for c in range(nc):
        labels = torch.tensor([c])
        for loss in LOSSES:
            ref, ref_grad = _loss_and_grad(lambda x: A.compute_loss(x, labels, loss), logits, "square")
            got, grad = _loss_and_grad(lambda x: answer_loss(x, labels, nc, loss), logits, "flat")
            assert torch.equal(got, ref) and torch.equal(grad, ref_grad), (loss, c)


def test_unknown_loss_and_margin_rank_with_one_choice_are_refused():
    logits, labels = torch.zeros(4, 1), torch.zeros(4, dtype=torch.long)
    for bad in ("hinge", "Cross_Entropy", None):
        with pytest.raises(ValueError, match="loss must be one of"):
            answer_loss(logits, labels, 1, bad)
    with pytest.raises(ValueError, match="at least 2 choices"):
        answer_loss(logits, labels, 1, "margin_rank")
    assert torch.equal(answer_loss(logits, labels, 1), torch.nn.functional.cross_entropy(logits, labels))


def test_split_train_step_refuses_a_bad_loss_before_anything_is_captured():
    nc, n, T, R = 5, 200, 4, 38
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, 4 * nc, seed=3)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, n, nc)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), nc, n)
    split = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, "cpu", T, R, labels=torch.arange(4) % nc)
    dec = qagnn_b200.QAGNN(None, 2, T, R, 48, 300, 64, 32, 2, 64, 1, 0.0, 0.0, 0.0).train()
    kw = dict(edge_capacity=flat.max_batch_edges(2), max_edges=flat.max_graph_edges())
    with pytest.raises(ValueError, match="loss must be one of"):
        SplitTrainStep(dec, split, 2, loss="hinge", **kw)


def test_evaluate_counts_against_a_hand_count():
    logits = torch.tensor([[0.1, 0.9, 0.0],    # pred 1, label 1: right
                           [2.0, 2.0, 1.0],    # tie: the first maximal choice, 0; label 1: wrong
                           [0.5, 0.5, 0.5],    # all tied: 0; label 0: right
                           [-1.0, -3.0, -0.5],  # pred 2, label 0: wrong
                           [0.0, 0.0, 7.0]])   # pred 2, label 2: right
    labels = torch.tensor([1, 1, 0, 0, 2])
    assert A.evaluate_counts(logits, labels) == (3, 5)
    assert A.evaluate_counts(logits[:1], labels[:1]) == (1, 1)
    assert A.evaluate_counts(logits[3:4], labels[3:4]) == (0, 1)
