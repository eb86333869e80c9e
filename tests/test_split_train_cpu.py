"""CPU-side checks of a split's labels (qagnn_b200.data.DeviceSplit(..., labels=)): validation at upload and a split
without labels.  A DeviceSplit on the CPU runs the same host code; no GPU needed."""
import os
import tempfile

import numpy as np
import pytest
import torch

from qagnn_b200 import data as Dt

T, R, N, NC, Q = 4, 38, 200, 5, 10


@pytest.fixture(scope="module")
def split():
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, Q * NC, seed=23)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N, NC)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC, N)
    return flat, cids, ntypes, scores, lens


def _labels():
    return torch.arange(Q) % NC


def test_labels_are_uploaded_as_int64(split):
    labels = _labels().to(torch.int32)
    s = Dt.DeviceSplit(*split, "cpu", T, R, labels=labels)
    assert s.labels.dtype == torch.int64 and torch.equal(s.labels, labels.long())
    s = Dt.DeviceSplit(*split, "cpu", T, R, labels=np.asarray(labels))
    assert torch.equal(s.labels, labels.long())


@pytest.mark.parametrize("q", [0, 4, Q - 1])
@pytest.mark.parametrize("value", [-1, NC, 10 ** 6])
def test_a_label_outside_the_choices_is_refused_naming_its_question(split, q, value):
    labels = _labels()
    labels[q] = value
    labels[-1] = NC + 1 if q < Q - 1 else labels[-1]  # a later bad label: the first one is named
    with pytest.raises(IndexError, match=f"question {q} has label {value},"):
        Dt.DeviceSplit(*split, "cpu", T, R, labels=labels)


@pytest.mark.parametrize("labels", [torch.zeros(Q - 1, dtype=torch.long), torch.zeros(Q + 1, dtype=torch.long),
                                    torch.zeros(Q, 1, dtype=torch.long), torch.zeros(Q, NC, dtype=torch.long),
                                    torch.zeros(Q), torch.zeros(Q, dtype=torch.bool)],
                         ids=["short", "long", "column", "one_hot", "float", "bool"])
def test_labels_of_another_shape_or_dtype_are_refused(split, labels):
    with pytest.raises(ValueError, match="labels"):
        Dt.DeviceSplit(*split, "cpu", T, R, labels=labels)


def test_a_split_without_labels_is_as_before(split):
    plain = Dt.DeviceSplit(*split, "cpu", T, R)
    labelled = Dt.DeviceSplit(*split, "cpu", T, R, labels=_labels())
    assert plain.labels is None
    for name in ("src", "tgt", "etype", "graph_ptr", "adj_lengths", "concept_ids", "node_type_ids", "node_scores"):
        assert torch.equal(getattr(plain, name), getattr(labelled, name)), name
    q = [3, 0, 7]
    a, b = plain.check(q, None), labelled.check(q, None)
    assert np.array_equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[3] == b[3]


def test_a_bad_split_without_labels_is_still_refused(split):
    flat, cids, ntypes, scores, lens = split
    lens = lens.clone()
    lens.reshape(-1)[13] = 0
    with pytest.raises(IndexError, match="question 2 "):
        Dt.DeviceSplit(flat, cids, ntypes, scores, lens, "cpu", T, R)
