"""Keyed dropout without a GPU: the numpy mirror's Philox4x32-10 against the published Random123 known answers, its keep
rate and independence across sites, choices, questions and draws, the pinned site table, the binding and the refusals that
need no device."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from qagnn_b200 import _lib, training
from tests import keyed_dropout_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ([0xffffffff] * 4, [0xffffffff] * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    got = O.philox4x32_10(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert " ".join(f"{v:08x}" for v in got) == want


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_keep_fraction_within_5_sigma(p):
    A, G, L, nc = 2, 10, 60001, 5  # 1.2e6 elements
    keep = O.keep_mask(A, G, L, p, seed=0x1234_5678_9ABC_DEF0, draw=3, qids=np.array([7, 4_000_000_001]), nc=nc, site=1)
    n = keep.size
    assert n >= 10 ** 6
    sigma = np.sqrt(n * p * (1 - p))
    assert abs(int(keep.sum()) - n * (1 - p)) < 5 * sigma


def _agree(a, b):
    return float((a == b).mean())


def test_masks_of_other_sites_choices_questions_and_draws_agree_at_chance():
    p, L = 0.5, 40000
    base = dict(A=1, G=2, L=L, p=p, seed=99, draw=0, qids=np.array([5]), nc=2, site=0)
    m = O.keep_mask(**base)[0]
    others = {
        "site": O.keep_mask(**{**base, "site": 1})[0, 0],
        "choice": m[1],
        "question": O.keep_mask(**{**base, "qids": np.array([6])})[0, 0],
        "draw": O.keep_mask(**{**base, "draw": 1})[0, 0],
        "seed": O.keep_mask(**{**base, "seed": 100})[0, 0],
    }
    chance = p * p + (1 - p) * (1 - p)
    tol = 5 * np.sqrt(chance * (1 - chance) / L)
    for what, other in others.items():
        assert abs(_agree(m[0], other) - chance) < tol, what


def test_p_edges():
    keep0 = O.keep_mask(1, 2, 1001, 0.0, 1, 0, [0], 2, 0)
    keep1 = O.keep_mask(1, 2, 1001, 1.0, 1, 0, [0], 2, 0)
    assert keep0.all() and not keep1.any()
    assert O.threshold(1.0) == 2 ** 32 - 1 and O.threshold(0.2) == int(0.2 * 2 ** 32)


def test_pack_bits():
    keep = np.zeros(70, dtype=bool)
    keep[[0, 31, 32, 69]] = True
    assert O.pack_bits(keep).tolist() == [0x80000001, 1, 1 << 5]


def test_site_table_is_pinned():
    """The site ids are part of the mask definition: changing one changes every mask drawn at that site."""
    assert (training.SITE_EMB, training.SITE_GNN_LAYER, training.SITE_GNN_OUT, training.SITE_POOL_ATTN,
            training.SITE_POOL_OUT, training.SITE_FC_IN, training.SITE_MLP) == (0, 1, 32, 33, 34, 35, 36)
    assert training.MAX_GNN_LAYERS == 31


def test_header_and_binding():
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    for name in ("qagnn_keyed_dropout_forward_typed", "qagnn_keyed_dropout_backward_typed"):
        assert re.search(rf"\b{name}\s*\(", header), name
        assert name in _lib.EXPORTS, name
    assert _lib.EXPORTS["qagnn_keyed_dropout_forward_typed"][1][5] is ctypes.c_int64  # the seed, all 64 bits


def test_host_argument_checks():
    lib = _lib.load()
    fwd, bwd = lib.qagnn_keyed_dropout_forward_typed, lib.qagnn_keyed_dropout_backward_typed
    ok = dict(dtype=0, A=1, G=4, L=8, p=0.2, seed=1, nc=2, site=0)

    def call(**kw):
        a = {**ok, **kw}
        return fwd(a["dtype"], a["A"], a["G"], a["L"], a["p"], a["seed"], None, None, a["nc"], a["site"], None, None, None, None)

    assert call(dtype=3) == -1
    assert call(p=-0.1) == -1 and call(p=1.5) == -1 and call(p=float("nan")) == -1
    assert call(nc=0) == -1 and call(nc=3) == -1  # nc must divide G
    assert call(site=256) == -1 and call(site=-1) == -1
    assert call() == -1  # null pointers with elements to write
    assert call(L=0) == 0  # empty: nothing to launch
    assert call(A=1 << 20, G=4, L=1 << 20) == -5
    assert bwd(0, 0, 0.5, None, None, None, None) == 0
    assert bwd(0, 8, 1.5, None, None, None, None) == -1
    assert bwd(1, 8, 0.5, None, None, None, None) == -1


def test_no_key_is_torch_dropout():
    """Outside keyed_dropout the sites are F.dropout: the same generator draws."""
    x = torch.randn(6, 50)
    torch.manual_seed(3)
    want = torch.nn.functional.dropout(x, 0.3, True)
    torch.manual_seed(3)
    assert torch.equal(training.dropout(x, 0.3, True, training.SITE_FC_IN), want)
    assert torch.equal(training.dropout(x, 0.3, False, training.SITE_FC_IN), x)


def test_key_refusals_without_a_device():
    with pytest.raises(ValueError):
        training.DropoutKey(-1, "cuda:0")
    with pytest.raises(ValueError):
        training.DropoutKey(2 ** 64, "cuda:0")
    with pytest.raises(ValueError):
        training.DropoutKey(0, "cpu")
