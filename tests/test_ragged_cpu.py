"""Ragged batches on the host: packing, node pointers, capacities and the C ABI of the ragged entry points.  No GPU."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from qagnn_b200 import _lib
from qagnn_b200 import data as Dt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_NODE, NC = 200, 5


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("ragged") / "dev.graph.adj.pk")
    Dt.synth_adj_pickle(path, 12 * NC, seed=3)
    cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    ei, et = Dt.load_sparse_adj_data_with_contextnode(path, N_NODE, NC)[4]
    return lens, flat, ei, et


def _nested(split, qs):
    _, _, ei, et = split
    return [ei[q] for q in qs], [et[q] for q in qs]


def test_ragged_packing_reoffset_by_graph_is_the_padded_packing(split):
    lens, flat, _, _ = split
    qs = [1, 4, 5, 9]
    ei, et = _nested(split, qs)
    pad = Dt.pack_adj(ei, et, N_NODE, pin=False)
    rag = Dt.pack_adj(ei, et, N_NODE, pin=False, adj_lengths=lens[qs])
    assert rag.ragged and not pad.ragged
    assert torch.equal(rag.graph_ptr, pad.graph_ptr) and rag.n_edges == pad.n_edges
    g = torch.repeat_interleave(torch.arange(len(qs) * NC), rag.graph_ptr[1:] - rag.graph_ptr[:-1])
    back = rag.edge_index - rag.node_ptr[g] + g * N_NODE
    assert torch.equal(back, pad.edge_index) and torch.equal(rag.edge_type, pad.edge_type)
    # every endpoint lies in its graph's rows
    assert bool(((rag.edge_index >= rag.node_ptr[g]) & (rag.edge_index < rag.node_ptr[g + 1])).all())
    # the flat cache cuts the same batch
    fr = flat.pack(np.asarray(qs), pin=False, adj_lengths=lens[qs])
    assert torch.equal(fr.edge_index, rag.edge_index) and torch.equal(fr.node_ptr, rag.node_ptr)
    fk = flat.pack(np.asarray(qs), pin=False, edge_capacity=rag.n_edges + 17, adj_lengths=lens[qs], node_capacity=5000)
    assert fk.edge_index.shape == (2, rag.n_edges + 17) and fk.node_capacity == 5000
    assert torch.equal(fk.edge_index[:, :rag.n_edges], rag.edge_index) and bool((fk.edge_index[:, rag.n_edges:] == 0).all())


def test_node_ptr_is_the_cumsum_of_adj_lengths(split):
    lens, flat, _, _ = split
    qs = [0, 2, 3]
    rag = flat.pack(np.asarray(qs), pin=False, adj_lengths=lens[qs])
    want = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(lens[qs].reshape(-1), 0)])
    assert torch.equal(rag.node_ptr, want)
    assert rag.node_capacity == int(want[-1])


def test_capacity_errors_fire_before_any_copy(split, monkeypatch):
    lens, flat, _, _ = split
    qs = [6, 7]
    rag = flat.pack(np.asarray(qs), pin=False, adj_lengths=lens[qs])
    ei, et = _nested(split, qs)

    def no_buffer(*a, **k):
        raise AssertionError("a buffer was allocated before the capacity check")
    for kw in ({"node_capacity": rag.node_capacity - 1}, {"edge_capacity": rag.n_edges - 1}):
        with monkeypatch.context() as m:
            m.setattr(torch, "empty", no_buffer)  # the [3, K] edge buffer
            with pytest.raises(ValueError, match="capacity"):
                flat.pack(np.asarray(qs), pin=False, adj_lengths=lens[qs], **kw)
        with pytest.raises(ValueError, match="capacity"):
            Dt.pack_adj(ei, et, N_NODE, pin=False, adj_lengths=lens[qs], **kw)
    with pytest.raises(ValueError, match="adj_lengths"):
        flat.pack(np.asarray(qs), pin=False, adj_lengths=torch.zeros(len(qs), NC, dtype=torch.long))


@pytest.mark.parametrize("bs", [1, 3, 5, 12])
def test_split_node_capacity_is_the_largest_batch_in_order(split, bs):
    lens = split[0]
    brute = 0
    for a in range(0, lens.size(0), bs):
        brute = max(brute, int(lens[a:a + bs].sum()))
    assert Dt.split_node_capacity(lens, bs) == brute
    assert Dt.split_node_capacity(lens, bs) <= bs * NC * N_NODE


RAGGED_EXPORTS = ("qagnn_graph_prep_ragged", "qagnn_gatconve_forward_ragged", "qagnn_mp_forward_ragged",
                  "qagnn_decoder_head_ragged", "qagnn_decoder_tail_ragged")


def test_ragged_entry_points_are_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    for name in RAGGED_EXPORTS:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert name in _lib.EXPORTS, name
    assert re.search(r"#define QAGNN_ABI_VERSION 3\b", header)


def test_ragged_tiled_kernel_adds_no_spills(tmp_path):
    """The ragged instantiations of the tiled message-passing kernel spill no more than the uniform ones they sit beside."""
    from qagnn_b200 import build as B
    out = subprocess.run([B._nvcc(), "-c", os.path.join(B.CSRC, "mp_headtile.cu"), "-o", str(tmp_path / "mp.o")] + B.NVCC_FLAGS,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    spills = {}
    for m in re.finditer(r"mp_headtile_kernelILi(\d)ELi(\d+)ELb(\d)E.*?\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads", out):
        spills[(m.group(1), m.group(2), m.group(3))] = (int(m.group(4)), int(m.group(5)))
    assert len(spills) == 8, out
    for (cpl, w, rag), (st, ld) in spills.items():
        if rag == "1":
            assert st <= spills[(cpl, w, "0")][0] and ld <= spills[(cpl, w, "0")][1], (cpl, w, st, ld)
