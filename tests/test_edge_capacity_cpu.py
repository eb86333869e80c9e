"""Packed batches at a fixed edge capacity (host side): buffer layout, overflow, the split-wide bounds of FlatAdjCache and
the equal shapes PackedAdjBatchGenerator yields with them."""
import numpy as np
import pytest
import torch

from qagnn_b200 import data as Dt


def _split(tmp_path, n_records=60, n=200, nc=5, seed=3):
    path = str(tmp_path / "split.graph.adj.pk")
    Dt.synth_adj_pickle(path, n_records, seed=seed)
    return Dt.load_flat_adj_cache(path, n, nc)


def _nested(rng, B, n, sizes):
    ei = [torch.from_numpy(rng.integers(0, n, (2, s))) for s in sizes]
    et = [torch.from_numpy(rng.integers(0, 38, s)) for s in sizes]
    return [ei[i:i + 5] for i in range(0, B, 5)], [et[i:i + 5] for i in range(0, B, 5)]


@pytest.mark.parametrize("packer", ["pack_adj", "flat"])
def test_pack_with_capacity_fills_the_first_columns_and_zeroes_the_tail(packer):
    rng = np.random.default_rng(0)
    n, sizes = 30, [7, 0, 12, 3, 9, 4, 11, 0, 5, 6]
    ei, et = _nested(rng, len(sizes), n, sizes)
    exact = Dt.pack_adj(ei, et, n, pin=False)
    E, K = sum(sizes), sum(sizes) + 17
    if packer == "pack_adj":
        got = Dt.pack_adj(ei, et, n, pin=False, edge_capacity=K)
    else:
        got = Dt.FlatAdjCache.from_nested(ei, et, n).pack([0, 1], pin=False, edge_capacity=K)
    assert got.buf.shape == (3, K) and got.edge_index.shape == (2, K) and got.edge_type.shape == (K,)
    assert got.n_edges == E == int(got.graph_ptr[-1]) and got.edge_capacity == K
    assert torch.equal(got.graph_ptr, exact.graph_ptr)
    assert torch.equal(got.edge_index[:, :E], exact.edge_index) and torch.equal(got.edge_type[:E], exact.edge_type)
    assert not got.buf[:, E:].any()
    # without a capacity the buffer is exactly the batch, and the two counts agree
    assert exact.n_edges == exact.edge_capacity == E
    # .to() keeps both host counts
    moved = got.to("cpu")
    assert moved.n_edges == E and moved.edge_capacity == K and moved.max_edges == max(sizes)


@pytest.mark.parametrize("packer", ["pack_adj", "flat"])
def test_pack_over_capacity_raises_before_copying(packer):
    rng = np.random.default_rng(1)
    ei, et = _nested(rng, 5, 20, [4, 4, 4, 4, 4])
    with pytest.raises(ValueError, match="edge capacity"):
        if packer == "pack_adj":
            Dt.pack_adj(ei, et, 20, pin=False, edge_capacity=19)
        else:
            Dt.FlatAdjCache.from_nested(ei, et, 20).pack([0], pin=False, edge_capacity=19)
    assert Dt.pack_adj(ei, et, 20, pin=False, edge_capacity=20).n_edges == 20  # exactly full is fine


def test_split_bounds_hold_for_every_batch_under_any_shuffle(tmp_path):
    cids, ntypes, scores, lens, flat = _split(tmp_path)
    counts = np.diff(flat.graph_ptr)
    assert flat.max_graph_edges() == int(counts.max())
    bs = 4
    K = flat.max_batch_edges(bs)
    assert K == int(np.sort(counts)[::-1][:bs * flat.num_choice].sum())
    assert flat.max_batch_edges(flat.n_questions() + 3) == int(counts.sum())  # larger than the split: every graph
    rng = np.random.default_rng(5)
    for _ in range(20):
        order = rng.permutation(flat.n_questions())
        for a in range(0, len(order), bs):
            p = flat.pack(order[a:a + bs], pin=False, edge_capacity=K)
            per_graph = np.diff(p.graph_ptr.numpy())
            assert p.n_edges <= K and per_graph.max(initial=0) <= flat.max_graph_edges()


def test_generator_yields_equal_shapes_for_every_full_batch(tmp_path):
    cids, ntypes, scores, lens, flat = _split(tmp_path, n_records=55)  # 11 questions: two full batches of 4 + one of 3
    Q, bs = flat.n_questions(), 4
    K = flat.max_batch_edges(bs)

    class Args:
        pass
    gen = Dt.PackedAdjBatchGenerator(Args(), "eval", "cpu", "cpu", bs, torch.randperm(Q, generator=torch.Generator().manual_seed(2)),
                                     [f"q{i}" for i in range(Q)], torch.zeros(Q, dtype=torch.long),
                                     tensors1=[cids, ntypes, scores, lens], adj_data=flat, edge_capacity=K)
    plain = Dt.PackedAdjBatchGenerator(Args(), "eval", "cpu", "cpu", bs, gen.indexes, [f"q{i}" for i in range(Q)],
                                       torch.zeros(Q, dtype=torch.long), tensors1=[cids, ntypes, scores, lens], adj_data=flat)
    batches, exact = list(gen), list(plain)
    assert len(batches) == 3
    for b, x in zip(batches, exact):
        adj = b[-2]
        assert isinstance(adj, Dt.PackedAdj) and adj.edge_capacity == K and b[-1].shape == (K,)
        E = adj.n_edges
        assert torch.equal(adj.edge_index[:, :E], x[-2].edge_index) and torch.equal(adj.graph_ptr, x[-2].graph_ptr)
    full = {(tuple(b[-2].edge_index.shape), tuple(b[2].shape)) for b in batches[:2]}
    assert len(full) == 1
    with pytest.raises(ValueError):
        Dt.PackedAdjBatchGenerator(Args(), "eval", "cpu", "cpu", bs, gen.indexes, [], torch.zeros(Q), adj_data=([], []),
                                   edge_capacity=K)
