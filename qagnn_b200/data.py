"""Batch packing on the caller side of the hot path (SURVEY.md §8f #1).

The reference ships every batch's adjacency as a [batch][num_choice] nested Python list of small
int64 tensors, moves each one to the device separately (utils/data_utils.py:64-68) and offsets /
concatenates them per forward (modeling_qagnn.py:244-251): 2*bs*nc tiny H2D copies and bs*nc tiny
kernels.  `pack_adj` does the same offsetting and concatenation ONCE on the host into two pinned
tensors, so a batch needs two H2D copies.  The nested-list format keeps working everywhere.
"""
import os
import pickle
from dataclasses import dataclass, replace

import numpy as np
import torch


@dataclass
class PackedAdj:
    """edge_index int64 [2, total_E] with per-graph node offsets already applied, edge_type int64 [total_E],
    graph_ptr int64 [n_graphs + 1] = first edge of each graph.  When built by FlatAdjCache.pack the two tensors are views
    of ONE [3, total_E] buffer (`buf`), so the whole adjacency of a batch moves to the device in a single copy.

    Packed with an edge capacity K, edge_index / edge_type are [2, K] / [K]: the batch's `n_edges` = graph_ptr[-1] edges
    fill the first columns and the rest is zero.  Every batch of a split then has the same shapes, and the one-launch
    graph prep reads the real edge count from graph_ptr on the device (include/qagnn_b200.h, qagnn_graph_prep_packed).

    RAGGED (eval only; built by pack_adj / FlatAdjCache.pack given the batch's adj_lengths): graph g's nodes are the rows
    [node_ptr[g], node_ptr[g+1]) of the batch, node_ptr int64 [n_graphs + 1] = the exclusive cumsum of adj_lengths, and its
    edge ids are offset by node_ptr[g] instead of g * n_nodes.  `n_nodes` stays the most rows one graph may have (the loader's
    max_node_num) and `node_capacity` N_cap is the number of rows of every node array of the batch: rows >= node_ptr[-1] are
    unused.  The modules take such a batch in .eval() with node arrays of N_cap rows and no padding."""
    edge_index: torch.Tensor
    edge_type: torch.Tensor
    graph_ptr: torch.Tensor
    n_nodes: int
    buf: torch.Tensor = None

    graph_ptr_dev: torch.Tensor = None   # graph_ptr on the device of edge_index (packed graph prep, one launch per batch)
    max_edges: int = -1                  # max edges of one sub-graph (host value; -1 = derive from graph_ptr)
    n_edges: int = -1                    # edges of the batch = graph_ptr[-1] (host value; -1 = unknown)
    edge_capacity: int = -1              # width of edge_index (host value; -1 = unknown)

    node_ptr: torch.Tensor = None        # ragged batches: first row of every graph, int64 [n_graphs + 1] (host)
    node_ptr_dev: torch.Tensor = None    # node_ptr on the device of edge_index
    node_capacity: int = -1              # ragged batches: rows of every node array (N_cap)

    @property
    def ragged(self):
        return self.node_ptr is not None or self.node_ptr_dev is not None

    def to(self, device, non_blocking=True):
        def up(t):
            if torch.cuda.is_available() and torch.device(device).type == "cuda" and not t.is_cuda and not t.is_pinned():
                t = t.pin_memory()
            return t.to(device, non_blocking=non_blocking)
        gpd = up(self.graph_ptr)
        npd = up(self.node_ptr) if self.node_ptr is not None else self.node_ptr_dev
        me = self.max_edges if self.max_edges >= 0 else (int((self.graph_ptr[1:] - self.graph_ptr[:-1]).max()) if self.graph_ptr.numel() > 1 else 0)
        if self.buf is not None:
            b = self.buf.to(device, non_blocking=non_blocking)
            return replace(self, edge_index=b[:2], edge_type=b[2], buf=b, graph_ptr_dev=gpd, max_edges=me, node_ptr_dev=npd)
        return replace(self, edge_index=self.edge_index.to(device, non_blocking=non_blocking),
                       edge_type=self.edge_type.to(device, non_blocking=non_blocking), graph_ptr_dev=gpd, max_edges=me,
                       node_ptr_dev=npd)

    # LM_QAGNN.forward slices inputs positionally and calls .size() only on tensors before the last two; everywhere an
    # (edge_index, edge_type) pair is expected a PackedAdj unpacks / indexes as that pair
    def __iter__(self):
        return iter((self.edge_index, self.edge_type))

    def __getitem__(self, i):
        return (self.edge_index, self.edge_type)[i]

    def __len__(self):
        return 2


def _capacity(total, edge_capacity):
    """Width of a packed batch's edge buffer; raises before anything is copied when the batch does not fit."""
    if edge_capacity is None:
        return total
    if int(edge_capacity) < total:
        raise ValueError(f"batch has {total} edges, more than the edge capacity {int(edge_capacity)}")
    return int(edge_capacity)


def _etype_int16(etype, what):
    """`etype` as int16, the width the flat cache and DeviceSplit store edge types in.  numpy's cast wraps (65541 -> 5), and
    a wrapped type is a valid but wrong relation, so a value outside int16 raises instead."""
    et = np.asarray(etype)
    if et.size and (int(et.min()) < -(1 << 15) or int(et.max()) >= 1 << 15):
        bad = int(et.max()) if int(et.max()) >= 1 << 15 else int(et.min())
        raise ValueError(f"{what}: edge type {bad} does not fit the int16 edge types of the flat adjacency")
    return np.ascontiguousarray(et, dtype=np.int16)


def node_ptr_of(adj_lengths, n_nodes, n_graphs):
    """node_ptr int64 [n_graphs + 1] = the exclusive cumsum of a batch's adj_lengths (any shape, one entry per graph); raises
    ValueError for a length outside [1, n_nodes]."""
    lens = torch.as_tensor(adj_lengths).reshape(-1).to("cpu", torch.long)
    if lens.numel() != n_graphs:
        raise ValueError(f"adj_lengths has {lens.numel()} entries for {n_graphs} graphs")
    if n_graphs and (int(lens.min()) < 1 or int(lens.max()) > n_nodes):
        raise ValueError(f"adj_lengths must lie in [1, {n_nodes}] (got {int(lens.min())}..{int(lens.max())})")
    ptr = torch.zeros(n_graphs + 1, dtype=torch.long)
    ptr[1:] = torch.cumsum(lens, 0)
    return ptr


def _node_capacity(total, node_capacity):
    """Rows of a ragged batch's node arrays; raises before anything is copied when the batch does not fit."""
    if node_capacity is None:
        return total
    if int(node_capacity) < total:
        raise ValueError(f"batch has {total} nodes, more than the node capacity {int(node_capacity)}")
    return int(node_capacity)


def largest_edges(counts, m):
    """Edges of the `m` largest sub-graphs of a split together, from its per-sub-graph edge counts."""
    m = min(int(m), len(counts))
    return int(np.sort(counts)[len(counts) - m:].sum()) if m > 0 else 0


def split_node_capacity(adj_lengths, batch_size):
    """Node capacity of a ragged split read in a FIXED batch order (dev and test splits are not shuffled): the largest
    sum(adj_lengths) over its batches of `batch_size` questions.  adj_lengths is the split's [Q, num_choice] (or [Q]) tensor.  A
    bound that held under any shuffle would be close to batch_size * num_choice * n and save nothing."""
    lens = torch.as_tensor(adj_lengths).to("cpu", torch.long)
    lens = lens.reshape(lens.size(0), -1).sum(1)
    return max((int(lens[a:a + batch_size].sum()) for a in range(0, lens.numel(), int(batch_size))), default=0)


def pack_adj(edge_index_nested, edge_type_nested, n_nodes, pin=True, edge_capacity=None, adj_lengths=None, node_capacity=None):
    """[batch][num_choice] nested lists (load_sparse_adj_data_with_contextnode format,
    utils/data_utils.py:189-190) -> PackedAdj, equal to LM_QAGNN.batch_graph's output.  With `edge_capacity` K the edges
    go into one pinned [3, K] buffer with a zero tail (ValueError if the batch has more than K edges).

    With the batch's `adj_lengths` the PackedAdj is RAGGED (see PackedAdj): node ids are offset by node_ptr[g] and the node
    arrays have `node_capacity` rows (default: the batch's node count; ValueError if the batch has more)."""
    flat_ei = [e for row in edge_index_nested for e in row] if isinstance(edge_index_nested[0], (list, tuple)) else list(edge_index_nested)
    flat_et = [e for row in edge_type_nested for e in row] if isinstance(edge_type_nested[0], (list, tuple)) else list(edge_type_nested)
    counts = torch.tensor([e.size(1) for e in flat_ei], dtype=torch.long)
    graph_ptr = torch.zeros(len(flat_ei) + 1, dtype=torch.long)
    graph_ptr[1:] = torch.cumsum(counts, 0)
    total = int(graph_ptr[-1])
    node_ptr, n_cap = None, -1
    offsets = torch.arange(len(flat_ei)) * n_nodes
    if adj_lengths is not None:
        node_ptr = node_ptr_of(adj_lengths, n_nodes, len(flat_ei))
        n_cap = _node_capacity(int(node_ptr[-1]), node_capacity)
        offsets = node_ptr[:-1]
    if edge_capacity is not None or node_ptr is not None:
        K = _capacity(total, edge_capacity)
        buf = torch.zeros(3, K, dtype=torch.long, pin_memory=pin and torch.cuda.is_available())
        if total:
            buf[:2, :total] = torch.cat(flat_ei, dim=1) + torch.repeat_interleave(offsets, counts)
            buf[2, :total] = torch.cat(flat_et, dim=0)
        return PackedAdj(buf[:2], buf[2], graph_ptr, n_nodes, buf, n_edges=total, edge_capacity=K, node_ptr=node_ptr,
                         node_capacity=n_cap)
    edge_index = torch.empty(2, total, dtype=torch.long, pin_memory=pin and torch.cuda.is_available())
    edge_type = torch.empty(total, dtype=torch.long, pin_memory=pin and torch.cuda.is_available())
    if total:
        torch.cat(flat_ei, dim=1, out=edge_index)
        torch.cat(flat_et, dim=0, out=edge_type)
        edge_index += torch.repeat_interleave(torch.arange(len(flat_ei)) * n_nodes, counts).unsqueeze(0)
    return PackedAdj(edge_index, edge_type, graph_ptr, n_nodes, n_edges=total, edge_capacity=total)


def load_sparse_adj_data_with_contextnode(adj_pk_path, max_node_num, num_choice, args=None, use_cache=True,
                                          write_cache=True):
    """Same contract as the reference loader (utils/data_utils.py:79-197): reads the `*.graph.adj.pk` list of
    {'adj': scipy COO (half_n_rel*n x n), 'concepts', 'qmask', 'amask', 'cid2score'} records (or the
    `.loaded_cache` pickle next to it, same 8-item layout) and returns

        concept_ids [Q, nc, n] int64, node_type_ids [Q, nc, n] int64, node_scores [Q, nc, n, 1] fp32,
        adj_lengths [Q, nc] int64, (edge_index, edge_type) nested lists [Q][nc] of int64 [2, E_g] / [E_g]

    with the context node at position 0 (concept id 0, type 3, cid2score key -1), concept ids shifted by +1, pad
    id 1 / type 2, relation ids shifted by +2 with context->question / context->answer edges as relations 0 / 1, edges
    to truncated nodes dropped and the inverse edges appended with `rel + half_n_rel`.  The per-record work is
    vectorised (no per-node Python loops), which is what makes the reference's loader take minutes on CSQA."""
    cache_path = adj_pk_path + ".loaded_cache"
    if use_cache and os.path.exists(cache_path):
        with open(cache_path, "rb") as f:
            (adj_lengths_ori, concept_ids, node_type_ids, node_scores, adj_lengths, edge_index, edge_type,
             half_n_rel) = pickle.load(f)
    else:
        with open(adj_pk_path, "rb") as fin:
            records = pickle.load(fin)
        n_samples = len(records)
        edge_index, edge_type = [], []
        adj_lengths = np.zeros(n_samples, dtype=np.int64)
        adj_lengths_ori = np.zeros(n_samples, dtype=np.int64)
        concept_ids = np.ones((n_samples, max_node_num), dtype=np.int64)
        node_type_ids = np.full((n_samples, max_node_num), 2, dtype=np.int64)
        node_scores = np.zeros((n_samples, max_node_num, 1), dtype=np.float32)
        half_n_rel = 0
        for idx, rec in enumerate(records):
            adj, concepts = rec["adj"], np.asarray(rec["concepts"])
            qm, am = np.asarray(rec["qmask"], dtype=bool), np.asarray(rec["amask"], dtype=bool)
            cid2score = rec["cid2score"]
            if len(concepts) != len(set(concepts.tolist())):
                raise ValueError(f"record {idx}: duplicate concepts")
            qam = qm | am
            if not qam[0] or np.any(np.diff(qam.astype(np.int8)) > 0):
                raise ValueError(f"record {idx}: question/answer concepts must form a prefix")
            num_concept = min(len(concepts), max_node_num - 1) + 1
            adj_lengths_ori[idx] = len(concepts)
            adj_lengths[idx] = num_concept
            kept = concepts[:num_concept - 1]
            concept_ids[idx, 0] = 0
            concept_ids[idx, 1:num_concept] = kept + 1
            if cid2score is not None:
                node_scores[idx, 0, 0] = cid2score[-1]
                node_scores[idx, 1:num_concept, 0] = [cid2score[int(c)] for c in kept]
            node_type_ids[idx, 0] = 3
            types = node_type_ids[idx, 1:num_concept]
            types[qm[:num_concept - 1]] = 0
            types[am[:num_concept - 1]] = 1
            n_node = adj.shape[1]
            half = adj.shape[0] // n_node
            rel = adj.row.astype(np.int64) // n_node + 2
            src = adj.row.astype(np.int64) % n_node + 1
            tgt = adj.col.astype(np.int64) + 1
            # context node -> question / answer concepts (relations 0 / 1); the reference's `> num_concept` bound
            limit = min(len(qm), num_concept)
            q_to = np.nonzero(qm[:limit])[0] + 1
            a_to = np.nonzero(am[:limit])[0] + 1
            rel = np.concatenate([rel, np.zeros(len(q_to), np.int64), np.ones(len(a_to), np.int64)])
            src = np.concatenate([src, np.zeros(len(q_to) + len(a_to), np.int64)])
            tgt = np.concatenate([tgt, q_to, a_to])
            half_n_rel = half + 2
            keep = (src < max_node_num) & (tgt < max_node_num)
            rel, src, tgt = rel[keep], src[keep], tgt[keep]
            edge_index.append(torch.from_numpy(np.stack([np.concatenate([src, tgt]), np.concatenate([tgt, src])])))
            edge_type.append(torch.from_numpy(np.concatenate([rel, rel + half_n_rel])))
        adj_lengths_ori = torch.from_numpy(adj_lengths_ori)
        adj_lengths = torch.from_numpy(adj_lengths)
        concept_ids = torch.from_numpy(concept_ids)
        node_type_ids = torch.from_numpy(node_type_ids)
        node_scores = torch.from_numpy(node_scores)
        if write_cache:
            with open(cache_path, "wb") as f:
                pickle.dump([adj_lengths_ori, concept_ids, node_type_ids, node_scores, adj_lengths, edge_index, edge_type,
                             half_n_rel], f)
    edge_index = [list(edge_index[i:i + num_choice]) for i in range(0, len(edge_index), num_choice)]
    edge_type = [list(edge_type[i:i + num_choice]) for i in range(0, len(edge_type), num_choice)]
    concept_ids, node_type_ids, node_scores, adj_lengths = [x.view(-1, num_choice, *x.size()[1:]) for x in
                                                            (concept_ids, node_type_ids, node_scores, adj_lengths)]
    return concept_ids, node_type_ids, node_scores, adj_lengths, (edge_index, edge_type)


def synth_adj_pickle(path, n_records, seed=0, n_rel=17, max_nodes=400):
    """Writes a synthetic `*.graph.adj.pk` in the reference's record schema (utils/graph.py:331-338): n_g ~
    clip(lognormal(ln 120, 0.6), 8, max_nodes) concepts, ~2.5*n_g forward edges over `n_rel` relations, 1-8 question
    and 1-3 answer concepts first, scores ~ N(0,1) incl. key -1 for the context node (SURVEY.md §8d cfg 3)."""
    from scipy.sparse import coo_matrix
    rng = np.random.default_rng(seed)
    records = []
    for _ in range(n_records):
        n = int(np.clip(rng.lognormal(np.log(120), 0.6), 8, max_nodes))
        concepts = rng.choice(700000, size=n, replace=False).astype(np.int64)
        nq = int(rng.integers(1, 9)); na = int(rng.integers(1, 4))
        nq = min(nq, n - 1); na = min(na, n - nq)
        qmask = np.zeros(n, dtype=bool); qmask[:nq] = True
        amask = np.zeros(n, dtype=bool); amask[nq:nq + na] = True
        ne = int(2.5 * n)
        r, s, t = rng.integers(0, n_rel, ne), rng.integers(0, n, ne), rng.integers(0, n, ne)
        key = np.unique(np.stack([r * n + s, t]), axis=1)
        adj = coo_matrix((np.ones(key.shape[1], dtype=bool), (key[0], key[1])), shape=(n_rel * n, n))
        cid2score = {int(c): float(v) for c, v in zip(concepts, rng.standard_normal(n))}
        cid2score[-1] = float(rng.standard_normal())
        records.append({"adj": adj, "concepts": concepts, "qmask": qmask, "amask": amask, "cid2score": cid2score})
    with open(path, "wb") as f:
        pickle.dump(records, f)
    return records


# ------------------------------------------------------------------------------------------------------------------
# Flat adjacency cache + pre-packed batch generator (SURVEY.md §8f #1 and #4)
# ------------------------------------------------------------------------------------------------------------------
class FlatAdjCache:
    """All sub-graphs of a split as three flat arrays + a row pointer (a CSR over graphs), instead of the reference's
    [n_samples][num_choice] nested lists of small tensors (utils/data_utils.py:174-190):

        src, tgt int32 [total_E] (LOCAL node ids), etype int16 [total_E], graph_ptr int64 [n_graphs + 1]

    Written once next to the reference's `.loaded_cache` as `<adj_pk_path>.flat_cache.npz` and memory-mapped afterwards;
    `pack(graph_ids)` cuts a batch out of it with three vectorised gathers into ONE pinned [3, E] int64 buffer."""

    def __init__(self, src, tgt, etype, graph_ptr, num_choice, n_nodes):
        self.src, self.tgt, self.etype, self.graph_ptr = src, tgt, etype, graph_ptr
        self.num_choice, self.n_nodes = int(num_choice), int(n_nodes)

    @classmethod
    def from_nested(cls, edge_index_nested, edge_type_nested, n_nodes):
        flat_ei = [e for row in edge_index_nested for e in row]
        flat_et = [e for row in edge_type_nested for e in row]
        counts = np.array([e.size(1) for e in flat_ei], dtype=np.int64)
        ptr = np.zeros(len(flat_ei) + 1, dtype=np.int64)
        ptr[1:] = np.cumsum(counts)
        if int(ptr[-1]):
            ei = torch.cat(flat_ei, dim=1).numpy()
            et = torch.cat(flat_et, dim=0).numpy()
        else:
            ei, et = np.zeros((2, 0), np.int64), np.zeros((0,), np.int64)
        return cls(ei[0].astype(np.int32), ei[1].astype(np.int32), _etype_int16(et, "FlatAdjCache"), ptr,
                   len(edge_index_nested[0]), n_nodes)

    def save(self, path):
        np.savez(path, src=self.src, tgt=self.tgt, etype=self.etype, graph_ptr=self.graph_ptr,
                 meta=np.array([self.num_choice, self.n_nodes], dtype=np.int64))

    @classmethod
    def load(cls, path):
        z = np.load(path, mmap_mode="r")
        meta = z["meta"]
        return cls(z["src"], z["tgt"], z["etype"], z["graph_ptr"], int(meta[0]), int(meta[1]))

    def n_graphs(self):
        return len(self.graph_ptr) - 1

    def n_questions(self):
        return self.n_graphs() // self.num_choice

    def max_graph_edges(self):
        """Edges of the largest sub-graph: a `max_edges` of the packed graph prep that holds for every batch of the split."""
        return int(np.diff(self.graph_ptr).max()) if self.n_graphs() else 0

    def max_batch_edges(self, batch_size):
        """Edges of the `batch_size * num_choice` largest sub-graphs together: an edge capacity that holds for every batch
        of `batch_size` questions, however the split is shuffled."""
        return largest_edges(np.diff(self.graph_ptr), int(batch_size) * self.num_choice)

    def __getitem__(self, i):
        """What LM_QAGNN_DataLoader does with `adj_data` besides handing it to the batch generator
        (modeling_qagnn.py:281-287,307-308): `len(adj_data[0])` must be the number of questions, and `adj_data[:n]` is taken
        when a split is subsampled.  An int gives a sized stand-in for the nested list, a slice the cache of those questions."""
        if isinstance(i, slice):
            a, b, step = i.indices(self.n_questions())
            if step != 1:
                raise IndexError("FlatAdjCache supports contiguous question ranges only")
            b = max(a, b)
            g0, g1 = a * self.num_choice, b * self.num_choice
            e0, e1 = int(self.graph_ptr[g0]), int(self.graph_ptr[g1])
            return FlatAdjCache(self.src[e0:e1], self.tgt[e0:e1], self.etype[e0:e1],
                                np.asarray(self.graph_ptr[g0:g1 + 1]) - e0, self.num_choice, self.n_nodes)
        if i in (0, 1, -1, -2):
            return range(self.n_questions())
        raise IndexError("FlatAdjCache stands in for the (edge_index, edge_type) pair: index 0 or 1")

    def pack(self, question_indexes, pin=True, edge_capacity=None, adj_lengths=None, node_capacity=None):
        """PackedAdj of the questions `question_indexes` (all their choices, in order) — equal to
        LM_QAGNN.batch_graph applied to the corresponding nested-list slice (modeling_qagnn.py:244-251).  With
        `edge_capacity` K the buffer is [3, K] with a zero tail (ValueError if the batch has more than K edges).  With the
        batch's `adj_lengths` ([bs, num_choice]) the PackedAdj is ragged at `node_capacity` rows, as in pack_adj."""
        q = np.asarray(question_indexes, dtype=np.int64).reshape(-1)
        gids = (q[:, None] * self.num_choice + np.arange(self.num_choice)[None, :]).reshape(-1)
        beg, end = self.graph_ptr[gids], self.graph_ptr[gids + 1]
        counts = end - beg
        ptr = np.zeros(len(gids) + 1, dtype=np.int64)
        ptr[1:] = np.cumsum(counts)
        total = int(ptr[-1])
        K = _capacity(total, edge_capacity)
        node_ptr, n_cap = None, -1
        if adj_lengths is not None:
            node_ptr = node_ptr_of(adj_lengths, self.n_nodes, len(gids))
            n_cap = _node_capacity(int(node_ptr[-1]), node_capacity)
        # flat positions of every edge of the batch: beg[g] + (0 .. counts[g]-1)
        pos = np.repeat(beg - ptr[:-1], counts) + np.arange(total, dtype=np.int64)
        first = node_ptr[:-1].numpy() if node_ptr is not None else np.arange(len(gids), dtype=np.int64) * self.n_nodes
        off = np.repeat(first, counts)
        buf = torch.empty(3, K, dtype=torch.long, pin_memory=pin and torch.cuda.is_available())
        b = buf.numpy()
        np.add(self.src[pos], off, out=b[0, :total], casting="unsafe")
        np.add(self.tgt[pos], off, out=b[1, :total], casting="unsafe")
        b[2, :total] = self.etype[pos]
        b[:, total:] = 0
        return PackedAdj(buf[:2], buf[2], torch.from_numpy(ptr), self.n_nodes, buf, n_edges=total, edge_capacity=K,
                         node_ptr=node_ptr, node_capacity=n_cap)


def load_flat_adj_cache(adj_pk_path, max_node_num, num_choice, args=None):
    """(concept_ids, node_type_ids, node_scores, adj_lengths, FlatAdjCache): the loader above with the adjacency as a flat
    cache; `<adj_pk_path>.flat_cache.npz` is written on first use and memory-mapped on later ones."""
    flat_path = adj_pk_path + ".flat_cache.npz"
    cids, ntypes, scores, lens, (ei, et) = load_sparse_adj_data_with_contextnode(adj_pk_path, max_node_num, num_choice, args)
    if os.path.exists(flat_path):
        flat = FlatAdjCache.load(flat_path)
        if flat.n_graphs() == cids.size(0) * num_choice and flat.n_nodes == max_node_num and flat.num_choice == num_choice:
            return cids, ntypes, scores, lens, flat
    flat = FlatAdjCache.from_nested(ei, et, max_node_num)
    flat.save(flat_path)
    return cids, ntypes, scores, lens, flat


class DeviceSplit:
    """A whole split on one GPU: the FlatAdjCache adjacency and the loader's decoder tensors, uploaded and validated once, so
    a batch's only per-call input is its question ids.  `batch(question_ids, K[, node_capacity=N_cap])` gives on the device
    what `flat.pack(question_ids, edge_capacity=K[, adj_lengths=..., node_capacity=N_cap]).to(device)` and the host-sliced
    node arrays give, bit for bit: the adjacency from qagnn_assemble_batch (include/qagnn_b200.h), the node rows from
    index_select.  Nothing reads the device: the batch checks and the PackedAdj's host fields come from host copies of the
    per-graph edge counts and adj_lengths.

    Held as: src / tgt int32 and etype int16 [E_split], graph_ptr int64 [G + 1], adj_lengths int64 [G], concept_ids and
    node_type_ids int64 [G, n], node_scores fp32 [G, n, 1], with G = Q * num_choice sub-graphs, and labels int64 [Q] when given.  At the loader's density
    (~584 edges per graph) a split of 50 k graphs takes about 0.3 GB of adjacency and 0.2 GB of node arrays."""

    def __init__(self, flat, concept_ids, node_type_ids, node_scores, adj_lengths, device, n_ntype, n_etype, *, labels=None):
        """What load_flat_adj_cache returns (concept_ids / node_type_ids [Q, nc, n], node_scores [Q, nc, n, 1], adj_lengths
        [Q, nc], flat a FlatAdjCache), uploaded to `device`.  Raises IndexError naming the first offending question when an
        edge's local ids leave [0, adj_length) of its graph, an etype leaves [0, n_etype), a node type leaves [0, n_ntype) or
        an adj_length leaves [1, n].

        `labels` (optional, integer [Q]: the loader's answer index per question, e.g. LM_QAGNN_DataLoader.train_labels) is
        uploaded as `self.labels` (int64) for pipeline.SplitTrainStep; a label outside [0, num_choice) raises IndexError naming
        its question, another shape or a non-integer dtype ValueError.  Without it `self.labels` is None."""
        self.device = torch.device(device)
        self.num_choice, self.n_nodes = flat.num_choice, flat.n_nodes
        nc, n = self.num_choice, self.n_nodes
        G = flat.n_graphs()
        self.n_questions = G // nc
        self.counts = np.diff(np.asarray(flat.graph_ptr, dtype=np.int64))  # host copies: every batch is checked from these
        self.lens = torch.as_tensor(adj_lengths).to("cpu", torch.long).reshape(-1)
        shapes = {"concept_ids": concept_ids.reshape(-1, n), "node_type_ids": node_type_ids.reshape(-1, n),
                  "node_scores": node_scores.reshape(-1, n, 1), "adj_lengths": self.lens}
        for name, t in shapes.items():
            if t.size(0) != G:
                raise ValueError(f"DeviceSplit: {name} has {t.size(0)} graphs, the adjacency {G}")
        if labels is not None:
            labels = torch.as_tensor(labels)
            if tuple(labels.shape) != (self.n_questions,) or labels.is_floating_point() or labels.is_complex() \
                    or labels.dtype == torch.bool:
                raise ValueError(f"DeviceSplit: labels must be integer [{self.n_questions}] (one per question), got "
                                 f"{tuple(labels.shape)} {labels.dtype}")
        dev = self.device
        self.src = torch.from_numpy(np.ascontiguousarray(flat.src, dtype=np.int32)).to(dev)
        self.tgt = torch.from_numpy(np.ascontiguousarray(flat.tgt, dtype=np.int32)).to(dev)
        if int(n_etype) > 1 << 15:  # the largest type, n_etype - 1, must fit the int16 edge types
            raise ValueError(f"DeviceSplit: n_etype = {int(n_etype)} does not fit the int16 edge types of the flat adjacency")
        self.etype = torch.from_numpy(_etype_int16(flat.etype, "DeviceSplit")).to(dev)
        self.graph_ptr = torch.from_numpy(np.ascontiguousarray(flat.graph_ptr, dtype=np.int64)).to(dev)
        self.adj_lengths = self.lens.to(dev)
        self.concept_ids = shapes["concept_ids"].to(dev, torch.long).contiguous()
        self.node_type_ids = shapes["node_type_ids"].to(dev, torch.long).contiguous()
        self.node_scores = shapes["node_scores"].to(dev, torch.float32).contiguous()
        self.labels = None if labels is None else labels.to(dev, torch.long).contiguous()
        self._validate(int(n_ntype), int(n_etype))

    def _validate(self, T, R):
        """The split's indices, checked once on the device (one synchronisation per check)."""
        nc, n, dev = self.num_choice, self.n_nodes, self.device
        G = self.lens.numel()
        edge_graph = torch.repeat_interleave(torch.arange(G, device=dev), torch.from_numpy(self.counts).to(dev))
        rows = self.adj_lengths[edge_graph]
        # int16 etype against R = 2^15 would cast R to int16 (-32768) and flag every edge; no int16 reaches 2^15 anyway
        etype_high = self.etype >= R if R < 1 << 15 else torch.zeros_like(self.etype, dtype=torch.bool)
        checks = (("an adj_length outside [1, %d]" % n, (self.adj_lengths < 1) | (self.adj_lengths > n), None),
                  ("an edge outside its graph's rows [0, adj_length)",
                   (self.src < 0) | (self.src >= rows) | (self.tgt < 0) | (self.tgt >= rows), edge_graph),
                  ("an edge type outside [0, %d)" % R, (self.etype < 0) | etype_high, edge_graph),
                  ("a node type outside [0, %d)" % T, ((self.node_type_ids < 0) | (self.node_type_ids >= T)).any(1), None))
        for what, bad, graph_of in checks:
            idx = torch.nonzero(bad)
            if idx.numel():
                g = int(idx[0, 0]) if graph_of is None else int(graph_of[idx[0, 0]])
                raise IndexError(f"DeviceSplit: question {g // nc} (graph {g}) has {what}")
        if self.labels is not None:  # the captured cross entropy must never see a target outside [0, nc)
            idx = torch.nonzero((self.labels < 0) | (self.labels >= nc))
            if idx.numel():
                q = int(idx[0, 0])
                raise IndexError(f"DeviceSplit: question {q} has label {int(self.labels[q])}, outside [0, {nc})")

    def max_batch_edges(self, batch_size):
        """FlatAdjCache.max_batch_edges of the split's adjacency: an edge capacity that holds for every batch of `batch_size`
        questions, however the split is shuffled."""
        return largest_edges(self.counts, int(batch_size) * self.num_choice)

    def check(self, question_ids, edge_capacity, node_capacity=None):
        """The host checks of one batch, O(bs * num_choice), with FlatAdjCache.pack's exceptions: IndexError for a question id
        outside [0, Q), ValueError for more than `edge_capacity` edges or (ragged) more than `node_capacity` rows.  Returns
        (question ids int64 [bs], graph_ptr [B + 1], node_ptr [B + 1] or None, K, N_cap or -1), all on the host."""
        q = np.asarray(question_ids, dtype=np.int64).reshape(-1)
        if q.size == 0:
            raise ValueError("DeviceSplit: an empty batch")
        lo, hi = int(q.min()), int(q.max())
        if lo < 0 or hi >= self.n_questions:
            raise IndexError(f"DeviceSplit: question id {lo if lo < 0 else hi} is outside [0, {self.n_questions})")
        gids = (q[:, None] * self.num_choice + np.arange(self.num_choice)[None, :]).reshape(-1)
        ptr = np.zeros(len(gids) + 1, dtype=np.int64)
        np.cumsum(self.counts[gids], out=ptr[1:])
        K = _capacity(int(ptr[-1]), edge_capacity)
        node_ptr, n_cap = None, -1
        if node_capacity is not None:
            node_ptr = node_ptr_of(self.lens[torch.from_numpy(gids)], self.n_nodes, len(gids))
            n_cap = _node_capacity(int(node_ptr[-1]), node_capacity)
        return q, torch.from_numpy(ptr), node_ptr, K, n_cap

    def buffers(self, batch_size, edge_capacity, node_capacity=None):
        """Device buffers for batches of `batch_size` questions at edge capacity K (and node capacity N_cap): the `out` of
        assemble() / batch(), which a captured step fills in every replay."""
        B, n, dev = int(batch_size) * self.num_choice, self.n_nodes, self.device
        out = {"concept_ids": torch.empty(B, n, dtype=torch.long, device=dev),
               "node_type_ids": torch.empty(B, n, dtype=torch.long, device=dev),
               "node_scores": torch.empty(B, n, 1, dtype=torch.float32, device=dev),
               "adj_lengths": torch.empty(B, dtype=torch.long, device=dev),
               "edges": torch.empty(3, int(edge_capacity), dtype=torch.long, device=dev),
               "graph_ptr": torch.empty(B + 1, dtype=torch.long, device=dev)}
        if node_capacity is not None:
            out["node_ptr"] = torch.empty(B + 1, dtype=torch.long, device=dev)
        return out

    def assemble(self, qids, edge_capacity, node_capacity=-1, out=None):
        """The device half of batch(): enqueues the batch of the question ids `qids` (device int64 [bs], already checked)
        without a host synchronisation.  Returns `out` (buffers()) filled; N_cap = -1 assembles a padded batch."""
        from . import _lib
        bs, K, N_cap = qids.numel(), int(edge_capacity), int(node_capacity)
        if out is None:
            out = self.buffers(bs, K, None if N_cap < 0 else N_cap)
        dev = self.device
        lib = _lib.load()
        with torch.cuda.device(dev):
            st = lib.qagnn_assemble_batch(_lib.ptr(self.src), _lib.ptr(self.tgt), _lib.ptr(self.etype), _lib.ptr(self.graph_ptr),
                                          _lib.ptr(self.adj_lengths), self.lens.numel(), self.num_choice, self.n_nodes,
                                          _lib.ptr(qids), bs, K, N_cap, _lib.ptr(out["edges"]), _lib.ptr(out["graph_ptr"]),
                                          _lib.ptr(out.get("node_ptr")) if N_cap >= 0 else None, _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_assemble_batch")
        # the rows of every choice of every question; ids are clamped as the kernel clamps them, so nothing reads out of range
        gids = (qids.clamp(0, self.n_questions - 1).unsqueeze(1) * self.num_choice
                + torch.arange(self.num_choice, device=dev).unsqueeze(0)).reshape(-1)
        torch.index_select(self.concept_ids, 0, gids, out=out["concept_ids"])
        torch.index_select(self.node_type_ids, 0, gids, out=out["node_type_ids"])
        torch.index_select(self.node_scores, 0, gids, out=out["node_scores"])
        torch.index_select(self.adj_lengths, 0, gids, out=out["adj_lengths"])
        return out

    def packed_adj(self, out, max_edges, edge_capacity, node_capacity=-1, graph_ptr=None, n_edges=-1, node_ptr=None):
        """The PackedAdj over the buffers `out` (views, no copy); the host fields are the caller's (None / -1 when unknown)."""
        e = out["edges"]
        ragged = int(node_capacity) >= 0
        return PackedAdj(edge_index=e[:2], edge_type=e[2], graph_ptr=graph_ptr, n_nodes=self.n_nodes, buf=e,
                         graph_ptr_dev=out["graph_ptr"], max_edges=int(max_edges), n_edges=int(n_edges),
                         edge_capacity=int(edge_capacity), node_ptr=node_ptr,
                         node_ptr_dev=out["node_ptr"] if ragged else None, node_capacity=int(node_capacity))

    def batch(self, question_ids, edge_capacity, node_capacity=None, out=None):
        """(concept_ids [B, n], node_type_ids [B, n], node_scores [B, n, 1], adj_lengths [B], PackedAdj) on the device for the
        questions `question_ids` (host ids, all their choices in order, B = bs * num_choice): the PackedAdj equals
        `flat.pack(question_ids, edge_capacity=K, ...).to(device)` (ragged at `node_capacity` N_cap when given), with
        graph_ptr_dev, node_ptr_dev, the batch's max_edges and both capacities set.  Checked on the host first (check()), so a
        bad batch raises before anything is enqueued.  `out` (buffers()) names static buffers to fill."""
        q, ptr, node_ptr, K, n_cap = self.check(question_ids, edge_capacity, node_capacity)
        if out is not None and out["edges"].size(1) != K:
            raise ValueError(f"DeviceSplit: the buffers hold {out['edges'].size(1)} edge columns, the batch needs {K}")
        qh = torch.from_numpy(q)
        qd = (qh.pin_memory() if self.device.type == "cuda" else qh).to(self.device, non_blocking=True)
        out = self.assemble(qd, K, n_cap, out)
        me = int((ptr[1:] - ptr[:-1]).max()) if ptr.numel() > 1 else 0
        adj = self.packed_adj(out, me, K, n_cap, ptr, int(ptr[-1]), node_ptr)
        return out["concept_ids"], out["node_type_ids"], out["node_scores"], out["adj_lengths"], adj


class PackedAdjBatchGenerator:
    """Drop-in for the reference's MultiGPUSparseAdjDataBatchGenerator (utils/data_utils.py:17-76): same constructor, same
    batch tuple  (qids, labels, *tensors0, *lists0, *tensors1, *lists1, edge_index, edge_type),  same partial-batch
    options — but `adj_data` may be a FlatAdjCache, in which case the adjacency of a batch is packed on the host into one
    pinned buffer and moved with ONE non-blocking copy; the `edge_index` slot then holds a PackedAdj (which
    LM_QAGNN.forward accepts) and the `edge_type` slot its edge_type view.  Tensors are staged through pinned memory as
    well, so every copy of a batch is asynchronous.  With nested-list `adj_data` it behaves exactly like the reference."""

    def __init__(self, args, mode, device0, device1, batch_size, indexes, qids, labels, tensors0=[], lists0=[], tensors1=[],
                 lists1=[], adj_data=None, prefetch=0, edge_capacity=None):
        """`prefetch` > 0 (not in the reference): a worker thread slices / packs / pins up to that many batches ahead on the
        host while the consumer trains on the current one; the device copies are still issued by the consuming thread (on
        ITS current stream), in order, so the batches and their order are exactly those of prefetch=0.

        `edge_capacity` K (not in the reference; needs a FlatAdjCache): every batch's adjacency is packed into a [3, K]
        buffer (see PackedAdj), so all full batches have the same shapes and can be written into the buffers of one captured
        step.  `adj_data.max_batch_edges(batch_size)` is a K that holds for every batch of the split."""
        if edge_capacity is not None and not isinstance(adj_data, FlatAdjCache):
            raise ValueError("edge_capacity needs adj_data to be a FlatAdjCache")
        self.args, self.mode = args, mode
        self.device0, self.device1 = device0, device1
        self.batch_size, self.indexes, self.qids, self.labels = batch_size, indexes, qids, labels
        self.tensors0, self.lists0, self.tensors1, self.lists1 = tensors0, lists0, tensors1, lists1
        self.adj_data = adj_data
        self.prefetch = int(prefetch)
        self.edge_capacity = edge_capacity

    def __len__(self):
        return (self.indexes.size(0) - 1) // self.batch_size + 1

    @staticmethod
    def _pin(obj, device):
        """Host side of a copy: page-locks a tensor bound for a CUDA device (nested lists element-wise)."""
        if isinstance(obj, (tuple, list)):
            return [PackedAdjBatchGenerator._pin(item, device) for item in obj]
        if isinstance(obj, PackedAdj):
            return obj  # FlatAdjCache.pack already wrote it into pinned memory
        if torch.cuda.is_available() and torch.device(device).type == "cuda" and not obj.is_pinned():
            return obj.pin_memory()
        return obj

    def _to_device(self, obj, device):
        if isinstance(obj, (tuple, list)):
            return [self._to_device(item, device) for item in obj]
        if isinstance(obj, PackedAdj):
            return obj.to(device, non_blocking=True)
        return self._pin(obj, device).to(device, non_blocking=True)

    def _host_batch(self, batch_indexes):
        """Everything of one batch that needs no device: slicing, adjacency packing, pinning."""
        d0, d1 = self.device0, self.device1
        qids = [self.qids[idx] for idx in batch_indexes]
        labels = self._pin(self.labels[batch_indexes], d1)
        tensors0 = [self._pin(x[batch_indexes], d0) for x in self.tensors0]
        tensors1 = [self._pin(x[batch_indexes], d1) for x in self.tensors1]
        lists0 = [self._pin([x[i] for i in batch_indexes], d0) for x in self.lists0]
        lists1 = [self._pin([x[i] for i in batch_indexes], d1) for x in self.lists1]
        if isinstance(self.adj_data, FlatAdjCache):
            adj = self.adj_data.pack(batch_indexes.numpy(), edge_capacity=self.edge_capacity)
        else:
            edge_index_all, edge_type_all = self.adj_data
            adj = (self._pin([edge_index_all[i] for i in batch_indexes], d1),
                   self._pin([edge_type_all[i] for i in batch_indexes], d1))
        return qids, labels, tensors0, lists0, tensors1, lists1, adj

    def _ship(self, host):
        qids, labels, tensors0, lists0, tensors1, lists1, adj = host
        d0, d1 = self.device0, self.device1
        if isinstance(adj, PackedAdj):
            packed = self._to_device(adj, d1)
            edge_index, edge_type = packed, packed.edge_type
        else:
            edge_index, edge_type = self._to_device(adj[0], d1), self._to_device(adj[1], d1)
        return tuple([qids, self._to_device(labels, d1), *[self._to_device(x, d0) for x in tensors0],
                      *[self._to_device(x, d0) for x in lists0], *[self._to_device(x, d1) for x in tensors1],
                      *[self._to_device(x, d1) for x in lists1], edge_index, edge_type])

    def _batch_ranges(self):
        bs = self.batch_size
        n = self.indexes.size(0)
        if self.mode == "train" and getattr(self.args, "drop_partial_batch", False):
            n = (n // bs) * bs
        elif self.mode == "train" and getattr(self.args, "fill_partial_batch", False):
            remain = n % bs
            if remain > 0:
                extra = np.random.choice(self.indexes[:-remain], size=(bs - remain), replace=False)
                self.indexes = torch.cat([self.indexes, torch.tensor(extra)])
                n = self.indexes.size(0)
        return [self.indexes[a:min(n, a + bs)] for a in range(0, n, bs)]

    def __iter__(self):
        batches = self._batch_ranges()
        if self.prefetch <= 0:
            for batch_indexes in batches:
                yield self._ship(self._host_batch(batch_indexes))
            return
        import queue
        import threading
        q = queue.Queue(maxsize=self.prefetch)
        stop = threading.Event()

        def put(item):  # a consumer that stops iterating early must not leave the worker blocked on a full queue
            while not stop.is_set():
                try:
                    q.put(item, timeout=0.1)
                    return True
                except queue.Full:
                    pass
            return False

        def work():
            try:
                for batch_indexes in batches:
                    if not put(("batch", self._host_batch(batch_indexes))):
                        return
                put(("end", None))
            except BaseException as e:  # surfaces in the consuming thread
                put(("error", e))

        t = threading.Thread(target=work, name="qagnn-batch-prefetch", daemon=True)
        t.start()
        try:
            while True:
                kind, item = q.get()
                if kind == "end":
                    break
                if kind == "error":
                    raise item
                yield self._ship(item)
        finally:
            stop.set()
            t.join()
