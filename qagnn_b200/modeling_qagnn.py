"""Drop-in modules for the reference's modeling/modeling_qagnn.py hot path.

Same class names, constructor arguments, forward signatures, return values and state_dict key
names as the reference (SURVEY.md §8b), but `GATConvE.forward` and
`QAGNN_Message_Passing.forward` run entirely in the hand-written sm_90a kernels of
libqagnn_b200.so, reached through the C ABI in include/qagnn_b200.h.  The nn.Modules below only
own parameters and device buffers (PyTorch = memory + streams).

    GATConvE                 <- modeling/modeling_qagnn.py:380-484
    QAGNN_Message_Passing    <- modeling/modeling_qagnn.py:7-95
    QAGNN                    <- modeling/modeling_qagnn.py:99-189   (caller side, plain PyTorch)
    LM_QAGNN                 <- modeling/modeling_qagnn.py:192-251  (caller side, plain PyTorch)

Modes: `.eval()` = the fused inference forward (dropout = identity, BatchNorm running statistics folded into the
weights) — the reference's `evaluate_accuracy` path (qagnn.py:30-38); `.train()` = dropout, BatchNorm batch statistics
and autograd through the CUDA message-passing forward / backward kernels (qagnn_b200/training.py; qagnn.py:249-278).
An `.eval()` call whose inputs require grad (under grad mode) takes that autograd path with eval semantics instead, so
`backward()` reaches every parameter as in the reference.  CPU tensors raise: there is no CPU fallback.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from . import training as TR
from .layers import GELU, MLP, CustomizedEmbedding, MultiheadAttPoolLayer

# head counts GATConvE accepts: every message-passing path (tiled, column-sliced, basic CSR, training backward) runs them
SUPPORTED_HEAD_COUNTS = (1, 2, 4, 8, 16)

def make_one_hot(labels, C_):
    """int64 [M] -> float32 one-hot [M, C] on labels.device (modeling_qagnn.py:352-367)."""
    out = torch.zeros(labels.size(0), C_, dtype=torch.float32, device=labels.device)
    return out.scatter_(1, labels.unsqueeze(1), 1.0)


def _version_key(tensors):
    return tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in tensors)


def _wants_autograd(module, *tensors):
    """The differentiable path (qagnn_b200/training.py) runs in .train(), and in .eval() when grad mode is on and an input
    requires grad (the rule MultiheadAttPoolLayer.forward applies); every other eval call runs the fused kernels, which
    are outside autograd."""
    return module.training or (torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors))


class _DeviceBlob:
    """A grow-only uint8 device buffer (workspace the C ABI asks the caller to own).  `on_replace` runs before the
    buffer is dropped for a larger one: captured CUDA graphs hold its raw address and must be discarded first."""

    def __init__(self, on_replace=None):
        self.buf = None
        self.on_replace = on_replace

    def get(self, nbytes, device):
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            if self.buf is not None and self.on_replace is not None:
                self.on_replace()
            self.buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
        return self.buf


CROSS_GRAPH = 8  # graph prep status bit: an edge crosses a sub-graph boundary
NODE_PTR = 32    # graph prep status bit: a ragged batch's node_ptr is not monotone, has a graph over n rows or ends past N


class GraphPrepIndexError(IndexError):
    """Indices a validating graph prep found out of range.  `bits` is its status word: 1 edge_index, 2 edge_type,
    4 node_type, CROSS_GRAPH, 16 graph_ptr disagreeing with the edges or with max_edges, NODE_PTR."""

    def __init__(self, bits):
        super().__init__(f"qagnn_graph_prep: index out of range (status bits {bits})")
        self.bits = bits


class GraphPrep:
    """Owns the opaque graph-prep workspace of one batched graph (qagnn_graph_prep)."""

    def __init__(self, edge_index, edge_type, node_type, n_ntype, n_etype, n_per_graph=0, validate=True, graph_ptr=None,
                 max_edges=-1, node_ptr=None):
        """graph_ptr (device int64 [n_graphs + 1]) + max_edges (host int): the batch is PACKED graph by graph — the whole
        prep is then one kernel launch (qagnn_graph_prep_packed) instead of twelve.  edge_index may then be an edge
        capacity wider than the batch: the real count graph_ptr[-1] is read on the device.  That prep raises QagnnError
        with status -5 when it refuses the shape (sub-graphs too large for one CTA).  Without graph_ptr every column of
        edge_index is an edge.  A validating prep raises GraphPrepIndexError.  graph_prep() picks which prep a batch gets.

        node_ptr (device int64 [n_graphs + 1], with graph_ptr): a RAGGED batch (qagnn_graph_prep_ragged): graph g owns the rows
        [node_ptr[g], node_ptr[g+1]) of the node_type.numel() rows and n_per_graph bounds its rows."""
        lib = _lib.load()
        ei = _lib.i64c(edge_index, "edge_index")
        et = _lib.i64c(edge_type, "edge_type")
        nt = _lib.i64c(node_type.reshape(-1), "node_type")
        if ei.dim() != 2 or ei.size(0) != 2 or et.dim() != 1 or et.numel() != ei.size(1):
            raise ValueError("edge_index must be [2,E] and edge_type [E]")
        self.N, self.E = nt.numel(), ei.size(1)
        self.T, self.R, self.n_per_graph = n_ntype, n_etype, int(n_per_graph)
        self.device = nt.device
        self.layout = _lib.PrepLayout()
        _lib.check(lib.qagnn_graph_prep_layout(self.N, self.E, C.byref(self.layout)), "qagnn_graph_prep_layout")
        self.buf = torch.empty(self.layout.total_bytes, dtype=torch.uint8, device=self.device)
        self._combo = None
        # built by qagnn_graph_prep_packed: the edge columns past graph_ptr[-1] are unused
        self.packed = graph_ptr is not None and max_edges >= 0 and self.n_per_graph > 0
        self.node_ptr = node_ptr if self.packed else None
        self.n_graphs = 0
        shape = _lib.Shape(self.N, self.E, 4, 1, n_ntype, n_etype, 0, self.n_per_graph)
        eptr, tptr = (_lib.ptr(ei), _lib.ptr(et)) if self.E else (None, None)
        with torch.cuda.device(self.device):
            if self.node_ptr is not None:
                gp, npt = _lib.i64c(graph_ptr, "graph_ptr"), _lib.i64c(node_ptr, "node_ptr")
                if gp.numel() != npt.numel() or gp.numel() < 2:
                    raise ValueError("graph_ptr and node_ptr must both have one entry per graph plus one")
                self.n_graphs = gp.numel() - 1
                st = lib.qagnn_graph_prep_ragged(eptr, tptr, _lib.ptr(nt), _lib.ptr(gp), _lib.ptr(npt), self.n_graphs,
                                                 int(max_edges), C.byref(shape), _lib.ptr(self.buf), self.buf.numel(),
                                                 int(bool(validate)), _lib.stream_ptr(self.device))
            elif self.packed:
                gp = _lib.i64c(graph_ptr, "graph_ptr")
                if gp.numel() != self.N // self.n_per_graph + 1:
                    raise ValueError("graph_ptr must have one entry per sub-graph plus one")
                st = lib.qagnn_graph_prep_packed(eptr, tptr, _lib.ptr(nt), _lib.ptr(gp), int(max_edges), C.byref(shape),
                                                 _lib.ptr(self.buf), self.buf.numel(), int(bool(validate)),
                                                 _lib.stream_ptr(self.device))
            else:
                st = lib.qagnn_graph_prep(eptr, tptr, _lib.ptr(nt), C.byref(shape), _lib.ptr(self.buf), self.buf.numel(),
                                          int(bool(validate)), _lib.stream_ptr(self.device))
        if st == -3:  # the validating prep has synchronised: its status word says which check failed
            raise GraphPrepIndexError(int(self.status_word().item()))
        _lib.check(st, "qagnn_graph_prep_ragged" if self.node_ptr is not None else
                   "qagnn_graph_prep_packed" if self.packed else "qagnn_graph_prep")
        self._keep = (ei, et, nt, graph_ptr, node_ptr)

    def real_edges(self):
        """Edges of the batch (self loops excluded).  Below E only for a packed prep on an edge capacity; read from the
        device then (synchronising), because graph_ptr lives there."""
        if not self.packed:
            return self.E
        return int(self.array("rowptr_src")[self.N].item()) - self.N

    def compact_edges(self, t):
        """Rows of an [E+N, ...] edge-id-ordered array without the unused ids [real_edges(), E) of an edge capacity: the
        [E'+N, ...] array the same batch packed without spare columns gives."""
        e = self.real_edges()
        return t if e == self.E else torch.cat([t[:e], t[self.E:]])

    def combo_sort(self):
        """(combo_count int64 [C], combo_order int32 [E+N]) from qagnn_combo_sort, computed once per prep and without a host
        synchronisation: E' = rowptr_src[N] is read on the device, and only the first E' entries of combo_order are
        written.  This is what the training forward and backward use."""
        if self._combo is None:
            lib = _lib.load()
            shape = _lib.Shape(self.N, self.E, 4, 1, self.T, self.R, 0, self.n_per_graph)
            nbytes = lib.qagnn_combo_sort_bytes(C.byref(shape))
            if nbytes == 0:
                raise _lib.QagnnError(f"qagnn_combo_sort_bytes: unsupported shape (T={self.T}, R={self.R})")
            count = torch.empty(self.R * self.T * self.T + self.T, dtype=torch.int64, device=self.device)
            order = torch.empty(self.N + self.E, dtype=torch.int32, device=self.device)
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            with torch.cuda.device(self.device):
                st = lib.qagnn_combo_sort(C.byref(shape), _lib.ptr(self.buf), _lib.ptr(count), _lib.ptr(order), _lib.ptr(scratch),
                                          nbytes, _lib.stream_ptr(self.device))
            _lib.check(st, "qagnn_combo_sort")
            self._combo = (count, order)
        return self._combo

    def combo_order(self):
        """int32 [E']: by-source edge positions stably sorted by combo (for the backward's edge-table gradient).  Cutting it
        to E' reads E' from the device for a packed prep (see real_edges); combo_sort() gives the uncut array without that."""
        return self.combo_sort()[1][:self.real_edges() + self.N]

    def combo_count(self):
        """int64 [C]: number of edges (self loops included) per combo index."""
        return self.combo_sort()[0]

    def status_word(self):
        """Device-side error bits of the last qagnn_graph_prep on this buffer (0 = all indices in range)."""
        return self.array("status")[0:1]

    def array(self, name):
        """int32 view of one prep array (tests / inspection)."""
        Ep = self.N + self.E
        n = {"rowptr_src": self.N + 1, "rowptr_tgt": self.N + 1, "status": 4}.get(name, Ep)
        off = getattr(self.layout, name)
        return self.buf[off:off + 4 * n].view(torch.int32)

    def edge_index_prime(self):
        """edge_index' = [edge_index | self loops] as int64 [2, E+N] (modeling_qagnn.py:436-438); E = real_edges()."""
        ei = torch.stack([self.array("src"), self.array("tgt")]).long()
        e = self.real_edges()
        return ei if e == self.E else torch.cat([ei[:, :e], ei[:, self.E:]], 1)


def graph_prep(A, node_type, n, n_ntype, n_etype, validate):
    """The GraphPrep of batch A, an (edge_index, edge_type) pair or a qagnn_b200.data.PackedAdj, with `n` nodes per
    sub-graph as a layout hint (0: none).  Every prep the modules build is chosen here:
      * a PackedAdj packed for n-node sub-graphs gets the one-launch packed prep;
      * when that prep refuses the shape, or the PackedAdj was packed for another node count, the general prep runs on
        the batch's real edge columns (graph_ptr[-1] of them, read on the host when A.n_edges is unknown);
      * an edge that crosses a sub-graph boundary (validate only) is legal, as in the reference: n is then dropped and
        the batch goes to the general CSR kernels."""
    ei, et, nt = A[0], A[1], node_type.reshape(-1)
    gp = getattr(A, "graph_ptr_dev", None)
    if getattr(A, "ragged", False):
        # a ragged batch has no padded layout to fall back to: an edge outside its graph's rows is an error
        if A.node_ptr_dev is None or gp is None or A.max_edges < 0:
            raise ValueError("a ragged PackedAdj must be on the device (PackedAdj.to) with graph_ptr and max_edges")
        try:
            return GraphPrep(ei, et, nt, n_ntype, n_etype, A.n_nodes, validate, graph_ptr=gp, max_edges=A.max_edges,
                             node_ptr=A.node_ptr_dev)
        except _lib.QagnnError as e:
            if e.status == -5:  # QAGNN_ERR_UNSUPPORTED
                combos = n_etype * n_ntype * n_ntype + n_ntype
                why = (f"{combos} edge-feature combos (n_etype * n_ntype^2 + n_ntype) exceed the 65536 that the one-CTA "
                       "graph prep's 16-bit combo ids hold" if combos > 65536 else
                       f"graphs of {A.n_nodes} nodes and {A.max_edges} edges do not fit the one-CTA graph prep")
                raise ValueError(f"ragged batch: {why}; run this batch padded") from e
            raise
    if gp is not None:
        if n > 0 and A.n_nodes == n and A.max_edges >= 0:
            try:
                return GraphPrep(ei, et, nt, n_ntype, n_etype, n, validate, graph_ptr=gp, max_edges=A.max_edges)
            except GraphPrepIndexError as e:
                if e.bits != CROSS_GRAPH:
                    raise
                n = 0
            except _lib.QagnnError as e:
                if e.status != -5:  # QAGNN_ERR_UNSUPPORTED
                    raise
        ne = A.n_edges if A.n_edges >= 0 else int(gp[-1])
        if not 0 <= ne <= ei.size(1):
            raise IndexError(f"graph_ptr[-1] = {ne} is outside the {ei.size(1)} columns of edge_index")
        ei, et = ei[:, :ne], et[:ne]
    try:
        return GraphPrep(ei, et, nt, n_ntype, n_etype, n, validate)
    except GraphPrepIndexError as e:
        if n == 0 or e.bits != CROSS_GRAPH:
            raise
    return GraphPrep(ei, et, nt, n_ntype, n_etype, 0, validate)


def _refuse_ragged_training(module, what):
    """A ragged batch runs in .eval() only, with or without gradients: the reference's training BatchNorm statistics include
    the padded rows, which a ragged batch does not have.  In eval a padding row is inert, so nothing else differs."""
    if module.training:
        raise ValueError(f"{what}: a ragged batch runs in .eval() only (gradients included); training keeps the padded "
                         "layout because BatchNorm batch statistics include the padded rows")


def _edge_encoder_params(enc):
    lin0, bn, lin3 = enc[0], enc[1], enc[3]
    ts = [lin0.weight, lin0.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var, lin3.weight, lin3.bias]
    return ts


def _layer_params(layer):
    bn = layer.mlp[1]
    return [layer.linear_key.weight, layer.linear_key.bias, layer.linear_msg.weight, layer.linear_msg.bias,
            layer.linear_query.weight, layer.linear_query.bias, layer.mlp[0].weight, layer.mlp[0].bias,
            bn.weight, bn.bias, bn.running_mean, bn.running_var, layer.mlp[3].weight, layer.mlp[3].bias]


class _FoldedWeights:
    """Folded-parameter blob (qagnn_fold_weights), refreshed whenever a source tensor changes."""

    def __init__(self):
        self.key = None
        self.blob = None
        self._keep = None

    def invalidate(self):
        """Forget the folded blob.  Needed after parameter edits that bypass autograd's version counter
        (`p.data.normal_()`, `bn.running_mean.data.fill_()`): the cache key is (data_ptr, _version, shape)."""
        self.key = None

    def get(self, shape, enc, layers, mp_tensors, device):
        lib = _lib.load()
        srcs = _edge_encoder_params(enc)
        for l in layers:
            srcs += _layer_params(l)
        if mp_tensors is not None:
            srcs += mp_tensors
        key = (_version_key(srcs), shape.D, shape.H, shape.T, shape.R, shape.k, str(device))
        if key == self.key:
            return self.blob
        cont = [_lib.f32c(t, "parameter") for t in srcs]
        it = iter(cont)
        ee = _lib.EdgeEncoderParams(*[t.data_ptr() for t in [next(it) for _ in range(8)]])
        larr = (_lib.LayerParams * max(len(layers), 1))()
        for i in range(len(layers)):
            larr[i] = _lib.LayerParams(*[t.data_ptr() for t in [next(it) for _ in range(14)]])
        mp = None
        if mp_tensors is not None:
            mp = _lib.MPParams(*[t.data_ptr() for t in [next(it) for _ in range(9)]])
        nbytes = lib.qagnn_fold_bytes(C.byref(shape))
        if nbytes == 0:
            raise _lib.QagnnError("qagnn_fold_bytes: invalid shape")
        blob = torch.empty(nbytes, dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            st = lib.qagnn_fold_weights(C.byref(shape), C.byref(ee), larr, C.byref(mp) if mp is not None else None,
                                        _lib.ptr(blob), nbytes, _lib.stream_ptr(device))
        _lib.check(st, "qagnn_fold_weights")
        self.key, self.blob, self._keep = key, blob, cont
        return blob


class GATConvE(nn.Module):
    """
    Args:
        emb_dim (int): dimensionality of GNN hidden states
        n_ntype (int): number of node types (e.g. 4)
        n_etype (int): number of edge relation types (e.g. 38)
    Same constructor as the reference (modeling_qagnn.py:387): `edge_encoder` is the shared
    Sequential(Linear, BatchNorm1d, ReLU, Linear); `head_count` defaults to 4.
    """

    def __init__(self, args, emb_dim, n_ntype, n_etype, edge_encoder, head_count=4, aggr="add"):
        super().__init__()
        if aggr != "add":
            raise ValueError("GATConvE only supports aggr='add' (the only mode the reference uses)")
        if head_count not in SUPPORTED_HEAD_COUNTS:
            # the general-graph and training kernels are instantiated per head count; the tiled kernel alone would take
            # any, so another value would work or fail depending on the batch layout
            raise ValueError(f"head_count must be one of {SUPPORTED_HEAD_COUNTS} (got {head_count})")
        if emb_dim % 2 != 0 or emb_dim % head_count != 0:
            raise ValueError("emb_dim must be even and divisible by head_count")
        self.args = args
        self.emb_dim = emb_dim
        self.n_ntype, self.n_etype = n_ntype, n_etype
        self.edge_encoder = edge_encoder
        self.head_count = head_count
        self.dim_per_head = emb_dim // head_count
        self.linear_key = nn.Linear(3 * emb_dim, head_count * self.dim_per_head)
        self.linear_msg = nn.Linear(3 * emb_dim, head_count * self.dim_per_head)
        self.linear_query = nn.Linear(2 * emb_dim, head_count * self.dim_per_head)
        self._alpha = None
        self.mlp = nn.Sequential(nn.Linear(emb_dim, emb_dim), nn.BatchNorm1d(emb_dim), nn.ReLU(),
                                 nn.Linear(emb_dim, emb_dim))
        self.check_indices = True
        self._folded = _FoldedWeights()
        self._ws = _DeviceBlob()
        self._prep_cache = (None, None)

    def _prep(self, edge_index, edge_type, node_type):
        gp = getattr(edge_index, "graph_ptr_dev", None)
        if gp is not None:  # a qagnn_b200.data.PackedAdj: one-launch packed prep
            A, n, srcs = edge_index, edge_index.n_nodes, [edge_index.edge_index, edge_index.edge_type, node_type, gp]
            if edge_index.ragged:
                srcs.append(edge_index.node_ptr_dev)
        else:
            A, n, srcs = (edge_index, edge_type), 0, [edge_index, edge_type, node_type]
        key = _version_key(srcs)
        if self._prep_cache[0] != key:
            self._prep_cache = (key, graph_prep(A, node_type, n, self.n_ntype, self.n_etype, self.check_indices))
        return self._prep_cache[1]

    def forward(self, x, edge_index, edge_type, node_type, node_feature_extra, return_attention_weights=False,
                prep=None, return_aggr=False):
        """x [N, emb_dim]; edge_index [2, E]; edge_type [E]; node_type [N]; node_feature_extra [N, emb_dim].
        Returns out [N, emb_dim], or (out, (edge_index' [2,E+N], alpha [E+N, heads])) with
        return_attention_weights=True (alpha = softmax before the out-degree rescale, :473).  edge_index may be a
        qagnn_b200.data.PackedAdj (edge_type is then ignored), also one packed at an edge capacity: E is then its real
        edge count.  A ragged PackedAdj (eval only) takes x / node_feature_extra [N_cap, emb_dim] and node_type [N_cap].
        In .train(), or in .eval() with inputs that require grad, the output is differentiable (qagnn_b200/training.py)."""
        if getattr(edge_index, "ragged", False):
            _refuse_ragged_training(self, "GATConvE")
        if _wants_autograd(self, x, node_feature_extra):  # autograd through the CUDA message passing, this module's mode
            if prep is None:
                prep = self._prep(edge_index, edge_type, node_type)
            tab = TR.edge_table(self.edge_encoder, TR.combo_onehot_table(self.n_ntype, self.n_etype, x.device), prep, 1)
            return TR.gatconve_autograd(self, x, node_feature_extra, node_type, prep, tab, return_attention_weights)
        lib = _lib.load()
        # under bf16 autocast: bf16 in and out, single-pass bf16 GEMMs (include/qagnn_b200.h, qagnn_gatconve_forward_typed)
        xc, dt = _lib.eval_dtype(x, "x")
        ex, _ = _lib.eval_dtype(node_feature_extra, "node_feature_extra")
        if ex.dtype != xc.dtype:  # the library takes both inputs in one dtype: bf16 here (dt is bf16 when they can differ)
            xc, ex = xc.to(dt), ex.to(dt)
        dev = xc.device
        N, D = xc.shape
        if D != self.emb_dim or ex.shape != xc.shape:
            raise ValueError("x / node_feature_extra must be [N, emb_dim]")
        if prep is None:
            prep = self._prep(edge_index, edge_type, node_type)
        if prep.N != N:
            raise ValueError("node_type and x disagree on the number of nodes")
        shape = _lib.Shape(N, prep.E, D, self.head_count, self.n_ntype, self.n_etype, 1, prep.n_per_graph)
        folded = self._folded.get(shape, self.edge_encoder, [self], None, dev)
        ws_bytes = lib.qagnn_forward_workspace_bytes(C.byref(shape))
        ws = self._ws.get(ws_bytes, dev)
        out = torch.empty(N, D, dtype=dt, device=dev)
        alpha = torch.empty(N + prep.E, self.head_count, dtype=torch.float32, device=dev) if return_attention_weights else None
        aggr = torch.empty(N, D, dtype=torch.float32, device=dev) if return_aggr else None
        with torch.cuda.device(dev):
            if prep.node_ptr is not None:
                st = lib.qagnn_gatconve_forward_ragged(C.byref(shape), _lib.DTYPE_CODES[dt], _lib.DTYPE_CODES[xc.dtype],
                                                       prep.n_graphs, _lib.ptr(prep.node_ptr), 0, _lib.ptr(xc), _lib.ptr(ex),
                                                       _lib.ptr(prep.buf), _lib.ptr(folded), _lib.ptr(out), _lib.ptr(alpha),
                                                       _lib.ptr(aggr), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
            else:
                st = lib.qagnn_gatconve_forward_typed(C.byref(shape), _lib.DTYPE_CODES[dt], _lib.DTYPE_CODES[xc.dtype], 0,
                                                      _lib.ptr(xc), _lib.ptr(ex),
                                                      _lib.ptr(prep.buf), _lib.ptr(folded), _lib.ptr(out), _lib.ptr(alpha),
                                                      _lib.ptr(aggr), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_gatconve_forward_typed")
        self._alpha = None
        res = out
        if return_attention_weights:
            res = (out, (prep.edge_index_prime(), prep.compact_edges(alpha)))
        if return_aggr:
            return res, aggr
        return res


class QAGNN_Message_Passing(nn.Module):
    def __init__(self, args, k, n_ntype, n_etype, input_size, hidden_size, output_size, dropout=0.1):
        super().__init__()
        if input_size != output_size or input_size != hidden_size:
            raise ValueError("QAGNN_Message_Passing requires input_size == hidden_size == output_size")
        self.args = args
        self.n_ntype, self.n_etype = n_ntype, n_etype
        self.hidden_size = hidden_size
        self.emb_node_type = nn.Linear(self.n_ntype, hidden_size // 2)
        self.basis_f = "sin"
        self.emb_score = nn.Linear(hidden_size // 2, hidden_size // 2)
        self.edge_encoder = nn.Sequential(nn.Linear(n_etype + 1 + n_ntype * 2, hidden_size), nn.BatchNorm1d(hidden_size),
                                          nn.ReLU(), nn.Linear(hidden_size, hidden_size))
        self.k = k
        self.gnn_layers = nn.ModuleList([GATConvE(args, hidden_size, n_ntype, n_etype, self.edge_encoder) for _ in range(k)])
        self.Vh = nn.Linear(input_size, output_size)
        self.Vx = nn.Linear(hidden_size, output_size)
        self.activation = GELU()
        self.dropout = nn.Dropout(dropout)
        self.dropout_rate = dropout
        # 1.1^j in float32, computed on the host exactly as torch.pow(1.1, arange) does in the
        # reference (:70-71); uploaded as a constant so host and device agree bit for bit
        self.register_buffer("_score_basis", torch.pow(1.1, torch.arange(hidden_size // 2).float()), persistent=False)
        self.check_indices = True
        # use_cuda_graph: capture graph prep + the whole k-layer launch sequence (~60 kernels) into one CUDA graph per
        # (input buffers, weights) and replay it; the returned tensor is then a static buffer that the next replay
        # overwrites.  A replay cannot synchronise to validate indices: see _graphed_forward.
        self.use_cuda_graph = False
        self._graphs = {}
        self._replayed = []  # pipeline.StatusWord of every replay whose status word has not been looked at yet
        self._folded = _FoldedWeights()
        # a captured graph bakes in the workspace / folded-blob addresses: drop the graphs before either is replaced
        self._ws = _DeviceBlob(on_replace=self._graphs.clear)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate())

    def invalidate(self):
        """Drops the folded weights and every captured CUDA graph.  Called automatically by load_state_dict() and
        .to()/.cuda(); call it yourself after in-place edits through `.data` (e.g. `p.data.normal_()`, EMA swaps),
        which do not bump the tensor version the caches are keyed on."""
        self._folded.invalidate()
        self._graphs.clear()

    def _apply(self, fn, *a, **kw):
        self.invalidate()
        return super()._apply(fn, *a, **kw)

    # -- helpers ------------------------------------------------------------------------------
    def _shape(self, N, E, n_per_graph):
        return _lib.Shape(N, E, self.hidden_size, self.gnn_layers[0].head_count if self.k else 4, self.n_ntype,
                          self.n_etype, self.k, n_per_graph)

    def _mp_tensors(self):
        return [self.emb_node_type.weight, self.emb_node_type.bias, self.emb_score.weight, self.emb_score.bias,
                self.Vh.weight, self.Vh.bias, self.Vx.weight, self.Vx.bias, self._score_basis]

    def check_batch(self, A, node_type):
        """Validates the indices of a batch once (synchronising); raises IndexError like forward() with check_indices."""
        graph_prep(A, node_type, node_type.size(1) if node_type.dim() == 2 else 0, self.n_ntype, self.n_etype, True)

    def prepare_graph(self, edge_index, edge_type, node_type):
        """Builds the layer-invariant graph workspace; pass it back via forward(..., prep=) to amortise
        it over repeated forwards on the same batch."""
        n = node_type.size(1) if node_type.dim() == 2 else 0
        return graph_prep((edge_index, edge_type), node_type, n, self.n_ntype, self.n_etype, self.check_indices)

    def mp_helper(self, _X, edge_index, edge_type, _node_type, _node_feature_extra):
        for layer in self.gnn_layers:
            _X = self.activation(layer(_X, edge_index, edge_type, _node_type, _node_feature_extra))
        return _X

    def node_feature_extra(self, node_type, node_score):
        """[B*n, D] = [GELU(emb_node_type(onehot(type))) ‖ GELU(emb_score(sin(1.1^j * score)))] (:62-73,86)."""
        lib = _lib.load()
        nt = _lib.i64c(node_type.reshape(-1), "node_type")
        sc = _lib.f32c(node_score.reshape(-1), "node_score")
        dev = nt.device
        shape = self._shape(nt.numel(), 0, 0)
        folded = self._folded.get(shape, self.edge_encoder, list(self.gnn_layers), self._mp_tensors(), dev)
        ws = self._ws.get(lib.qagnn_forward_workspace_bytes(C.byref(shape)), dev)
        out = torch.empty(nt.numel(), self.hidden_size, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            st = lib.qagnn_node_feature_extra(C.byref(shape), _lib.ptr(nt), _lib.ptr(sc), _lib.ptr(folded), _lib.ptr(out),
                                              _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_node_feature_extra")
        return out

    def forward(self, H, A, node_type, node_score, cache_output=False, prep=None, return_layers=False):
        """
        H: tensor of shape (batch_size, n_node, d_node) — node features from the previous layer
        A: (edge_index [2, total_E], edge_type [total_E]) of the batched graph
        node_type: long tensor (batch_size, n_node): 0 question entity, 1 answer entity, 2 other, 3 context
        node_score: tensor (batch_size, n_node, 1)
        returns (batch_size, n_node, d_node)

        With A a ragged qagnn_b200.data.PackedAdj (eval only): H [N_cap, d_node], node_type [N_cap], node_score [N_cap, 1],
        one row per node of the batch (rows past A.node_ptr[-1] unused); returns [N_cap, d_node].

        In .train(), or in .eval() with H or node_score requiring grad, the output is differentiable (qagnn_b200/training.py).
        """
        ragged = getattr(A, "ragged", False)
        if ragged:
            _refuse_ragged_training(self, "QAGNN_Message_Passing")
        for status in self._replayed:  # never waits for the GPU: a replay whose copy has not landed is looked at later
            status.check("QAGNN_Message_Passing")
        self._replayed = [s for s in self._replayed if s.pending is not None]
        if _wants_autograd(self, H, node_score):  # autograd through the CUDA message passing, this module's mode (training.py)
            if prep is None:  # a PackedAdj (possibly at an edge capacity) gets the packed prep, a plain pair the general one
                n = H.size(1) if getattr(A, "graph_ptr_dev", None) is not None else 0
                prep = graph_prep(A, node_type, n, self.n_ntype, self.n_etype, self.check_indices)
            self._last_prep = prep
            return TR.mp_forward_autograd(self, H, A, node_type, node_score, prep)
        if self.use_cuda_graph and prep is None and not return_layers:
            return self._graphed_forward(H, A, node_type, node_score)
        lib = _lib.load()
        # under bf16 autocast: bf16 in and out, single-pass bf16 GEMMs (include/qagnn_b200.h, qagnn_mp_forward_typed)
        Hc, dt = _lib.eval_dtype(H, "H")
        if ragged:
            if Hc.dim() != 2 or Hc.size(1) != self.hidden_size:
                raise ValueError("H of a ragged batch must be [node_capacity, hidden_size]")
            Hc = Hc.unsqueeze(0)
        if Hc.dim() != 3 or Hc.size(2) != self.hidden_size:
            raise ValueError("H must be [batch, n_node, hidden_size]")
        B, n, D = Hc.shape
        dev = Hc.device
        nt = _lib.i64c(node_type.reshape(-1), "node_type")
        sc = _lib.f32c(node_score.reshape(-1), "node_score")
        if nt.numel() != B * n or sc.numel() != B * n:
            raise ValueError("node_type / node_score must be [batch, n_node(, 1)]")
        edge_index, edge_type = A  # a (edge_index, edge_type) pair, or a qagnn_b200.data.PackedAdj (iterates as that pair)
        if prep is None:
            prep = graph_prep(A, nt, n, self.n_ntype, self.n_etype, self.check_indices)
        self._last_prep = prep
        if prep.N != B * n:
            raise ValueError("graph workspace was built for a different number of nodes")
        shape = self._shape(B * n, prep.E, prep.n_per_graph)
        folded = self._folded.get(shape, self.edge_encoder, list(self.gnn_layers), self._mp_tensors(), dev)
        ws = self._ws.get(lib.qagnn_forward_workspace_bytes(C.byref(shape)), dev)
        out = torch.empty(B, n, D, dtype=dt, device=dev)
        layers = torch.empty(self.k, B * n, D, dtype=torch.float32, device=dev) if return_layers else None
        with torch.cuda.device(dev):
            if prep.node_ptr is not None:
                st = lib.qagnn_mp_forward_ragged(C.byref(shape), _lib.DTYPE_CODES[dt], _lib.DTYPE_CODES[Hc.dtype], prep.n_graphs,
                                                 _lib.ptr(prep.node_ptr), _lib.ptr(Hc), _lib.ptr(nt), _lib.ptr(sc),
                                                 _lib.ptr(prep.buf), _lib.ptr(folded), _lib.ptr(out), _lib.ptr(layers),
                                                 _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
            else:
                st = lib.qagnn_mp_forward_typed(C.byref(shape), _lib.DTYPE_CODES[dt], _lib.DTYPE_CODES[Hc.dtype], _lib.ptr(Hc),
                                                _lib.ptr(nt), _lib.ptr(sc), _lib.ptr(prep.buf), _lib.ptr(folded), _lib.ptr(out),
                                                _lib.ptr(layers), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
        _lib.check(st, "qagnn_mp_forward_typed")
        if ragged:
            out = out[0]
        if return_layers:
            return out, layers
        return out

    def _graphed_forward(self, H, A, node_type, node_score):
        """CUDA-graph replay of forward() for inputs that live in the same device buffers as when it was captured.  With
        check_indices on at capture, each replay's index checks reach the host through its graph's StatusWord: forward()
        raises IndexError once the copy of a bad replay has landed, also after the graph was evicted or invalidated."""
        tensors = [H, A[0], A[1], node_type, node_score]
        if getattr(A, "graph_ptr_dev", None) is not None:
            tensors.append(A.graph_ptr_dev)
        if getattr(A, "ragged", False):
            tensors.append(A.node_ptr_dev)
        # the autocast dtype selects the kernels and the output dtype: an fp32 capture must not replay under bf16 autocast
        key = (tuple((t.data_ptr(), tuple(t.shape), t.dtype) for t in tensors),
               _version_key(list(self.parameters()) + list(self.buffers())), _lib.autocast_dtype())
        entry = self._graphs.get(key)
        if entry is None:
            from .pipeline import capture
            captured = capture(self, A, node_type, "QAGNN_Message_Passing", lambda: self.forward(H, A, node_type, node_score))
            if len(self._graphs) >= 8:
                self._graphs.pop(next(iter(self._graphs)))
            # the entry keeps alive everything whose address the graph baked in: the inputs and what capture() kept
            entry = self._graphs[key] = captured + (tensors,)
        graph, out, status = entry[:3]
        graph.replay()
        status.replayed()
        if status not in self._replayed:
            self._replayed.append(status)
        return out


def decoder_tail(pooler, sent_vecs, gnn_output, node_type_ids, adj_lengths, fused=True, dropout=None):
    """The decoder tail of a padded batch (modeling_qagnn.py:172-187): (cat(graph_vecs, sent_vecs, Z) [B, 2D + S], pool_attn).
    With `fused` it first tries pooler.pool_concat, mask + pooling + cat in one kernel, which runs in eval only, where
    dropout is the identity.  When that is off or refuses the shape: the pool mask, pooler(...) and torch.cat, with
    `dropout` (if given) applied to the concat."""
    if fused:
        out = pooler.pool_concat(sent_vecs, gnn_output, node_type_ids, adj_lengths)
        if out is not None:
            return out
    pos = torch.arange(gnn_output.size(1), device=gnn_output.device)
    mask = (pos >= adj_lengths.unsqueeze(1)) | (node_type_ids == 3)
    mask[:, 0] = mask[:, 0] & ~mask.all(1)  # a fully masked row keeps node 0 (:176; written without a host sync)
    graph_vecs, pool_attn = pooler(sent_vecs, gnn_output, mask)
    concat = torch.cat((graph_vecs, sent_vecs, gnn_output[:, 0]), 1)
    return (concat if dropout is None else dropout(concat)), pool_attn


class QAGNN(nn.Module):
    """Decoder around the message passing (modeling_qagnn.py:99-189); plain PyTorch on the caller side."""

    def __init__(self, args, k, n_ntype, n_etype, sent_dim, n_concept, concept_dim, concept_in_dim, n_attention_head,
                 fc_dim, n_fc_layer, p_emb, p_gnn, p_fc, pretrained_concept_emb=None, freeze_ent_emb=True,
                 init_range=0.02):
        super().__init__()
        self.init_range = init_range
        self.concept_emb = CustomizedEmbedding(concept_num=n_concept, concept_out_dim=concept_dim, use_contextualized=False,
                                               concept_in_dim=concept_in_dim, pretrained_concept_emb=pretrained_concept_emb,
                                               freeze_ent_emb=freeze_ent_emb)
        self.svec2nvec = nn.Linear(sent_dim, concept_dim)
        self.concept_dim = concept_dim
        self.activation = GELU()
        self.gnn = QAGNN_Message_Passing(args, k=k, n_ntype=n_ntype, n_etype=n_etype, input_size=concept_dim,
                                         hidden_size=concept_dim, output_size=concept_dim, dropout=p_gnn)
        self.pooler = MultiheadAttPoolLayer(n_attention_head, sent_dim, concept_dim)
        self.fc = MLP(concept_dim + sent_dim + concept_dim, fc_dim, 1, n_fc_layer, p_fc, layer_norm=True)
        self.dropout_e = nn.Dropout(p_emb)
        self.dropout_fc = nn.Dropout(p_fc)
        if init_range > 0:
            self.apply(self._init_weights)

    def _init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.init_range)
            if getattr(module, "bias", None) is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def pooled_features(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj, emb_data=None,
                        cache_output=False):
        """Everything up to (and excluding) the answer MLP: returns (concat [B, 2*concept_dim+sent_dim], pool_attn).
        Split out so a data-parallel caller can all-gather `concat` before `fc` (qagnn_b200.distributed)."""
        if getattr(adj, "ragged", False):
            return self._pooled_features_ragged(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj, emb_data,
                                                cache_output)
        n = node_scores.size(1)
        fused_head = (not self.training and not torch.is_grad_enabled() and emb_data is None and node_scores.is_cuda
                      and not self.concept_emb.use_contextualized and self.concept_dim % 4 == 0
                      and concept_ids.device == node_scores.device and sent_vecs.dtype == torch.float32)
        if fused_head:
            # one kernel: context-node injection + concept rows gathered from the pre-projected table + score
            # normalisation (:153-167); the [B, sent_dim] svec2nvec GEMM stays a library call
            lib = _lib.load()
            B_ = concept_ids.size(0)
            table = self.concept_emb.projected_table()
            # the head kernel reads fp32: under autocast ctx comes out in the autocast dtype (its rounding is kept, as the
            # PyTorch head's torch.cat promotes it to fp32 too)
            ctx = self.activation(self.svec2nvec(sent_vecs)).float().contiguous()
            cid = _lib.i64c(concept_ids, "concept_ids")
            sc = _lib.f32c(node_scores.reshape(B_, n), "node_scores")
            al = _lib.i64c(adj_lengths, "adj_lengths")
            gnn_input = torch.empty(B_, n, self.concept_dim, dtype=torch.float32, device=sc.device)
            s = torch.empty(B_, n, dtype=torch.float32, device=sc.device)
            with torch.cuda.device(sc.device):
                st = lib.qagnn_decoder_head(B_, n, self.concept_dim, _lib.ptr(cid), table.size(0), _lib.ptr(table), _lib.ptr(ctx),
                                            _lib.ptr(sc), _lib.ptr(al), _lib.ptr(gnn_input), _lib.ptr(s), _lib.stream_ptr(sc.device))
            _lib.check(st, "qagnn_decoder_head")
            s = s.unsqueeze(2)
        else:
            gnn_input, s = self._head(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, emb_data)

        gnn_output = self.gnn(gnn_input, adj, node_type_ids, s)
        fc_in = self.dropout_fc
        concat, pool_attn = decoder_tail(self.pooler, sent_vecs, gnn_output, node_type_ids, adj_lengths,
                                         fused=not self.training,
                                         dropout=lambda c: TR.dropout(c, fc_in.p, fc_in.training, TR.SITE_FC_IN))
        if cache_output:
            self.concept_ids, self.adj, self.pool_attn = concept_ids, adj, pool_attn
        return concat, pool_attn

    def _head(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, emb_data):
        """The input assembly in PyTorch ops (modeling_qagnn.py:153-167): (gnn_input [B, n, D], normalised scores [B, n, 1])."""
        n = node_scores.size(1)
        gnn_input0 = self.activation(self.svec2nvec(sent_vecs)).unsqueeze(1)
        gnn_input1 = self.concept_emb(concept_ids[:, 1:] - 1, emb_data).to(node_type_ids.device)
        gnn_input = TR.dropout(torch.cat([gnn_input0, gnn_input1], dim=1), self.dropout_e.p, self.dropout_e.training,
                               TR.SITE_EMB)
        valid = (torch.arange(n, device=node_scores.device) < adj_lengths.unsqueeze(1)).float()
        s = -node_scores
        s = (s - s[:, 0:1, :]).squeeze(2) * valid
        mean_norm = s.abs().sum(dim=1) / adj_lengths
        return gnn_input, (s / (mean_norm.unsqueeze(1) + 1e-05)).unsqueeze(2)

    def _pooled_features_ragged(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj, emb_data,
                                cache_output):
        """pooled_features on a ragged PackedAdj (eval): the head writes only the valid positions of the padded [B, n] inputs
        as packed rows (qagnn_decoder_head_ragged), the message passing runs on adj.node_capacity rows and the tail pools each
        graph over its own rows (qagnn_decoder_tail_ragged); `pool_attn` keeps the padded [n_head*B, n] layout.
        Under grad mode the head is the PyTorch one (as in the padded layout), its rows gathered into the packed layout, so
        autograd scatters dL/d(packed rows) back to the padded positions; the padded batch's gradients result."""
        _refuse_ragged_training(self, "QAGNN")
        if (emb_data is not None or not node_scores.is_cuda or self.concept_emb.use_contextualized or self.concept_dim % 4 != 0
                or concept_ids.device != node_scores.device or sent_vecs.dtype != torch.float32):
            raise ValueError("QAGNN: a ragged batch needs the fused decoder head (CUDA inputs, fp32 sent_vecs, no contextualized "
                             "embeddings, concept_dim % 4 == 0)")
        B_, n = concept_ids.shape
        N_cap = adj.node_capacity
        dev = node_scores.device
        node_ptr = _lib.i64c(adj.node_ptr_dev, "node_ptr")
        if node_ptr.numel() != B_ + 1 or N_cap <= 0:
            raise ValueError("ragged PackedAdj: node_ptr must have one entry per graph plus one and node_capacity be set")
        al = _lib.i64c(adj_lengths, "adj_lengths")
        if torch.is_grad_enabled():
            gnn_input, s, nt = self._head_ragged(sent_vecs, concept_ids, node_type_ids, node_scores, al, node_ptr, N_cap)
        else:
            lib = _lib.load()
            table = self.concept_emb.projected_table()
            ctx = self.activation(self.svec2nvec(sent_vecs)).float().contiguous()
            gnn_input = torch.empty(N_cap, self.concept_dim, dtype=torch.float32, device=dev)
            s = torch.empty(N_cap, 1, dtype=torch.float32, device=dev)
            nt = torch.empty(N_cap, dtype=torch.int64, device=dev)
            with torch.cuda.device(dev):
                st = lib.qagnn_decoder_head_ragged(B_, n, self.concept_dim, N_cap, _lib.ptr(_lib.i64c(concept_ids, "concept_ids")),
                                                   table.size(0), _lib.ptr(table), _lib.ptr(ctx),
                                                   _lib.ptr(_lib.f32c(node_scores.reshape(B_, n), "node_scores")), _lib.ptr(al),
                                                   _lib.ptr(_lib.i64c(node_type_ids, "node_type_ids")), _lib.ptr(node_ptr),
                                                   _lib.ptr(gnn_input), _lib.ptr(s), _lib.ptr(nt), _lib.stream_ptr(dev))
            _lib.check(st, "qagnn_decoder_head_ragged")
        gnn_output = self.gnn(gnn_input, adj, nt, s)
        concat, pool_attn = self.pooler.pool_concat_ragged(sent_vecs, gnn_output, node_ptr, nt, adj_lengths, n)
        if cache_output:
            self.concept_ids, self.adj, self.pool_attn = concept_ids, adj, pool_attn
        return concat, pool_attn

    def _head_ragged(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, node_ptr, N_cap):
        """(gnn_input [N_cap, D], scores [N_cap, 1], node types [N_cap]): the PyTorch head's values at the rows
        qagnn_decoder_head_ragged writes.  Packed row r of graph b = position r - node_ptr[b] < adj_lengths[b]; the tail rows
        get zeros, score 0 and type 2.  A gather, so its gradient is a scatter to exactly one padded position per row."""
        B_, n = concept_ids.shape
        gnn_input, s = self._head(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, None)
        r = torch.arange(N_cap, device=node_ptr.device)
        g = (torch.searchsorted(node_ptr, r, right=True) - 1).clamp_(0, B_ - 1)
        i = r - node_ptr[g]
        valid = (r < node_ptr[-1]) & (i < adj_lengths[g].clamp(max=n))
        src = torch.where(valid, g * n + i, 0)
        v = valid.unsqueeze(1)
        gnn_input = torch.where(v, gnn_input.reshape(B_ * n, -1)[src], 0)
        s = torch.where(v, s.reshape(B_ * n, 1)[src], 0)
        nt = torch.where(valid, node_type_ids.reshape(-1)[src], 2)
        return gnn_input, s, nt

    def forward(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj, emb_data=None,
                cache_output=False):
        """sent_vecs (B, dim_sent); concept_ids (B, n_node); adj = (edge_index, edge_type);
        adj_lengths (B,); node_type_ids (B, n_node); node_scores (B, n_node, 1).  Returns (logits (B,1), pool_attn)."""
        concat, pool_attn = self.pooled_features(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj,
                                                 emb_data, cache_output)
        return self.fc(concat), pool_attn


class LM_QAGNN(nn.Module):
    """Text encoder + QAGNN decoder with the reference's positional-input forward (modeling_qagnn.py:192-251)."""

    def __init__(self, args, model_name, k, n_ntype, n_etype, n_concept, concept_dim, concept_in_dim, n_attention_head,
                 fc_dim, n_fc_layer, p_emb, p_gnn, p_fc, pretrained_concept_emb=None, freeze_ent_emb=True,
                 init_range=0.0, encoder_config={}):
        super().__init__()
        from .modeling_encoder import TextEncoder
        self.encoder = TextEncoder(model_name, **encoder_config)
        self.decoder = QAGNN(args, k, n_ntype, n_etype, self.encoder.sent_dim, n_concept, concept_dim, concept_in_dim,
                             n_attention_head, fc_dim, n_fc_layer, p_emb, p_gnn, p_fc,
                             pretrained_concept_emb=pretrained_concept_emb, freeze_ent_emb=freeze_ent_emb,
                             init_range=init_range)

    def forward(self, *inputs, layer_id=-1, cache_output=False, detail=False):
        """inputs = (*lm_inputs, concept_ids, node_type_ids, node_scores, adj_lengths, edge_index, edge_type) with a
        leading (batch, num_choice) pair of dims on the tensors and [batch][num_choice] nested lists for the last two
        (or a PackedAdj, see qagnn_b200.data).  Returns (logits [batch, num_choice], pool_attn)."""
        from .data import PackedAdj
        bs, nc = inputs[0].size(0), inputs[0].size(1)
        edge_index_orig, edge_type_orig = inputs[-2:]
        flat = [x.reshape(x.size(0) * x.size(1), *x.size()[2:]) for x in inputs[:-2]]
        *lm_inputs, concept_ids, node_type_ids, node_scores, adj_lengths = flat
        if isinstance(edge_index_orig, PackedAdj):  # pre-packed batch (qagnn_b200.data.pack_adj); edge_type slot unused
            adj = edge_index_orig.to(node_type_ids.device)  # keeps graph_ptr: graph prep is then one launch per batch
        else:
            edge_index, edge_type = self.batch_graph(sum(edge_index_orig, []), sum(edge_type_orig, []), concept_ids.size(1))
            adj = (edge_index.to(node_type_ids.device), edge_type.to(node_type_ids.device))
        sent_vecs, all_hidden_states = self.encoder(*lm_inputs, layer_id=layer_id)
        logits, attn = self.decoder(sent_vecs.to(node_type_ids.device), concept_ids, node_type_ids, node_scores,
                                    adj_lengths, adj, emb_data=None, cache_output=cache_output)
        logits = logits.view(bs, nc)
        if not detail:
            return logits, attn
        return (logits, attn, concept_ids.view(bs, nc, -1), node_type_ids.view(bs, nc, -1), edge_index_orig,
                edge_type_orig)

    def batch_graph(self, edge_index_init, edge_type_init, n_nodes):
        """list of [2,E_i] / [E_i] -> one [2, total_E] / [total_E] with node ids offset by i*n_nodes (:244-251)."""
        n_examples = len(edge_index_init)
        offsets = torch.repeat_interleave(
            torch.arange(n_examples, device=edge_index_init[0].device) * n_nodes,
            torch.tensor([e.size(1) for e in edge_index_init], device=edge_index_init[0].device))
        edge_index = torch.cat(edge_index_init, dim=1) + offsets.unsqueeze(0)
        edge_type = torch.cat(edge_type_init, dim=0)
        return edge_index, edge_type
