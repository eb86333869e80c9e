"""Host<->device streaming and whole-step CUDA graphs around the hot path (caller side, SURVEY.md §8e / §8f #1-2).

`DecoderStep` is the step a data-parallel rank runs on its shard of sub-graphs (modeling_qagnn.py:170-188):

    QAGNN_Message_Passing.forward -> pool mask -> MultiheadAttPoolLayer -> cat(graph_vecs, sent_vecs, Z)
      -> [ONE all_gather_into_tensor over the ranks] -> answer MLP `fc` on the whole batch

captured as ONE CUDA graph (graph prep, the k layers, the fused pooling kernel, the NCCL all-gather and the answer MLP
are all graph nodes; inputs and outputs are static device buffers).  With world_size == 1 the collective is absent.

`StreamedRunner` feeds batches that live in pinned host memory through such a step (or through a bare
`QAGNN_Message_Passing`) with the copies on their own CUDA streams: while batch i computes, batch i+1 is uploaded and
the result of batch i-1 is downloaded (PCIe is full duplex), each batch in one of `depth` device buffer sets.  Every
batch still pays its own H2D and D2H; they just stop serialising with the kernels.

`TrainStep` is the training counterpart of DecoderStep: QAGNN.forward in .train() and its backward as two CUDA graphs,
behind one autograd node, for the micro-steps of qagnn.py:252-278.

`SplitEvalStep` evaluates a split held on the GPU (qagnn_b200.data.DeviceSplit): one CUDA graph assembles a batch from its
question ids and runs QAGNN.forward in .eval() on it, so nothing of the batch is packed or uploaded on the host.

`SplitTrainStep` trains from such a split: its forward graph assembles the micro-batch, gathers its labels and takes the
cross-entropy or margin-rank loss; its backward graph adds the parameter gradients into `.grad` itself.
"""
import contextlib

import torch

from . import distributed as _dist
from .data import PackedAdj
from .modeling_qagnn import _version_key, decoder_tail
from .training import answer_loss, check_answer_loss

_EVAL_AUTOCAST = (None, torch.bfloat16)
_TRAIN_AUTOCAST = (None, torch.float16, torch.bfloat16)


def _checked_autocast(dtype, allowed):
    """`dtype` when it is one of `allowed` (None: no autocast), else ValueError."""
    if dtype not in allowed:
        names = [str(d) for d in allowed]
        raise ValueError(f"autocast_dtype must be {', '.join(names[:-1])} or {names[-1]}")
    return dtype


def _autocast(dtype):
    """The context a step captures and runs under: torch.autocast(dtype, cache_enabled=False), or none for dtype None."""
    if dtype is None:
        return contextlib.nullcontext()
    return torch.autocast("cuda", dtype=dtype, cache_enabled=False)


class StatusWord:
    """Graph prep's index checks across CUDA-graph replays, without blocking the host.  A replay cannot synchronise to
    validate a batch, so inside the capture `record(word)` ORs graph prep's status word into a device word and copies that
    to pinned memory.  `replayed()` marks the end of a replay, and `check()` raises IndexError once the copy of a replay
    has landed with a bit set: at a later call, never by waiting for the GPU.  Built without a device (index checks off),
    the word does nothing."""

    def __init__(self, device=None):
        self.accum = None if device is None else torch.zeros(1, dtype=torch.int32, device=device)
        self.host = None if device is None else torch.zeros(1, dtype=torch.int32).pin_memory()
        self.pending = None  # event after the last replay's copy

    def record(self, word):
        if self.accum is not None:
            self.accum.bitwise_or_(word)
            self.host.copy_(self.accum, non_blocking=True)

    def replayed(self):
        if self.accum is not None:
            self.pending = torch.cuda.Event()
            self.pending.record()

    def check(self, what):
        if self.pending is None or not self.pending.query():  # the accumulated word is looked at again later
            return
        self.pending = None
        bits = int(self.host.item())
        if bits != 0:
            self.accum.zero_()
            self.host.zero_()
            raise IndexError(f"qagnn_b200: a {what} replay saw edge_index / edge_type / node_type values out of range or "
                             f"crossing a sub-graph boundary (status bits {bits}); its results were computed from clamped indices")


@contextlib.contextmanager
def capture_guard(gnn, adj, node_type, what, warmup):
    """Prepares the capture of CUDA graphs that run QAGNN_Message_Passing `gnn` on the batch (adj, node_type) and yields the
    StatusWord the capture records graph prep's status word into (one that does nothing with gnn.check_indices off).
    Before it yields, it validates the batch once, eagerly, and runs `warmup` twice on a side stream: that folds the
    weights, sizes the workspaces and loads the kernels.  Inside, gnn.use_cuda_graph and gnn.check_indices are off: the
    module's kernels become nodes of the caller's graph, and a replay cannot synchronise.  Both are restored on exit.

    An adjacency that carries graph_ptr must get the packed prep, else ValueError: the general prep would keep the edge
    count of the batch it was captured on for every later batch written into the same buffers."""
    saved = gnn.use_cuda_graph, gnn.check_indices
    gnn.use_cuda_graph = False
    try:
        if saved[1]:
            gnn.check_batch(adj, node_type)
        gnn.check_indices = False
        dev = node_type.device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                warmup()
        torch.cuda.current_stream(dev).wait_stream(side)
        if getattr(adj, "graph_ptr_dev", None) is not None and not gnn._last_prep.packed:
            raise ValueError(f"{what}: the packed graph prep refuses these sub-graphs (too large for one CTA); a captured "
                             "general prep would keep the edge count of this batch for every later one")
        yield StatusWord(dev if saved[1] else None)
    finally:
        gnn.use_cuda_graph, gnn.check_indices = saved


def capture(gnn, adj, node_type, what, fn):
    """`fn()` captured as one CUDA graph under capture_guard, with graph prep's status word recorded at its end.  Returns
    (graph, what fn returned, StatusWord, kept).  `kept` holds the buffers of `gnn` whose addresses the graph baked in
    (workspace, folded weights, graph prep): the caller keeps it as long as it keeps the graph, else a later replay reads
    freed memory once gnn replaces them."""
    with capture_guard(gnn, adj, node_type, what, fn) as status:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = fn()
            status.record(gnn._last_prep.status_word())
    return graph, out, status, (gnn._ws.buf, gnn._folded.blob, gnn._last_prep)


class DecoderStep:
    """MP forward + pooling + (all-gather) + answer MLP on static device buffers, replayed as one CUDA graph.

    inputs (dict of device tensors, kept by reference): H [B,n,D], edge_index [2,E], edge_type [E], node_type [B,n],
    node_score [B,n,1], sent_vecs [B,S], adj_lengths [B].  Results (static buffers, overwritten by every run):
    `logits` [world*B, 1] (every rank holds all of them), `pool_attn` [n_head*B, n], `gnn_out` [B,n,D]."""

    FIELDS = ("H", "edge_index", "edge_type", "node_type", "node_score", "sent_vecs", "adj_lengths")
    PACKED_FIELDS = FIELDS + ("graph_ptr",)  # + first edge of every sub-graph, int64 [B + 1] (packed batches)
    # ragged batches: the packed fields with H [N_cap, D], node_type [N_cap] and node_score [N_cap, 1] holding one row per node
    # (qagnn_b200.data.PackedAdj with node_ptr); node_ptr itself is rebuilt from adj_lengths on the device in every run
    RAGGED_FIELDS = PACKED_FIELDS

    def __init__(self, gnn, pooler, fc, inputs, world_size=1, group=None, use_cuda_graph=True, max_edges=-1,
                 autocast_dtype=None, max_nodes=None):
        """`autocast_dtype` (None or torch.bfloat16) runs capture and calls under torch.autocast(cache_enabled=False): the
        message passing then runs its bf16 forward (single-pass bf16 GEMMs, `gnn_out` bf16) and the pooling reads that output
        directly.

        `inputs` may carry "graph_ptr" (device int64 [B + 1]) with `max_edges` = an upper bound of the edges of one sub-graph
        for every batch that will be written into these buffers: graph prep is then ONE launch (qagnn_graph_prep_packed).
        edge_index / edge_type may then be an edge capacity K wider than any batch (qagnn_b200.data.PackedAdj): the real
        edge count is read from graph_ptr on the device, so one capture serves every batch of a split that fits K and
        `max_edges`.  A capture raises ValueError if the packed prep refuses the shape, since the general prep would freeze
        the edge count of the batch it was captured on.

        A RAGGED step (inputs with 2-D H, RAGGED_FIELDS) runs the batch without padding rows: the node arrays have N_cap =
        H.size(0) rows (qagnn_b200.data.split_node_capacity), graph b's from node_ptr[b] = sum(adj_lengths[:b]) on, and
        `max_nodes` n bounds one graph's rows (the loader's max_node_num; `pool_attn` is [n_head*B, n]).  node_ptr is rebuilt
        from adj_lengths on the device in every run, so one capture at N_cap and the edge capacity serves every full batch of a
        split.  `gnn_out` is then [N_cap, D].  Single GPU only."""
        self.autocast_dtype = _checked_autocast(autocast_dtype, _EVAL_AUTOCAST)
        self.gnn, self.pooler, self.fc = gnn, pooler, fc
        self.inp = {k: inputs[k] for k in self.FIELDS}
        self.adj = (self.inp["edge_index"], self.inp["edge_type"])
        self.ragged = self.inp["H"].dim() == 2
        self._node_ptr = None
        if self.ragged:
            if world_size > 1:
                raise ValueError("DecoderStep: ragged batches run on one GPU (world_size == 1)")
            if "graph_ptr" not in inputs or max_edges < 0 or max_nodes is None:
                raise ValueError("DecoderStep: a ragged step needs inputs['graph_ptr'], max_edges and max_nodes")
            al = self.inp["adj_lengths"]
            self._node_ptr = torch.zeros(al.numel() + 1, dtype=torch.int64, device=al.device)
            self._update_node_ptr()
        if self.ragged or ("graph_ptr" in inputs and max_edges >= 0):
            self.inp["graph_ptr"] = inputs["graph_ptr"]
            self.adj = PackedAdj(edge_index=self.inp["edge_index"], edge_type=self.inp["edge_type"], graph_ptr=None,
                                 n_nodes=int(max_nodes) if self.ragged else self.inp["H"].size(1),
                                 graph_ptr_dev=self.inp["graph_ptr"], max_edges=int(max_edges),
                                 edge_capacity=self.inp["edge_index"].size(1), node_ptr_dev=self._node_ptr,
                                 node_capacity=self.inp["H"].size(0) if self.ragged else -1)
        self.world, self.group = world_size, group
        dev = self.inp["H"].device
        B, D = self.inp["sent_vecs"].size(0), self.inp["H"].size(-1)
        S = self.inp["sent_vecs"].size(1)
        self.full = torch.empty(world_size * B, 2 * D + S, device=dev) if world_size > 1 else None
        self.graph = None
        self.logits = self.pool_attn = self.gnn_out = None
        self.mode = "eager"
        if use_cuda_graph:
            self._capture()

    @torch.no_grad()
    def _eager(self):
        with _autocast(self.autocast_dtype):
            return self._eager_body()

    def _update_node_ptr(self):
        torch.cumsum(self.inp["adj_lengths"], 0, out=self._node_ptr[1:])

    def _eager_body(self):
        d = self.inp
        if self.ragged:
            self._update_node_ptr()
            out = self.gnn(d["H"], self.adj, d["node_type"], d["node_score"])
            concat, pool_attn = self.pooler.pool_concat_ragged(d["sent_vecs"], out, self._node_ptr, d["node_type"],
                                                               d["adj_lengths"], self.adj.n_nodes)
            return self.fc(concat), pool_attn, out
        out = self.gnn(d["H"], self.adj, d["node_type"], d["node_score"])
        concat, pool_attn = decoder_tail(self.pooler, d["sent_vecs"], out, d["node_type"], d["adj_lengths"])  # :172-187
        full = _dist.all_gather_rows(concat, self.world, self.group, True, self.full)       # the path's one collective
        return self.fc(full), pool_attn, out                                                # :188

    def _capture(self):
        # the warm-up also opens the NCCL channels of the all-gather
        self.graph, (self.logits, self.pool_attn, self.gnn_out), self._status, self._keep = capture(
            self.gnn, self.adj, self.inp["node_type"], "DecoderStep", self._eager)
        self.mode = "one CUDA graph (prep + k layers + pooling" + (" + all-gather" if self.world > 1 else "") + " + fc)"

    def run(self):
        """Enqueues one step on the current stream; returns (logits, pool_attn, gnn_out).  A replay whose batch had an
        index out of range (or an edge crossing its sub-graph) raises IndexError at a later call, once the copy of the
        status word has landed; its results were computed from clamped indices."""
        if self.graph is not None:
            self._status.check("DecoderStep")
            self.graph.replay()
            self._status.replayed()
        else:
            self.logits, self.pool_attn, self.gnn_out = self._eager()
        return self.logits, self.pool_attn, self.gnn_out


class _TrainingGraphs:
    """What TrainStep and SplitTrainStep share: the training forward and its backward captured as two CUDA graphs in one
    pool, after capture_guard's validation and warm-up, and the checks before and bookkeeping after every replay."""

    what = None  # the class name in messages

    def _init_training(self, decoder, autocast_dtype):
        self.autocast_dtype = _checked_autocast(autocast_dtype, _TRAIN_AUTOCAST)
        if not decoder.training:
            raise ValueError(f"{self.what} captures the training forward: call decoder.train() first")
        self.decoder = decoder
        self.deterministic = torch.are_deterministic_algorithms_enabled()
        self._fwd = None
        self.mode = "eager"

    def _addresses(self):
        return tuple(t.data_ptr() for t in self._params + self._buffers)

    def _capture_graphs(self, adj, node_type, forward, backward, owned=()):
        """Captures `forward()` -> (y, ...) and `backward(y, dy)` as two CUDA graphs in one pool, on the batch (adj,
        node_type) already in the static buffers.  capture_guard first validates that batch and runs forward + backward twice
        (dy = 1) on a side stream; the forward graph ends by recording graph prep's status word into self._status.  The
        warm-up really runs: the decoder's buffers, the .grad of its trainable parameters (self._params), the tensors `owned`
        and the CUDA RNG state are put back afterwards.  Returns (forward's outputs, the static dy buffer, backward's result)."""
        dec = self.decoder
        dev = node_type.device
        self._params = [p for p in dec.parameters() if p.requires_grad]
        self._buffers = list(dec.buffers())

        def warmup():  # also builds the cached tables of the training path
            out = forward()
            backward(out[0], torch.ones_like(out[0]))

        saved = [b.detach().clone() for b in self._buffers + list(owned)]
        grads = [None if p.grad is None else p.grad.detach().clone() for p in self._params]
        rng = torch.cuda.get_rng_state(dev)
        try:
            with capture_guard(dec.gnn, adj, node_type, self.what, warmup) as status:
                pool = torch.cuda.graph_pool_handle()
                fwd, bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(fwd, pool=pool):
                    out = forward()
                    status.record(dec.gnn._last_prep.status_word())
                dy = torch.empty_like(out[0])
                with torch.cuda.graph(bwd, pool=pool):
                    res = backward(out[0], dy)
            self._fwd, self._bwd, self._status = fwd, bwd, status
            self._bn_buffers = [b for m in dec.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)
                                for b in (m.running_mean, m.running_var, m.num_batches_tracked) if b is not None]
            self._ptrs = self._addresses()
            self.mode = "two CUDA graphs (forward + backward)"
            return out, dy, res
        finally:
            with torch.no_grad():
                for b, s in zip(self._buffers + list(owned), saved):
                    b.copy_(s)
            for p, g in zip(self._params, grads):
                p.grad = g
            torch.cuda.set_rng_state(rng, dev)

    def _check_replay(self):
        """Before a replay: RuntimeError when the graphs no longer fit the decoder, IndexError when an earlier replay's graph
        prep flagged its batch."""
        what = self.what
        if not self.decoder.training:
            raise RuntimeError(f"{what} replays the training forward: call decoder.train() first")
        if self._addresses() != self._ptrs:
            raise RuntimeError(f"{what}: the decoder's parameters or buffers moved since capture (.to() / .cuda() / "
                               f".half()?); the graphs would read the old addresses. Build a new {what}.")
        if torch.are_deterministic_algorithms_enabled() != self.deterministic:
            raise RuntimeError(f"{what} was captured with torch.use_deterministic_algorithms({self.deterministic}) and "
                               f"its backward graph holds that mode's kernels; the flag changed since. Build a new {what}.")
        self._status.check(what)

    def _replayed(self):
        self._status.replayed()
        # the replay changed the running statistics behind autograd's back: the eval path's folded weights key on versions
        torch.autograd.graph.increment_version(self._bn_buffers)


class _TrainReplay(torch.autograd.Function):
    """The captured forward and backward of a TrainStep as one autograd node.  Gradient accumulation into `.grad` stays in
    autograd, outside the graphs.  The backward hands out the static gradient buffers themselves: autograd then copies
    them into a `.grad` that is still None instead of adopting them, which the next replay would overwrite."""

    @staticmethod
    def forward(ctx, step, sent_vecs, node_scores, *params):
        for static, given in ((step._sv, sent_vecs), (step._ns, node_scores)):
            if static.data_ptr() != given.data_ptr():
                static.copy_(given)
        step._fwd.replay()
        ctx.step = step
        logits, pool_attn = step._logits.detach(), step._pool_attn.detach()
        ctx.mark_non_differentiable(pool_attn)
        return logits, pool_attn

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_logits, _d_pool_attn):
        step = ctx.step
        step._g_logits.copy_(d_logits)
        step._bwd.replay()
        return (None,) + tuple(g if need else None for g, need in zip(step._grads, ctx.needs_input_grad[1:]))


class TrainStep(_TrainingGraphs):
    """QAGNN.forward in .train() and its backward, each replayed as one CUDA graph: the training counterpart of DecoderStep
    for the loop body of qagnn.py:252-278, on packed batches at a fixed edge capacity K
    (qagnn_b200.data.PackedAdjBatchGenerator(..., edge_capacity=K)):

        sent_vecs, _ = model.encoder(*lm_inputs)                                    # eager
        logits, pool_attn = step(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, packed_adj)
        loss = compute_loss(logits.view(bs, nc), labels)
        scaler.scale(loss).backward()     # replays the backward graph; dL/dsent_vecs flows on into the encoder

    Every call copies its batch into static buffers, so a batch with any edge count up to K and sub-graphs of at most
    `max_edges` edges replays the same two graphs; a larger batch raises ValueError before anything is copied.  Parameter
    gradients accumulate into `.grad` as in eager mode; dL/dsent_vecs reaches `sent_vecs`, and dL/dnode_scores reaches
    `node_scores` when it requires grad.  `pool_attn` is returned without a gradient.  Both outputs are static buffers that
    the next call overwrites.  Dropout draws a new mask on every replay and BatchNorm running statistics advance on every
    replay, as in eager mode.  `autocast_dtype` (None, torch.float16 or torch.bfloat16) runs capture and calls under
    torch.autocast(cache_enabled=False); the message-passing kernels read and write that dtype and compute in fp32 inside, and
    the edge encoder's BatchNorm moments stay fp32.  fp16 needs a GradScaler as above; bf16 has fp32's exponent range and needs
    none (`loss.backward()`).  Construction runs two warm-up iterations
    and restores the buffers, `.grad` and the CUDA RNG state it found.

    Out-of-range indices in a later batch raise IndexError at a later call, as with DecoderStep, without blocking the host;
    that batch's results were computed from clamped indices.  The graphs hold the addresses of the parameters and buffers:
    in-place optimiser steps and load_state_dict keep them, `.to()` / `.cuda()` / `.half()` do not, and a call after one
    raises RuntimeError (build a new TrainStep).  `use_cuda_graph=False` runs the same code eagerly.

    Under torch.use_deterministic_algorithms(True) at construction, the backward graph holds the message-passing core's
    deterministic backward (edge-table gradients summed in a fixed order), so two replays of one batch from one CUDA RNG state
    give the same gradients bit for bit.  `deterministic` records that mode; a graph call after the flag changed raises
    RuntimeError (build a new TrainStep)."""

    what = "TrainStep"

    def __init__(self, decoder, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, packed_adj, *, max_edges,
                 edge_capacity=None, autocast_dtype=None, use_cuda_graph=True):
        """The example batch (device tensors with the shapes of every later batch, valid indices, `packed_adj` a PackedAdj)
        sizes the static buffers and is what warm-up and capture run on.  `edge_capacity` K defaults to the width of
        packed_adj's edge buffer; `max_edges` bounds the edges of one sub-graph over the whole split
        (FlatAdjCache.max_graph_edges())."""
        self._init_training(decoder, autocast_dtype)
        dev = node_type_ids.device
        B, n = node_type_ids.shape
        K = int(edge_capacity) if edge_capacity is not None else packed_adj.edge_index.size(1)
        self.edge_capacity, self.max_edges = K, int(max_edges)
        self._sv = sent_vecs.detach().clone().requires_grad_(True)
        self._ns = node_scores.detach().clone().requires_grad_(True)
        self._cid, self._nt, self._al = concept_ids.clone(), node_type_ids.clone(), adj_lengths.clone()
        self._edges = torch.zeros(3, K, dtype=torch.int64, device=dev)
        self._gp = torch.zeros(B + 1, dtype=torch.int64, device=dev)
        self._adj = PackedAdj(edge_index=self._edges[:2], edge_type=self._edges[2], graph_ptr=None, n_nodes=n,
                              buf=self._edges, graph_ptr_dev=self._gp, max_edges=self.max_edges, edge_capacity=K)
        self._copy_batch(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, packed_adj)
        if use_cuda_graph:
            self._capture()

    def _copy_batch(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj):
        for name, t, static in (("sent_vecs", sent_vecs, self._sv), ("concept_ids", concept_ids, self._cid),
                                ("node_type_ids", node_type_ids, self._nt), ("node_scores", node_scores, self._ns),
                                ("adj_lengths", adj_lengths, self._al)):
            if t.shape != static.shape or t.dtype != static.dtype:
                raise ValueError(f"TrainStep: {name} is {tuple(t.shape)} {t.dtype}, the step was built for "
                                 f"{tuple(static.shape)} {static.dtype}")
        gp = adj.graph_ptr if adj.graph_ptr is not None else adj.graph_ptr_dev
        gp = gp.cpu() if gp.is_cuda else gp  # PackedAdj keeps graph_ptr on the host: no synchronisation
        if gp.numel() != self._gp.numel():
            raise ValueError(f"TrainStep: graph_ptr has {gp.numel()} entries, the step was built for {self._gp.numel()}")
        ne = adj.n_edges if adj.n_edges >= 0 else int(gp[-1])
        if ne > self.edge_capacity:
            raise ValueError(f"TrainStep: batch has {ne} edges, more than the edge capacity {self.edge_capacity}")
        me = int((gp[1:] - gp[:-1]).max()) if gp.numel() > 1 else 0
        if me > self.max_edges:
            raise ValueError(f"TrainStep: a sub-graph has {me} edges, more than max_edges = {self.max_edges}")
        for static, t in ((self._cid, concept_ids), (self._nt, node_type_ids), (self._al, adj_lengths)):
            static.copy_(t, non_blocking=True)
        if adj.buf is not None and adj.buf.shape == self._edges.shape:
            self._edges.copy_(adj.buf, non_blocking=True)
        elif ne > 0:
            self._edges[:2, :ne].copy_(adj.edge_index[:, :ne], non_blocking=True)
            self._edges[2, :ne].copy_(adj.edge_type[:ne], non_blocking=True)
        self._gp.copy_(adj.graph_ptr_dev if adj.graph_ptr_dev is not None else gp, non_blocking=True)

    def _capture(self):
        def forward():
            with _autocast(self.autocast_dtype):
                return self.decoder(self._sv, self._cid, self._nt, self._ns, self._al, self._adj)

        def backward(logits, d_logits):
            return torch.autograd.grad(logits, [self._sv, self._ns] + self._params, d_logits, allow_unused=True)

        (logits, pool_attn), self._g_logits, self._grads = self._capture_graphs(self._adj, self._nt, forward, backward)
        self._logits, self._pool_attn = logits.detach(), pool_attn.detach()

    def __call__(self, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, packed_adj):
        """Returns (logits [B, 1], pool_attn) of one micro-batch; `.backward()` through logits replays the backward graph."""
        if self._fwd is not None:
            self._check_replay()
        self._copy_batch(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, packed_adj)
        with _autocast(self.autocast_dtype):
            if self._fwd is None:
                return self.decoder(sent_vecs, self._cid, self._nt, node_scores, self._al, self._adj)
            out = _TrainReplay.apply(self, sent_vecs, node_scores, *self._params)
        self._replayed()
        return out


class _SplitBatches:
    """What SplitEvalStep and SplitTrainStep share: static buffers for batches of `batch_size` questions of a DeviceSplit at
    one edge capacity (and, ragged, one node capacity), the per-call check and upload of the question ids, and the
    assembly and decoder call their graphs hold.  A subclass provides `what` (its name in messages), `unit` (what a
    partial batch is called), `decoder`, `_sv` and `_check_sent_vecs`."""

    def _init_split(self, split, batch_size, edge_capacity, max_edges, node_capacity=None):
        self.split, self.batch_size = split, int(batch_size)
        self.edge_capacity, self.max_edges = int(edge_capacity), int(max_edges)
        self.node_capacity = node_capacity
        self._n_cap = -1 if node_capacity is None else int(node_capacity)
        self._qids = torch.zeros(self.batch_size, dtype=torch.int64, device=split.device)
        self._out = split.buffers(self.batch_size, self.edge_capacity, node_capacity)
        self._adj = split.packed_adj(self._out, self.max_edges, self.edge_capacity, self._n_cap)
        self.logits = self.pool_attn = None
        self.captures = 0

    def _load_ids(self, question_ids, sent_vecs):
        """Checks a call's question ids on the host (DeviceSplit.check), its batch size and its sent_vecs, and only then
        enqueues the upload of the ids: a refused call leaves the static buffers as they were."""
        q = self.split.check(question_ids, self.edge_capacity, self.node_capacity)[0]
        if q.size != self.batch_size:
            raise ValueError(f"{self.what}: {q.size} questions, the step was built for {self.batch_size}; run a partial "
                             f"{self.unit} through split.batch + decoder")
        self._check_sent_vecs(sent_vecs)
        # a pinned block from the caching host allocator per call: it is not reused before this copy has run
        self._qids.copy_(torch.from_numpy(q).pin_memory(), non_blocking=True)

    def _assemble(self):
        """Enqueues the assembly of the loaded ids' batch into the static buffers; returns them."""
        return self.split.assemble(self._qids, self.edge_capacity, self._n_cap, self._out)

    def _decode(self, out):
        """decoder(...) on the assembled buffers `out` and the step's sent_vecs: (logits, pool_attn)."""
        return self.decoder(self._sv, out["concept_ids"], out["node_type_ids"], out["node_scores"], out["adj_lengths"],
                            self._adj)


class SplitEvalStep(_SplitBatches):
    """Evaluation of a split held on the GPU (qagnn_b200.data.DeviceSplit) as one CUDA graph per step: batch assembly from the
    question ids (qagnn_assemble_batch), the node-row gathers and `decoder(...)` itself under no_grad, i.e. QAGNN.forward in
    .eval() (head kernel -> message passing -> pooling tail -> fc).  A call's only inputs are the question ids and sent_vecs:

        step = SplitEvalStep(model.decoder.eval(), split, bs, edge_capacity=K, max_edges=M)
        logits, pool_attn = step(qids, sent_vecs)      # static buffers, overwritten by the next call

    Each call checks the batch on the host (DeviceSplit.check: IndexError / ValueError before anything is enqueued), copies
    the ids and sent_vecs (as fp32, which both decoder heads read) into static buffers and replays the graph.  The results
    equal `decoder(sent_vecs.float(), *split.batch(qids, K, node_capacity))` under the same autocast, bit for bit.
    `node_capacity` N_cap (data.split_node_capacity) makes the step ragged; `max_edges` bounds one sub-graph's edges over the
    split (FlatAdjCache.max_graph_edges()).  `autocast_dtype` is None or torch.bfloat16, as for DecoderStep.  One GPU.

    The graph bakes in the folded weights and the projected concept table.  A call whose decoder changed since capture (an
    optimiser step, load_state_dict, .to(): the parameter and buffer versions, the folded weights' and the projected table's
    cache keys) captures again first, so results are never computed from stale weights; in-place `.data` edits need
    `decoder.gnn.invalidate()` / `decoder.concept_emb.invalidate_table()` as for eager calls.  The first call captures, on its own
    batch; a capture raises ValueError when the packed graph prep refuses the split's sub-graphs.  Every call needs exactly
    `batch_size` questions: run a final partial batch eagerly through split.batch + decoder, or with a step of its size.

    A split built with `labels` is also scored, as evaluate_accuracy and the test loop of qagnn.py:30-38,298-310 score it,
    inside the graph: pred = logits.view(bs, nc).argmax(1) (the first maximal choice on ties), `(pred == label).sum()` added
    into `n_correct` and bs into `n_scored` (0-dim int64), and pred written into `predictions` (int64 [Q], -1 for a question
    not scored since the last reset).  A question that appears more than once in a batch counts once per appearance and keeps
    its last appearance's prediction.  These device tensors are allocated once and keep accumulating across recaptures;
    `accuracy()` reads them once, `reset_scores()` starts over, and `score(question_ids, logits)` scores a final partial batch
    run through split.batch + decoder with the same ops.  A split without labels is not scored."""

    what, unit = "SplitEvalStep", "batch"

    def __init__(self, decoder, split, batch_size, *, edge_capacity, max_edges, node_capacity=None, autocast_dtype=None,
                 use_cuda_graph=True):
        self.autocast_dtype = _checked_autocast(autocast_dtype, _EVAL_AUTOCAST)
        if decoder.training:
            raise ValueError("SplitEvalStep runs the eval forward: call decoder.eval() first")
        self.decoder = decoder
        self._init_split(split, batch_size, edge_capacity, max_edges, node_capacity)
        dev = split.device
        self._sv = torch.zeros(self.batch_size * split.num_choice, decoder.svec2nvec.in_features, dtype=torch.float32,
                               device=dev)
        self.use_cuda_graph = use_cuda_graph
        self.graph, self._status, self._key = None, StatusWord(), None
        self.mode = "eager"
        self.n_correct = self.n_scored = self.predictions = None
        if split.labels is not None:
            self.n_correct = torch.zeros((), dtype=torch.int64, device=dev)
            self.n_scored = torch.zeros((), dtype=torch.int64, device=dev)
            # one slot past the split takes the predictions of earlier appearances of a repeated id, which nobody reads
            self._pred_slots = torch.full((split.n_questions + 1,), -1, dtype=torch.int64, device=dev)
            self.predictions = self._pred_slots[:-1]

    def _weights_key(self):
        """What the decoder's caches key on: parameter and buffer versions, the folded weights' key and the projected table's."""
        dec = self.decoder
        return (_version_key(list(dec.parameters()) + list(dec.buffers())), dec.gnn._folded.key,
                getattr(dec.concept_emb, "_ptab_key", None))

    def _check_sent_vecs(self, sent_vecs):
        if tuple(sent_vecs.shape) != tuple(self._sv.shape):
            raise ValueError(f"SplitEvalStep: sent_vecs is {tuple(sent_vecs.shape)}, the step was built for {tuple(self._sv.shape)}")

    @torch.no_grad()
    def _body(self):
        with _autocast(self.autocast_dtype):
            logits, pool_attn = self._decode(self._assemble())
        if self.n_correct is not None:
            self._score(self._qids, logits)
        return logits, pool_attn

    @torch.no_grad()
    def _score(self, qids, logits):
        """Enqueues the scoring of the questions `qids` (device int64 [bs], checked) from their logits; no host read."""
        bs = qids.numel()
        pred = logits.reshape(bs, self.split.num_choice).argmax(1)
        self.n_correct.add_((pred == torch.index_select(self.split.labels, 0, qids)).sum())
        self.n_scored.add_(bs)
        # each id is written by its last appearance only (the others go to the spare slot), so no two writes race
        pos = torch.arange(bs, device=qids.device)
        again_later = ((qids[:, None] == qids[None, :]) & (pos[:, None] < pos[None, :])).any(1)
        slot = torch.where(again_later, self.split.n_questions, qids)
        self._pred_slots.index_copy_(0, slot, pred)

    def _capture(self):
        self.graph, self._status = None, StatusWord()  # frees the previous capture's pool before the next one is made
        self._assemble()  # capture_guard validates this batch
        # capture_guard's warm-up really runs the body twice: keep it out of the scores
        scores = [] if self.n_correct is None else [self.n_correct, self.n_scored, self._pred_slots]
        saved = [t.clone() for t in scores]
        try:
            self.graph, (self.logits, self.pool_attn), self._status, kept = capture(
                self.decoder.gnn, self._adj, self._out["node_type_ids"], "SplitEvalStep", self._body)
        finally:
            for t, v in zip(scores, saved):
                t.copy_(v)
        self._keep = kept + (getattr(self.decoder.concept_emb, "_ptab", None),)  # the graph reads the projected table too
        self._key = self._weights_key()
        self.captures += 1
        self.mode = "one CUDA graph (assembly + gathers + head + prep + k layers + pooling + fc)"

    def __call__(self, question_ids, sent_vecs):
        """(logits [bs*nc, 1], pool_attn) of the questions `question_ids` (host ids, bs of them) with their sent_vecs
        [bs*nc, S] (device); static buffers that the next call overwrites."""
        if self.decoder.training:
            raise RuntimeError("SplitEvalStep runs the eval forward: call decoder.eval() first")
        self._status.check("SplitEvalStep")
        self._load_ids(question_ids, sent_vecs)
        if self._sv.data_ptr() != sent_vecs.data_ptr():
            self._sv.copy_(sent_vecs)
        if not self.use_cuda_graph:
            self.logits, self.pool_attn = self._body()
            return self.logits, self.pool_attn
        if self.graph is None or self._weights_key() != self._key:
            self._capture()  # on the batch just loaded, which the host checks accepted
        self.graph.replay()
        self._status.replayed()
        return self.logits, self.pool_attn

    def _require_labels(self):
        if self.n_correct is None:
            raise ValueError("SplitEvalStep: the split has no labels, so nothing is scored; build the DeviceSplit with labels=")

    def score(self, question_ids, logits):
        """Scores the questions `question_ids` (host ids, any number) from their logits [bs*nc, 1] or [bs, nc] (device), e.g.
        a final partial batch run through split.batch + decoder; the same ops the graph runs, enqueued on the current stream."""
        self._require_labels()
        q = self.split.check(question_ids, None)[0]
        if logits.numel() != q.size * self.split.num_choice:
            raise ValueError(f"SplitEvalStep.score: {logits.numel()} logits for {q.size} questions of "
                             f"{self.split.num_choice} choices")
        qids = torch.from_numpy(q).pin_memory().to(self.split.device, non_blocking=True)
        self._score(qids, logits)

    def accuracy(self):
        """n_correct / n_scored as a float: the one host read of the scores."""
        self._require_labels()
        correct, scored = torch.stack((self.n_correct, self.n_scored)).tolist()
        if scored == 0:
            raise ValueError("SplitEvalStep: no question was scored since the last reset")
        return correct / scored

    def reset_scores(self):
        """Zeroes n_correct and n_scored and sets every prediction to -1 (enqueued on the current stream)."""
        self._require_labels()
        self.n_correct.zero_()
        self.n_scored.zero_()
        self._pred_slots.fill_(-1)


class _SplitTrainReplay(torch.autograd.Function):
    """The captured forward and backward of a SplitTrainStep as one autograd node.  Its inputs are a zero-element anchor that
    always requires grad, so the node exists when sent_vecs does not (a frozen encoder), and sent_vecs.  The parameters are
    not inputs: the backward graph adds their gradients into the step-owned `.grad` buffers."""

    @staticmethod
    def forward(ctx, step, anchor, sent_vecs):
        if step._sv.data_ptr() != sent_vecs.data_ptr():
            step._sv.copy_(sent_vecs)
        step._fwd.replay()
        ctx.step, ctx.call = step, step.calls
        return step._loss.detach()

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_loss):
        step = ctx.step
        if ctx.call != step.calls:
            raise RuntimeError("SplitTrainStep: backward through the loss of an earlier call; the next call's forward replay "
                               "has overwritten its activations. Run each call's backward before the next call.")
        step._own_grads()
        step._d_loss.copy_(d_loss)
        step._bwd.replay()
        return None, None, step._g_sv if ctx.needs_input_grad[2] else None


class SplitTrainStep(_TrainingGraphs, _SplitBatches):
    """A training micro-step on a split held on the GPU (qagnn_b200.data.DeviceSplit built with `labels`) as two CUDA graphs:
    the loop body of qagnn.py:252-278 with `--loss cross_entropy` or `--loss margin_rank`, whose only per-call inputs are the
    question ids and sent_vecs:

        step = SplitTrainStep(model.decoder.train(), split, mbs, edge_capacity=K, max_edges=M, autocast_dtype=torch.float16,
                              loss=args.loss)
        loss = step(qids, sent_vecs) * len(qids) / bs     # qids: mbs host ids; the micro-batch's mean loss, fp32
        scaler.scale(loss).backward()                     # replays the backward graph

    The forward graph holds split.assemble (qagnn_assemble_batch and the node-row gathers), the gather of the micro-batch's
    labels, `decoder(...)` in .train() on the padded batch and training.answer_loss(logits, labels, num_choice, loss), under
    torch.autocast(autocast_dtype, cache_enabled=False) (None, torch.float16 or torch.bfloat16).  `loss` is "cross_entropy"
    (F.cross_entropy(logits.view(-1, num_choice), labels)) or "margin_rank" (the reference's margin-rank loss, with gathers
    where the reference selects with boolean masks); any other name, or "margin_rank" with one choice, raises ValueError at
    construction.  The results equal `decoder(sent_vecs, *split.batch(qids, K))` and the reference's loss under the same
    autocast.  A call checks the ids on the host (DeviceSplit.check: IndexError / ValueError before anything is enqueued),
    uploads them (8 bytes per question), copies sent_vecs into a static buffer (shape and dtype fixed by the first call, else
    ValueError) and replays the forward graph.  It returns the loss as a 0-dim fp32 tensor; `logits` [mbs*nc, 1] and `pool_attn` are static buffers for logging.
    The next call overwrites all three, so each call's backward must run before the next call (else RuntimeError).

    The backward graph is torch.autograd.grad of the loss, seeded with the scalar autograd hands the step's node (the loss
    weight times the GradScaler scale, read on the device), followed by one torch._foreach_add_ of the parameter gradients
    into step-owned buffers.  Before every backward replay each trainable parameter's `.grad` becomes its buffer: zeroed
    when `.grad` was None (zero_grad()), loaded from `.grad` when that was another tensor (zero_grad(set_to_none=False), an
    assignment).  So `.grad` holds what eager accumulation would, and GradScaler.unscale_, clip_grad_norm_ and the optimiser
    use it unchanged.  There is no AccumulateGrad node for the decoder's parameters: hooks registered on them
    (register_hook, register_post_accumulate_grad_hook) do not fire on replays (register_hook fires during the first
    call's capture, whose warm-up runs autograd.grad and discards the result).  dL/dsent_vecs flows on into the encoder when
    sent_vecs requires grad; with a frozen encoder backward() still accumulates the decoder's gradients.  A parameter the
    loss does not reach keeps `.grad` None, as in eager mode.

    The first call captures, on its own batch: the warm-up that precedes the capture restores BatchNorm buffers, `.grad` and
    the CUDA RNG state.  Dropout draws a new mask on every replay and BatchNorm running statistics advance on every replay.
    Optimiser steps and load_state_dict keep the parameters' addresses, so the graphs stay valid; a call raises RuntimeError
    after `.to()` / `.cuda()`, after torch.use_deterministic_algorithms changed, after a change in which decoder parameters
    require grad, and in .eval() (build a new SplitTrainStep).  Every call needs exactly `batch_size` questions: run a final
    partial micro-batch eagerly through split.batch + decoder + training.answer_loss.  Padded batches on one GPU only."""

    what, unit = "SplitTrainStep", "micro-batch"

    def __init__(self, decoder, split, batch_size, *, edge_capacity, max_edges, autocast_dtype=None, loss="cross_entropy"):
        """`edge_capacity` K bounds the edges of every micro-batch (FlatAdjCache.max_batch_edges(batch_size)), `max_edges` M
        those of one sub-graph over the split (FlatAdjCache.max_graph_edges()): one capture then serves every micro-batch."""
        self._init_training(decoder, autocast_dtype)
        if split.labels is None:
            raise ValueError("SplitTrainStep: the split has no labels; build the DeviceSplit with labels=")
        check_answer_loss(loss, split.num_choice)
        self.loss = loss
        largest = int(split.counts.max()) if split.counts.size else 0
        if int(max_edges) < largest:
            raise ValueError(f"SplitTrainStep: max_edges = {int(max_edges)}, the split has a sub-graph of {largest} edges")
        self._init_split(split, batch_size, edge_capacity, max_edges)
        self._labels = torch.zeros(self.batch_size, dtype=torch.int64, device=split.device)
        self._anchor = torch.empty(0, device=split.device, requires_grad=True)
        self._sv = None  # sized by the first call
        self.calls = 0

    def _check_sent_vecs(self, sent_vecs):
        want = (self.batch_size * self.split.num_choice, self.decoder.svec2nvec.in_features)
        if self._sv is None and (tuple(sent_vecs.shape) != want or not sent_vecs.is_floating_point()):
            raise ValueError(f"SplitTrainStep: sent_vecs is {tuple(sent_vecs.shape)} {sent_vecs.dtype}, the step needs "
                             f"floating-point {want}")
        if self._sv is not None and (sent_vecs.shape != self._sv.shape or sent_vecs.dtype != self._sv.dtype):
            raise ValueError(f"SplitTrainStep: sent_vecs is {tuple(sent_vecs.shape)} {sent_vecs.dtype}, the step was built "
                             f"for {tuple(self._sv.shape)} {self._sv.dtype}")

    def _forward(self):
        with _autocast(self.autocast_dtype):
            out = self._assemble()
            torch.index_select(self.split.labels, 0, self._qids, out=self._labels)
            logits, pool_attn = self._decode(out)
            loss = answer_loss(logits, self._labels, self.split.num_choice, self.loss)
        return loss, logits, pool_attn

    def _capture(self):
        bufs = [torch.zeros_like(p) for p in self.decoder.parameters() if p.requires_grad]
        used = []

        def backward(loss, d_loss):
            grads = torch.autograd.grad(loss, [self._sv] + self._params, d_loss, allow_unused=True)
            used[:] = [i for i, g in enumerate(grads[1:]) if g is not None]
            torch._foreach_add_([bufs[i] for i in used], [grads[1 + i] for i in used])
            return grads[0]

        self._assemble()  # capture_guard validates this batch
        (self._loss, logits, pool_attn), self._d_loss, self._g_sv = self._capture_graphs(
            self._adj, self._out["node_type_ids"], self._forward, backward, owned=bufs)
        self.logits, self.pool_attn = logits.detach(), pool_attn.detach()
        self._owned = [(self._params[i], bufs[i]) for i in used]
        self._requires_grad = [p.requires_grad for p in self.decoder.parameters()]
        self.captures += 1

    def _own_grads(self):
        """Makes every accumulated parameter's .grad the step's buffer, holding what .grad held (None counts as zeros)."""
        fresh = [b for p, b in self._owned if p.grad is None]
        if fresh:
            torch._foreach_zero_(fresh)
        for p, b in self._owned:
            if p.grad is not b:
                if p.grad is not None:
                    b.copy_(p.grad)
                p.grad = b

    def __call__(self, question_ids, sent_vecs):
        """The mean loss (0-dim fp32) of the questions `question_ids` (host ids, batch_size of them) with their
        sent_vecs [batch_size*nc, S] (device); `.backward()` replays the backward graph."""
        if not self.decoder.training:
            raise RuntimeError("SplitTrainStep replays the training forward: call decoder.train() first")
        if self._fwd is not None:
            self._check_replay()
            if [p.requires_grad for p in self.decoder.parameters()] != self._requires_grad:
                raise RuntimeError("SplitTrainStep: which decoder parameters require grad changed since capture; the "
                                   "backward graph accumulates the old set. Build a new SplitTrainStep.")
        self._load_ids(question_ids, sent_vecs)
        if self._fwd is None:
            self._sv = sent_vecs.detach().clone().requires_grad_(True)
            try:
                self._capture()  # on the micro-batch just loaded, which the host checks accepted
            except BaseException:
                self._sv = None
                raise
        self.calls += 1
        loss = _SplitTrainReplay.apply(self, self._anchor, sent_vecs)
        self._replayed()
        return loss


def packed_host_batch(adj, H, node_type, node_score, sent_vecs, adj_lengths):
    """The host-batch dict StreamedRunner(fields=DecoderStep.PACKED_FIELDS) uploads, from one batch of
    qagnn_b200.data.PackedAdjBatchGenerator (with device "cpu"): `adj` its PackedAdj, packed at an edge capacity so that
    every batch has the same shapes; node_type / node_score / adj_lengths its [bs, nc, ...] decoder tensors; H [bs*nc, n, D]
    and sent_vecs [bs*nc, S] the node features and sentence vectors of the same graphs.  Every tensor is pinned."""
    def pin(t):
        t = t.contiguous()
        return t if t.is_pinned() else t.pin_memory()
    n = H.size(1)
    return {"H": pin(H), "edge_index": pin(adj.edge_index), "edge_type": pin(adj.edge_type),
            "node_type": pin(node_type.reshape(-1, n)), "node_score": pin(node_score.reshape(-1, n, 1)),
            "sent_vecs": pin(sent_vecs), "adj_lengths": pin(adj_lengths.reshape(-1)), "graph_ptr": pin(adj.graph_ptr)}


class StreamedRunner:
    """Pinned host memory -> device -> pinned host memory, every batch, with copy/compute overlap across batches.

    `make_step(dev_inputs)` returns an object with `.run()` -> tuple of device tensors and `download` names which of them
    (by position) are copied back to the host; the default wraps a bare QAGNN_Message_Passing and downloads its
    [B,n,D] output."""

    FIELDS = ("H", "edge_index", "edge_type", "node_type", "node_score")

    def __init__(self, module, example, device, depth=2, make_step=None, fields=None, download=(0,)):
        """`example`: dict of pinned host tensors (keys `fields`) giving the shapes/dtypes of every batch."""
        self.module, self.device, self.depth = module, device, depth
        self.fields = tuple(fields) if fields is not None else self.FIELDS
        self.download = tuple(download)
        self.h2d, self.compute, self.d2h = (torch.cuda.Stream(device=device) for _ in range(3))
        self.dev = [{k: torch.empty_like(example[k], device=device) for k in self.fields} for _ in range(depth)]
        self.ev_up = [torch.cuda.Event() for _ in range(depth)]
        self.ev_done = [torch.cuda.Event() for _ in range(depth)]
        self.ev_down = [torch.cuda.Event() for _ in range(depth)]
        self.count = 0
        self.dev_out = [None] * depth   # device results of the last batch submitted to each slot
        self.host_out = [None] * depth  # pinned host copies of the downloaded results
        if make_step is None:
            class _Bare:
                def __init__(s, mod, d):
                    s.mod, s.d = mod, d

                def run(s):
                    return (s.mod(s.d["H"], (s.d["edge_index"], s.d["edge_type"]), s.d["node_type"], s.d["node_score"]),)
            make_step = lambda d: _Bare(module, d)  # noqa: E731
        for s in range(depth):  # the first upload also gives the capture valid indices to look at
            for k in self.fields:
                self.dev[s][k].copy_(example[k])
        self.steps = [make_step(self.dev[s]) for s in range(depth)]
        cur = torch.cuda.current_stream(device)
        for s in (self.h2d, self.compute, self.d2h):
            s.wait_stream(cur)

    def h2d_bytes(self):
        return sum(v.numel() * v.element_size() for v in self.dev[0].values())

    def d2h_bytes(self):
        return sum(t.numel() * t.element_size() for t in (self.host_out[0] or []))

    def submit(self, host_batch):
        """Enqueues one batch (dict of pinned host tensors); returns the slot whose `host_out` will hold the results
        once `ev_down[slot]` has completed (or after `drain()`)."""
        s = self.count % self.depth
        self.count += 1
        self.h2d.wait_event(self.ev_done[s])        # the previous batch in this slot no longer reads the inputs
        with torch.cuda.stream(self.h2d):
            for k in self.fields:
                self.dev[s][k].copy_(host_batch[k], non_blocking=True)
            self.ev_up[s].record(self.h2d)
        self.compute.wait_event(self.ev_up[s])
        self.compute.wait_event(self.ev_down[s])    # the slot's output buffers have been downloaded
        with torch.cuda.stream(self.compute):
            outs = self.steps[s].run()
            self.dev_out[s] = outs
            self.ev_done[s].record(self.compute)
        if self.host_out[s] is None:
            self.host_out[s] = [torch.empty(outs[i].shape, dtype=outs[i].dtype).pin_memory() for i in self.download]
        self.d2h.wait_event(self.ev_done[s])
        with torch.cuda.stream(self.d2h):
            for j, i in enumerate(self.download):
                self.host_out[s][j].copy_(outs[i], non_blocking=True)
            self.ev_down[s].record(self.d2h)
        return s

    def drain(self):
        cur = torch.cuda.current_stream(self.device)
        for s in (self.h2d, self.compute, self.d2h):
            cur.wait_stream(s)
