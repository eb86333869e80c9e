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
"""
import torch

from . import distributed as _dist


class DecoderStep:
    """MP forward + pooling + (all-gather) + answer MLP on static device buffers, replayed as one CUDA graph.

    inputs (dict of device tensors, kept by reference): H [B,n,D], edge_index [2,E], edge_type [E], node_type [B,n],
    node_score [B,n,1], sent_vecs [B,S], adj_lengths [B].  Results (static buffers, overwritten by every run):
    `logits` [world*B, 1] (every rank holds all of them), `pool_attn` [n_head*B, n], `gnn_out` [B,n,D]."""

    FIELDS = ("H", "edge_index", "edge_type", "node_type", "node_score", "sent_vecs", "adj_lengths")
    PACKED_FIELDS = FIELDS + ("graph_ptr",)  # + first edge of every sub-graph, int64 [B + 1] (packed batches)

    def __init__(self, gnn, pooler, fc, inputs, world_size=1, group=None, use_cuda_graph=True, max_edges=-1):
        """`inputs` may carry "graph_ptr" (device int64 [B + 1]) with `max_edges` = an upper bound of the edges of one sub-graph
        for every batch that will be written into these buffers: graph prep is then ONE launch (qagnn_graph_prep_packed).
        edge_index / edge_type may then be an edge capacity K wider than any batch (qagnn_b200.data.PackedAdj): the real
        edge count is read from graph_ptr on the device, so one capture serves every batch of a split that fits K and
        `max_edges`.  A capture raises ValueError if the packed prep refuses the shape, since the general prep would freeze
        the edge count of the batch it was captured on."""
        self.gnn, self.pooler, self.fc = gnn, pooler, fc
        self.inp = {k: inputs[k] for k in self.FIELDS}
        self.adj = (self.inp["edge_index"], self.inp["edge_type"])
        if "graph_ptr" in inputs and max_edges >= 0:
            from .data import PackedAdj
            self.inp["graph_ptr"] = inputs["graph_ptr"]
            self.adj = PackedAdj(self.inp["edge_index"], self.inp["edge_type"], None, self.inp["H"].size(1), None,
                                 self.inp["graph_ptr"], int(max_edges), -1, self.inp["edge_index"].size(1))
        self.world, self.group = world_size, group
        dev = self.inp["H"].device
        B, n, D = self.inp["H"].shape
        S = self.inp["sent_vecs"].size(1)
        self.full = torch.empty(world_size * B, 2 * D + S, device=dev) if world_size > 1 else None
        self.graph = None
        self._status = None  # (device accumulator, pinned host copy) of graph prep's status word over the replays
        self._pending = None  # event after the last replay's copy of it
        self.logits = self.pool_attn = self.gnn_out = None
        self.mode = "eager"
        if use_cuda_graph:
            self._capture()

    @torch.no_grad()
    def _eager(self):
        d = self.inp
        out = self.gnn(d["H"], self.adj, d["node_type"], d["node_score"])
        fused = self.pooler.pool_concat(d["sent_vecs"], out, d["node_type"], d["adj_lengths"])  # :172-187 in one kernel
        if fused is not None:
            concat, pool_attn = fused
        else:
            n = out.size(1)
            pos = torch.arange(n, device=out.device)
            mask = (pos >= d["adj_lengths"].unsqueeze(1)) | (d["node_type"] == 3)        # modeling_qagnn.py:174-175
            mask[:, 0] = mask[:, 0] & ~mask.all(1)                                          # :176
            graph_vecs, pool_attn = self.pooler(d["sent_vecs"], out, mask)                  # :180
            concat = torch.cat((graph_vecs, d["sent_vecs"], out[:, 0]), 1)                  # :187 (dropout = identity in eval)
        full = _dist.all_gather_rows(concat, self.world, self.group, True, self.full)       # the path's one collective
        return self.fc(full), pool_attn, out                                                # :188

    def _capture(self):
        dev = self.inp["H"].device
        saved = self.gnn.use_cuda_graph
        self.gnn.use_cuda_graph = False  # its kernels become nodes of THIS graph
        check, self.gnn.check_indices = self.gnn.check_indices, False
        try:
            if check:  # validate once, eagerly (a synchronising call), before trusting the capture
                self.gnn.check_indices = True
                self.gnn.check_batch(self.adj, self.inp["node_type"])
                self.gnn.check_indices = False
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(2):  # warm-up: folds the weights, sizes the workspaces, opens the NCCL channels
                    self._eager()
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            if "graph_ptr" in self.inp and not self.gnn._last_prep.packed:
                raise ValueError("DecoderStep: the packed graph prep refuses these sub-graphs (too large for one CTA); a "
                                 "captured general prep would keep the edge count of this batch for every later one")
            # batches written into the buffers later are validated without a sync: every replay ORs graph prep's status
            # word into a device accumulator and copies it to pinned memory, which run() looks at once it has landed
            status = (torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32).pin_memory())
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self.logits, self.pool_attn, self.gnn_out = self._eager()
                if check:
                    status[0].bitwise_or_(self.gnn._last_prep.status_word())
                    status[1].copy_(status[0], non_blocking=True)
            self.graph = graph
            if check:
                self._status = status
            self._keep = (self.gnn._ws.buf, self.gnn._folded.blob, self.gnn._last_prep)  # addresses baked into the graph
            self.mode = "one CUDA graph (prep + k layers + pooling" + (" + all-gather" if self.world > 1 else "") + " + fc)"
        finally:
            self.gnn.use_cuda_graph, self.gnn.check_indices = saved, check

    def run(self):
        """Enqueues one step on the current stream; returns (logits, pool_attn, gnn_out).  A replay whose batch had an
        index out of range (or an edge crossing its sub-graph) raises IndexError at a later call, once the copy of the
        status word has landed; its results were computed from clamped indices."""
        if self.graph is not None:
            self._raise_status()
            self.graph.replay()
            if self._status is not None:
                self._pending = torch.cuda.Event()
                self._pending.record()
        else:
            self.logits, self.pool_attn, self.gnn_out = self._eager()
        return self.logits, self.pool_attn, self.gnn_out

    def _raise_status(self):
        if self._pending is None or not self._pending.query():  # never blocks: the accumulated word is looked at later
            return
        self._pending = None
        accum, host = self._status
        if int(host.item()) != 0:
            bits = int(host.item())
            accum.zero_()
            host.zero_()
            raise IndexError("qagnn_b200: a DecoderStep replay saw edge_index / edge_type / node_type values out of range or "
                             f"crossing a sub-graph boundary (status bits {bits}); its results were computed from clamped indices")


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
