"""Data-parallel use of the path across the GPUs of one box (SURVEY.md §8e).

Sub-graphs are independent (LM_QAGNN.batch_graph only offsets node ids, modeling_qagnn.py:244-251), weights are
tiny and replicated, so the (question, all-choices) groups are sharded across ranks with no collective inside the k
GNN layers.  The single exchange is an all-gather of the pooled features right before the answer MLP
(modeling_qagnn.py:187-188): every rank ends up with the logits of the whole batch.
"""
import contextlib
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .training import answer_loss, keyed_dropout


def shard_bounds(n_questions, rank, world_size):
    """Contiguous block of whole questions for `rank` (all choices of a question stay together)."""
    per = (n_questions + world_size - 1) // world_size
    lo = min(rank * per, n_questions)
    return lo, min(lo + per, n_questions)


def shard_batch(inputs, rank, world_size):
    """Slices an LM_QAGNN-style positional input tuple (tensors with a leading batch dim + the two nested
    [batch][num_choice] adjacency lists at the end) down to this rank's questions."""
    *tensors, edge_index, edge_type = inputs
    lo, hi = shard_bounds(tensors[0].size(0), rank, world_size)
    return tuple(t[lo:hi] for t in tensors) + (edge_index[lo:hi], edge_type[lo:hi]), (lo, hi)


def all_gather_rows(local, world_size, group=None, equal_shards=True, out=None):
    """The path's ONE collective: all-gather of the ranks' row blocks [B_r, F] -> [sum B_r, F].

    equal_shards=True (how `shard_bounds` cuts a batch whose question count divides by the world size, and cfg4 of
    BASELINE.json): a single `all_gather_into_tensor`, no size exchange, no host synchronisation — capturable in a CUDA
    graph.  `out` optionally names the [world_size * B_r, F] result buffer (static address for graph replay).
    equal_shards=False: blocks may differ in length (a short last shard): sizes are exchanged first, then padded blocks."""
    if world_size == 1:
        return local
    if equal_shards:
        if out is None:
            out = local.new_empty((world_size * local.size(0),) + tuple(local.shape[1:]))
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    n = torch.tensor([local.size(0)], device=local.device, dtype=torch.long)
    sizes = [torch.zeros_like(n) for _ in range(world_size)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s) for s in sizes]
    mx = max(sizes)
    pad = local.new_zeros((mx,) + tuple(local.shape[1:]))
    pad[: local.size(0)] = local
    out = [torch.empty_like(pad) for _ in range(world_size)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[:s] for o, s in zip(out, sizes)], dim=0)


def decoder_forward_sharded(decoder, sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj, world_size,
                            group=None, equal_shards=True):
    """QAGNN.forward on this rank's shard + all-gather of the pooled features + the answer MLP on the full batch
    (modeling_qagnn.py:172-188).  Returns (logits of ALL graphs [B_total, 1], local pool_attn)."""
    concat, pool_attn = decoder.pooled_features(sent_vecs, concept_ids, node_type_ids, node_scores, adj_lengths, adj)
    full = all_gather_rows(concat, world_size, group, equal_shards)
    return decoder.fc(full), pool_attn


def bind_to_gpu_numa_node(device_index):
    """Pins this process (and the pinned host buffers it allocates afterwards, by first touch) to the CPUs of the NUMA node
    the GPU hangs off.  8 ranks streaming ~110 MB per step through pinned memory otherwise cross the socket interconnect
    for half of the GPUs (SCALE_r01: e2e efficiency 0.74 at N=8 with device-side efficiency 0.97).  Returns the node or None."""
    import os
    try:
        props = torch.cuda.get_device_properties(device_index)
        bus = f"{props.pci_domain_id:04x}:{props.pci_bus_id:02x}:{props.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bus}/numa_node").read())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return node
    except Exception:  # noqa: BLE001 - affinity is an optimisation, never a failure
        return None


# ---- data-parallel training of a split (INTEGRATION §3) ------------------------------------------------------------------

def slot_columns(numels):
    """(cols, ld): the column of each tensor's first element in a gradient-slot row and the row length, for tensors of
    `numels` elements packed in order, each starting on a 16-byte boundary so that the ordered sum reads float4."""
    cols, c = [], 0
    for n in numels:
        cols.append(c)
        c += (int(n) + 3) // 4 * 4
    return cols, max(c, 4)


def ordered_grad_sum_(grads, slots, n_valid, init_from_grad):
    """The ordered sum of per-micro-batch gradients into `grads`, in place, in one sm_90a launch per 512 tensors
    (csrc/grad_reduce.cu).  `grads`: contiguous fp32 CUDA tensors of one device; `slots`: fp32 [S, ld] on that device with unit
    column stride, row j holding micro-batch j's gradients laid out by `slot_columns([g.numel() for g in grads])`;
    `init_from_grad`: one bool, or one per tensor.  Per element, each add one fp32 add rounded to nearest:

        g = g + slots[0] if init_from_grad else slots[0];   g = g + slots[j] for j = 1 ... n_valid - 1

    That is what accumulating the micro-batches into `.grad` one after another does, so the result is that loop's bit for bit,
    whatever the grid.  Rows at or past `n_valid` are not read.  Nothing is read on the host."""
    grads = list(grads)
    if not grads:
        return
    n_valid = int(n_valid)
    if isinstance(init_from_grad, bool):
        init_from_grad = [init_from_grad] * len(grads)
    init_from_grad = [bool(x) for x in init_from_grad]
    if len(init_from_grad) != len(grads):
        raise ValueError(f"ordered_grad_sum_: {len(init_from_grad)} init_from_grad flags for {len(grads)} tensors")
    if not slots.is_cuda or slots.dtype != torch.float32 or slots.dim() != 2 or (slots.size(1) > 1 and slots.stride(1) != 1):
        raise ValueError(f"ordered_grad_sum_: slots must be a 2-D fp32 CUDA tensor with unit column stride, got "
                         f"{tuple(slots.shape)} {slots.dtype} on {slots.device}")
    if not 1 <= n_valid <= slots.size(0):
        raise ValueError(f"ordered_grad_sum_: n_valid = {n_valid}, slots has {slots.size(0)} rows")
    cols, ld = slot_columns([g.numel() for g in grads])
    if slots.size(1) < ld:
        raise ValueError(f"ordered_grad_sum_: slot rows of {slots.size(1)} elements, the gradients need {ld}")
    for g in grads:
        if g.device != slots.device or g.dtype != torch.float32 or not g.is_contiguous():
            raise ValueError(f"ordered_grad_sum_: every gradient must be a contiguous fp32 tensor on {slots.device}, got "
                             f"{g.dtype} on {g.device}")
    lib = _lib.load()
    n = len(grads)
    with torch.cuda.device(slots.device):
        _lib.check(lib.qagnn_ordered_grad_sum(
            n, (C.c_void_p * n)(*[g.data_ptr() for g in grads]), (C.c_int64 * n)(*[g.numel() for g in grads]),
            (C.c_int64 * n)(*cols), (C.c_int32 * n)(*init_from_grad), _lib.ptr(slots), slots.stride(0), n_valid,
            _lib.stream_ptr(slots.device)), "qagnn_ordered_grad_sum")


class GradSlots:
    """Micro-batch j's gradients of the fp32 `tensors` in row j of `slots` [rows, >= ld], laid out by slot_columns (ld its
    row length), and their ordered sum onto the tensors' `.grad`; `flat` [>= ld] takes the sums that start from no tensor of
    the caller's.  The caller allocates both.  `rows[j]` and `own` are row j and `flat` as views shaped like the tensors."""

    def __init__(self, tensors, slots, flat):
        self.tensors, self.slots = list(tensors), slots
        self.cols = slot_columns([t.numel() for t in self.tensors])[0]
        self.rows = [self._views(row) for row in slots]
        self.own = self._views(flat)

    def _views(self, flat):
        return [flat[c:c + t.numel()].view_as(t) for t, c in zip(self.tensors, self.cols)]

    def copy_row_(self, j, grads):
        """Copies `grads`, one per tensor, into row j; None counts as zeros."""
        dst = self.rows[j]
        if grads and all(g is not None for g in grads):
            torch._foreach_copy_(dst, list(grads))
        else:
            for d, g in zip(dst, grads):
                d.zero_() if g is None else d.copy_(g)

    def sum_(self, starts, n_valid):
        """ordered_grad_sum_ of rows 0 ... n_valid - 1 onto `starts`, one per tensor, and each tensor's `.grad` the sum: a start
        of None sums into `own`, a non-contiguous one is first copied there, a contiguous one is added onto in place."""
        sums = []
        for s, own in zip(starts, self.own):
            if s is not None and not s.is_contiguous():
                own.copy_(s)
            sums.append(s if s is not None and s.is_contiguous() else own)
        ordered_grad_sum_(sums, self.slots, n_valid, [s is not None for s in starts])
        for t, s in zip(self.tensors, sums):
            t.grad = s


def fold_running_stats(start, ends, counts, momentum):
    """The running statistics one process would hold after W ranks' BatchNorm updates in rank order, from each rank's own:
    `start` [L] the common starting values R_0, `ends` [W, L] rank r's values R_r after `counts` [W, L] updates of its own from
    R_0, `momentum` a float or [L].  With a = 1 - momentum, N the total count and N_after_r the count on later ranks:

        a^N R_0 + sum_r a^N_after_r (R_r - a^n_r R_0)

    in fp64 (the inputs are widened), which is exact in exact arithmetic because every update is R <- a R + momentum x."""
    start, ends, counts = start.double(), ends.double(), counts.double()
    a = 1.0 - (momentum.double() if torch.is_tensor(momentum) else float(momentum))
    a = torch.as_tensor(a, dtype=torch.float64, device=start.device)
    total = counts.sum(0)
    after = total - counts.cumsum(0)
    return torch.pow(a, total) * start + (torch.pow(a, after) * (ends - torch.pow(a, counts) * start)).sum(0)


class BatchNormFold:
    """The running statistics of `decoder`'s BatchNorms that track them, read as one flat [mean_0, var_0, mean_1, var_1, ...]
    vector of L elements and T num_batches_tracked counts, and folded into the live buffers from copies that several branches
    or ranks (`across`) updated on their own.  Raises ValueError, naming the caller `what`, for a BatchNorm with momentum=None."""

    def __init__(self, decoder, what, across):
        self.bns = [m for m in decoder.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)
                    and m.track_running_stats]
        if any(m.momentum is None for m in self.bns):
            raise ValueError(f"{what}: a BatchNorm with momentum=None (a cumulative average) cannot be folded across {across}")
        self.live = [t for m in self.bns for t in (m.running_mean, m.running_var)]
        self.live_counts = [m.num_batches_tracked for m in self.bns]
        self.sizes = [t.numel() for t in self.live]
        dev = self.live[0].device if self.live else None
        owner = [i for i, m in enumerate(self.bns) for _ in range(2 * m.running_mean.numel())]
        self._owner = torch.tensor(owner, dtype=torch.int64, device=dev)
        self._momentum = torch.tensor([float(self.bns[i].momentum) for i in owner], dtype=torch.float64, device=dev)

    def read(self, stats=None, counts=None):
        """(the flat statistics [L], num_batches_tracked [T]) of the live buffers, written into `stats` / `counts` if given."""
        return torch.cat(self.live, out=stats), torch.stack(self.live_counts, out=counts)

    def fold_(self, start, ends):
        """The live buffers after the updates of every row of `ends` (stats [W, L], counts [W, T]), in row order, each row's
        from `start` (stats [L], counts [T], as read() returns them): fold_running_stats in fp64, rounded once, and
        num_batches_tracked the start count plus the exact sum of the rows' counts."""
        (stats, counts), (end_stats, end_counts) = start, ends
        n = end_counts - counts
        with torch.no_grad():
            folded = fold_running_stats(stats, end_stats, n.index_select(1, self._owner), self._momentum)
            torch._foreach_copy_(self.live, list(folded.to(stats.dtype).split(self.sizes)))
            torch._foreach_copy_(self.live_counts, list((counts + n.sum(0).to(counts.dtype)).unbind(0)))

    @contextlib.contextmanager
    def pointing_at(self, stats, counts):
        """The modules' buffers pointing at `stats` [L] and `counts` [T] (rows of a [rows, L] / [rows, T] pair) in the block."""
        self._point(stats.split(self.sizes), counts)
        try:
            yield
        finally:
            self._point(self.live, self.live_counts)

    def _point(self, stats, counts):
        for i, m in enumerate(self.bns):
            m.running_mean, m.running_var, m.num_batches_tracked = stats[2 * i], stats[2 * i + 1], counts[i]


class DataParallelSplitTrain:
    """Data-parallel training of a split held on the GPU across the ranks of one box, equal to the one-GPU loop.

    Every rank holds the whole split (its own DeviceSplit), the same model and the same SplitTrainStep over
    `micro_batch_size` questions, and walks the same permutation.  An optimiser batch of n questions splits into
    M = ceil(n / micro_batch_size) micro-batches in order, the last one possibly partial; rank r runs the contiguous block
    [r m, min(M, (r + 1) m)), m = ceil(M / W), which `micro_batches(batch)` returns.  A rank may get none in a short final
    batch.  `reduce_(n)` then leaves every rank with what one GPU holds after all M micro-batches:

    - the decoder's `.grad`, bit for bit: `micro_step()` gives each micro-batch's gradient its own row of a gradient-slot
      buffer, one all_gather_into_tensor collects the [W m, P] rows, and ordered_grad_sum_ adds them in micro-batch order,
      onto `.grad` when it was not None before the batch.  A decoder parameter no micro-step reaches keeps `.grad` None;
    - the gradients of `other_params` (the text encoder), accumulated locally as usual: summed by reduce_scatter_tensor and
      all_gather_into_tensor of one fp32 bucket, so each sum is formed on one rank and every rank holds the same bits.  They
      are sums in another order than one GPU's, equal to within fp32 summation error.  Which of them require grad is read
      per batch (freeze_net / unfreeze_net may change it between batches): one that does not is left alone, and one the loss
      does not reach keeps `.grad` None.  The reached set is exchanged on the host once per requires-grad pattern; it is the
      same for every micro-batch, and rank 0 always runs one, so a reached parameter is reached on some rank in every batch;
    - the decoder's BatchNorm running statistics: fold_running_stats of every rank's, in fp64 from one small all-gather,
      rounded once to fp32, and num_batches_tracked summed exactly.  One GPU rounds after every update instead, so the
      statistics agree to within the rounding of the updates, not bit for bit.

    The recipe's tail (GradScaler.unscale_, clip_grad_norm_, the scheduler and optimiser steps) then runs unchanged on every
    rank and takes the same step.  That step is the one-GPU step bit for bit when the encoder is frozen or the clip's norm
    leaves its gradients out; otherwise the encoder's sums can move the clip coefficient in its last bits.  Dropout: with the
    step's `dropout_key` (training.DropoutKey, the same seed on every rank) every micro-batch, the eager partial one in
    `loss()` included, draws the masks one GPU draws for its questions, and the above holds at any dropout; advance the key
    on every rank once per optimiser batch, after the optimiser step.  Without a key each rank seeds its own dropout stream,
    so the ranks draw other masks than one GPU would: the run is then the one-GPU run in distribution, not bit for bit.  With
    one rank (W = 1, no process group) the reduction is the ordered sum of the local rows and nothing else changes.

    Construction raises ValueError when step.batch_size is not `micro_batch_size`, when `batch_size` is less than it, when a
    full batch would leave a rank without a micro-batch or start a rank's block with the partial micro-batch (every rank
    captures its step on the first batch, which must be full), and for a BatchNorm with momentum=None."""

    def __init__(self, step, split, batch_size, micro_batch_size, other_params=(), group=None):
        self.step, self.split, self.group = step, split, group
        self.batch_size, self.micro_batch_size = int(batch_size), int(micro_batch_size)
        if dist.is_available() and dist.is_initialized():
            self.world_size, self.rank = dist.get_world_size(group), dist.get_rank(group)
        else:
            self.world_size, self.rank = 1, 0
        W, mbs = self.world_size, self.micro_batch_size
        if step.batch_size != mbs or step.split is not split:
            raise ValueError(f"DataParallelSplitTrain: the step runs {step.batch_size} questions of its own split, the loop "
                             f"{mbs} of this one")
        if self.batch_size < mbs:
            raise ValueError(f"DataParallelSplitTrain: batch_size {self.batch_size} < micro_batch_size {mbs}")
        M = -(-self.batch_size // mbs)
        for r in range(W):
            lo, hi = shard_bounds(M, r, W)
            if hi == lo or (lo == M - 1 and self.batch_size % mbs):
                raise ValueError(f"DataParallelSplitTrain: a full batch of {M} micro-batches leaves rank {r} of {W} "
                                 f"{'none' if hi == lo else 'only the partial one'}; every rank must capture its step on a "
                                 f"full micro-batch of the first batch")
        self._bn = BatchNormFold(step.decoder, "DataParallelSplitTrain", "ranks")
        self._params = [p for p in step.decoder.parameters() if p.requires_grad]
        self._other = list(other_params)
        self._reached = None       # indices into self._params the step's capture reaches, in order
        self._grad_slots = None         # the reached parameters' GradSlots
        self._other_pattern = None  # the requires-grad flags of self._other that self._other_reached was exchanged for
        self._other_reached = None  # indices into self._other the loss reaches under that pattern
        self._batch = None         # (n, M, m, first row, count) between micro_batches() and reduce_()

    # -- the loop -------------------------------------------------------------------------------------------------------

    def micro_batches(self, batch):
        """This rank's micro-batches of the optimiser batch `batch` (host question ids), in order; starts the batch."""
        if self._batch is not None:
            raise RuntimeError("DataParallelSplitTrain: micro_batches() again before reduce_() of the last batch")
        batch = np.asarray(batch)
        n, mbs, W = len(batch), self.micro_batch_size, self.world_size
        if not 1 <= n <= self.batch_size:
            raise ValueError(f"DataParallelSplitTrain: a batch of {n} questions; the loop takes 1 to {self.batch_size}")
        M = -(-n // mbs)
        lo, hi = shard_bounds(M, self.rank, W)
        self._batch = (n, M, -(-M // W), lo, hi - lo)
        self._done = 0
        # .grad from before the batch: the decoder's adds on top of it in order; the other parameters' after the sum
        own = {id(g) for g in self._grad_slots.own} if self._grad_slots is not None else set()
        self._before = [g if g is None or id(g) in own else g.detach().clone() for g in (p.grad for p in self._params)]
        self._pattern = tuple(p.requires_grad for p in self._other)
        self._trainable = [i for i, t in enumerate(self._pattern) if t]
        self._other_before = {i: self._other[i].grad for i in self._trainable}
        for p in self._params:
            p.grad = None
        for i in self._trainable:
            self._other[i].grad = None
        self._bn_start = self._bn.read() if W > 1 and self._bn.bns else None
        return [batch[j * mbs:(j + 1) * mbs] for j in range(lo, hi)]

    @contextlib.contextmanager
    def micro_step(self):
        """Around one micro-batch's loss and backward: the decoder's `.grad` it leaves goes to the micro-batch's slot row."""
        if self._batch is None or self._done == self._batch[4]:
            raise RuntimeError("DataParallelSplitTrain: micro_step() outside this rank's micro-batches of a batch")
        for p in self._params:
            p.grad = None
        yield
        if self._reached is None:
            self._set_layout()
        if any(self._params[i].grad is not None for i in self._unreached):
            raise RuntimeError("DataParallelSplitTrain: a micro-step reached decoder parameters its step's capture does not")
        self._grad_slots.copy_row_(self._batch[2] * self.rank + self._done, [p.grad for p in self._grad_slots.tensors])
        self._done += 1

    def loss(self, question_ids, sent_vecs):
        """The micro-batch's mean loss: the step's for a full micro-batch, else the eager decoder and answer loss of the
        same autocast and dropout key, as the one-GPU loop runs its partial micro-batch."""
        step = self.step
        if len(question_ids) == step.batch_size:
            return step(question_ids, sent_vecs)
        from .pipeline import _autocast
        q = torch.from_numpy(np.asarray(question_ids, dtype=np.int64)).to(self.split.device)
        keyed = (contextlib.nullcontext() if step.dropout_key is None
                 else keyed_dropout(step.dropout_key, q, self.split.num_choice))
        with _autocast(step.autocast_dtype), keyed:
            logits, _ = step.decoder(sent_vecs, *self.split.batch(question_ids, step.edge_capacity))
            return answer_loss(logits, self.split.labels[q], self.split.num_choice, step.loss)

    def reduce_(self, batch_len):
        """After this rank's last micro-step of the batch: every rank's `.grad` and BatchNorm statistics become one GPU's.
        Collective: every rank calls it for every batch.  No host read, except that the first call, and the first call after
        the requires-grad pattern of `other_params` changed, exchange which parameters the loss reaches."""
        if self._batch is None or int(batch_len) != self._batch[0]:
            raise ValueError(f"DataParallelSplitTrain: reduce_({int(batch_len)}) for a batch of "
                             f"{None if self._batch is None else self._batch[0]} questions")
        if self._done != self._batch[4]:
            raise RuntimeError(f"DataParallelSplitTrain: reduce_() after {self._done} of this rank's {self._batch[4]} "
                               f"micro-steps")
        if self._reached is None:
            raise RuntimeError("DataParallelSplitTrain: no micro-step has run yet; the first batch must be full")
        if self._pattern != self._other_pattern:
            self._exchange_reached()
        self._gather_slots()
        self._sum_slots()
        local = self._reduce_other()
        self._fold_bn()
        ran = self._batch[4] > 0
        self._batch = None
        if ran and local != self._other_reached:  # after the collectives, so that the other ranks are not left waiting
            raise RuntimeError("DataParallelSplitTrain: this batch's loss reached other parameters than the first batch under "
                               "the same requires-grad pattern did; the set must not depend on the micro-batch")

    # -- the parts of reduce_ -------------------------------------------------------------------------------------------

    def _gather_slots(self):
        if self.world_size > 1:
            m = self._batch[2]
            rows = self._grad_slots.slots[:self.world_size * m]
            dist.all_gather_into_tensor(rows, rows[self.rank * m:(self.rank + 1) * m], group=self.group)

    def _sum_slots(self):
        self._grad_slots.sum_([self._before[i] for i in self._reached], self._batch[1])
        for i in self._unreached:
            self._params[i].grad = self._before[i]

    def _reduce_other(self):
        """Sums the reached other parameters' .grad over the ranks; returns the ones this rank reached."""
        local = [i for i in self._trainable if self._other[i].grad is not None]
        idx = self._other_reached
        params = [self._other[i] for i in idx]
        if self.world_size == 1:
            sums = [p.grad for p in params]
        else:
            W = self.world_size
            n = sum(p.numel() for p in params)
            n = -(-max(n, 1) // W) * W
            bucket = torch.zeros(n, dtype=torch.float32, device=self.split.device)
            views, off = [], 0
            for p in params:
                views.append(bucket[off:off + p.numel()].view_as(p))
                off += p.numel()
            have = [(v, p.grad) for v, p in zip(views, params) if p.grad is not None]
            if have:
                torch._foreach_copy_([v for v, _ in have], [g for _, g in have])
            part = torch.empty(n // W, dtype=torch.float32, device=bucket.device)
            dist.reduce_scatter_tensor(part, bucket, op=dist.ReduceOp.SUM, group=self.group)
            dist.all_gather_into_tensor(bucket, part, group=self.group)
            sums = [v if v.dtype == p.dtype else v.to(p.dtype) for v, p in zip(views, params)]
        for i, s in zip(idx, sums):
            before = self._other_before[i]
            if before is not None and s is not None:
                before.add_(s)
            self._other[i].grad = before if before is not None else s
        for i in set(self._trainable) - set(idx):
            self._other[i].grad = self._other_before[i]
        return local

    def _fold_bn(self):
        if self.world_size == 1 or not self._bn.bns:
            return
        stats, counts = self._bn.read()
        mine = torch.cat([stats.double(), counts.double()])
        every = torch.empty(self.world_size * mine.numel(), dtype=torch.float64, device=mine.device)
        dist.all_gather_into_tensor(every, mine, group=self.group)
        every = every.view(self.world_size, -1)
        self._bn.fold_(self._bn_start, (every[:, :stats.numel()], every[:, stats.numel():]))

    # -- helpers --------------------------------------------------------------------------------------------------------

    def _set_layout(self):
        """The decoder parameters the step's capture reaches and their gradient slots, the rows of a full batch."""
        step = self.step
        if step._fwd is None:
            raise RuntimeError("DataParallelSplitTrain: the first micro-step ran eagerly; the first batch must be full")
        where = {id(p): i for i, p in enumerate(self._params)}
        self._reached = sorted(where[id(p)] for p, _ in step._owned)
        self._unreached = sorted(set(range(len(self._params))) - set(self._reached))
        reached = [self._params[i] for i in self._reached]
        ld = slot_columns([p.numel() for p in reached])[1]
        full = -(-self.batch_size // self.micro_batch_size)
        m = -(-full // self.world_size)
        dev = self.split.device
        self._grad_slots = GradSlots(reached, torch.empty(self.world_size * m, ld, dtype=torch.float32, device=dev),
                                torch.empty(ld, dtype=torch.float32, device=dev))

    def _exchange_reached(self):
        """Once per requires-grad pattern of other_params: every rank's reached decoder parameters must agree; the other
        parameters reached on any rank are kept."""
        mine = (self._reached, [i for i in self._trainable if self._other[i].grad is not None])
        every = [mine]
        if self.world_size > 1:
            every = [None] * self.world_size
            dist.all_gather_object(every, mine, group=self.group)
        if any(e[0] != mine[0] for e in every):
            raise RuntimeError("DataParallelSplitTrain: the ranks' steps reach different decoder parameters")
        self._other_reached = sorted(set().union(*(e[1] for e in every)))
        self._other_pattern = self._pattern
