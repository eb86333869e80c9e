"""Times an optimiser batch replayed as one CUDA graph (pipeline.SplitTrainBatchGraph) against the eager composition it
replaces, SplitTrainBatch chunks + GradScaler backward + optim.CapturedTail + DropoutKey.advance_(), on two copies of one
decoder in one process, alternated:

    python tools/bench_batch_graph.py --out profiles/h100_batch_graph.jsonl

Workload: tools/bench_split_train.py's loader-shaped synthetic split and decoder (n = 200, 38 relations, k = 5, D = 200,
sent_dim 1024, dropout 0.2 with a DropoutKey) at the csqa recipe's -bs 64 -mbs 2 with 5 choices and 8 branches in fp16 and
bf16, and the obqa recipe's -bs 128 -mbs 1 with 4 choices and 32 branches in fp16; --loss cross_entropy, optim.RAdam,
clip 1.0, a frozen encoder (sent_vecs a fixed device tensor the graph side copies into its static buffer every batch).

Per configuration one line: host ms per optimiser batch (the enqueue loop of a window, before its device synchronise) and
wall ms per optimiser batch (through that synchronise), medians and spreads over --reps windows of --batches batches, both
sides alternated; the first step's host time (it trains its batch directly and captures), the graph's instantiation time,
its node count (top level, and every node of it and its child graphs), and the device memory the batch graph adds over the
SplitTrainBatch and tail it is built on (memory_allocated before and after its first step).  The card's name, power limit
and largest SM clock are read in the same run."""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_split_train import AMPS, SENT_DIM, make_decoder  # noqa: E402
from bench_split_train_batch import make_split  # noqa: E402
from bench_stream_split import gpu_info  # noqa: E402

# name: (batch size, micro-batch size, choices, branches, autocast)
CONFIGS = {"bs64_mbs2_nc5_S8_fp16": (64, 2, 5, 8, "fp16"), "bs64_mbs2_nc5_S8_bf16": (64, 2, 5, 8, "bf16"),
           "bs128_mbs1_nc4_S32_fp16": (128, 1, 4, 32, "fp16")}


class Side:
    """One decoder copy with its SplitTrainBatch, RAdam, scaler, CapturedTail and DropoutKey; `graph` adds the batch graph."""

    def __init__(self, base, split, mbs, S, amp, dev):
        from qagnn_b200 import optim
        from qagnn_b200.pipeline import SplitTrainBatch
        from qagnn_b200.training import DropoutKey
        self.dec = copy.deepcopy(base)
        self.key = DropoutKey(7, dev)
        self.tb = SplitTrainBatch(self.dec, split, mbs, branches=S, edge_capacity=split.max_batch_edges(mbs),
                                  max_edges=int(split.counts.max()), autocast_dtype=amp, dropout_key=self.key)
        self.params = [p for p in self.dec.parameters() if p.requires_grad]
        self.opt = optim.RAdam(self.params, lr=1e-5)
        self.scaler = torch.amp.GradScaler("cuda") if amp == torch.float16 else None
        self.tail = optim.CapturedTail(self.opt, self.scaler, None, 1.0, self.params)
        self.gb = None

    def eager(self, batch, sv, w):
        mbs, rows = self.tb.batch_size, self.tb.batch_size * self.tb.split.num_choice
        self.opt.zero_grad(set_to_none=True)
        j0 = 0
        for chunk in self.tb.chunks(batch):
            losses = self.tb(chunk, [sv[(j0 + j) * rows:(j0 + j + 1) * rows] for j in range(len(chunk))])
            x = (losses * w[:len(chunk)]).sum()
            (self.scaler.scale(x) if self.scaler is not None else x).backward()
            j0 += len(chunk)
        self.tail()
        self.key.advance_()

    def graph(self, batch, sv, w):
        self.gb.sent_vecs.copy_(sv)
        self.gb.step()

    def window(self, run, batches, sv, w):
        if self.gb is not None:
            self.gb.set_epoch(np.concatenate(batches))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in batches:
            run(b, sv, w)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / len(batches) * 1e3, (t1 - t0) / len(batches) * 1e3


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=list(CONFIGS), choices=list(CONFIGS))
    ap.add_argument("--batches", type=int, default=4, help="optimiser batches per timed window")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch_graph.py: needs a CUDA device")
    from qagnn_b200.pipeline import SplitTrainBatchGraph
    dev = torch.device("cuda:0")
    gpu = gpu_info()
    lines = []
    for name in args.configs:
        bs, mbs, nc, S, amp_name = CONFIGS[name]
        amp = AMPS[amp_name]
        n_q = args.batches * bs
        flat, split = make_split(n_q, nc, args.seed, dev)
        rng = np.random.default_rng(args.seed)
        base = make_decoder(dev, 0.2)
        sv = torch.randn(bs * nc, SENT_DIM, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        w = torch.full((S,), mbs / bs, device=dev)
        eager, graph = Side(base, split, mbs, S, amp, dev), Side(base, split, mbs, S, amp, dev)
        first = list(rng.permutation(n_q)[:bs].reshape(1, bs))
        eager.window(eager.eager, first, sv, w)  # captures the branches and the tail
        graph.window(graph.eager, first, sv, w)
        torch.cuda.synchronize()
        mem0 = torch.cuda.memory_allocated(dev)
        graph.gb = SplitTrainBatchGraph(graph.tb, bs, scaler=graph.scaler, tail=graph.tail)
        graph.gb.set_epoch(rng.permutation(n_q))  # the length every window's order has: no capture inside them
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.gb.step()  # trains this batch directly, then captures
        first_ms = (time.perf_counter() - t0) * 1e3
        torch.cuda.synchronize()
        extra = torch.cuda.memory_allocated(dev) - mem0
        host, wall, ehost, ewall = [], [], [], []
        for r in range(args.reps):
            batches = list(rng.permutation(n_q).reshape(args.batches, bs))
            for side, run, hs, ws in ((graph, graph.graph, host, wall), (eager, eager.eager, ehost, ewall)):
                wl, h = side.window(run, batches, sv, w)
                hs.append(h)
                ws.append(wl)
        line = {"gpu": gpu, "config": name, "batch_size": bs, "micro_batch_size": mbs, "num_choice": nc, "branches": S,
                "micro_batches": bs // mbs, "chunks_per_batch": -(-(bs // mbs) // S), "autocast": amp_name,
                "loss": "cross_entropy", "optimiser": "radam", "clip": 1.0, "dropout": 0.2, "encoder": "frozen",
                "batches_per_window": args.batches, "reps": args.reps,
                "graph_host_ms_per_batch": stats(host), "graph_wall_ms_per_batch": stats(wall),
                "eager_host_ms_per_batch": stats(ehost), "eager_wall_ms_per_batch": stats(ewall),
                "host_speedup": statistics.median(ehost) / statistics.median(host),
                "wall_speedup": statistics.median(ewall) / statistics.median(wall),
                "first_step_ms": first_ms, "instantiate_ms": graph.gb.instantiate_ms,
                "graph_nodes": graph.gb.node_count(), "graph_nodes_recursive": graph.gb.node_count(recursive=True),
                "extra_memory_bytes": extra}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del eager, graph, split
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
