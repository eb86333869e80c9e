"""Times an optimiser batch whose micro-steps run concurrently on one GPU (pipeline.SplitTrainBatch) against the plain
SplitTrainStep loop, alternated in one process:

    python tools/bench_split_train_batch.py --out profiles/h100_split_train_batch.jsonl

Workload: tools/bench_split_train.py's loader-shaped synthetic split and decoder (n = 200, 38 relations, k = 5, D = 200,
sent_dim 1024, dropout 0.2) at the recipes' two shapes: -bs 64 -mbs 2 with 5 choices (CSQA) and -bs 128 -mbs 1 with 4
choices (OBQA), --loss cross_entropy, in fp16 autocast with a GradScaler, bf16 autocast and fp32.  The encoder is a stand-in:
each micro-batch's sent_vecs is a fixed random leaf, once requiring grad (encoder unfrozen) and once not (frozen).  An
optimiser batch is zero_grad, the micro-steps, GradScaler.unscale_, optim.clip_grad_norm_, the optim.RAdam step and the
scaler update; both loops run that same tail.

Per shape, precision and branches S in {1, 2, 4, 8, 16, 32} one line: wall ms per optimiser batch (each window of
--batches batches ends in a device synchronise) and host ms per optimiser batch (the enqueue loop before that
synchronise), medians and spreads over --reps windows, the SplitTrainBatch's windows alternated with the plain loop's on
another copy of the same decoder; peak device memory (max_memory_allocated) from building the SplitTrainBatch through its
windows; and, for the --profile-amps precisions, from a separate torch.profiler pass over one optimiser batch's micro-steps
with a device synchronise after every chunk, the sum of kernel time against the wall time of each chunk (its traced span,
and its device time between CUDA events in a pass without the profiler).  The gzip-compressed trace is written under
--trace-dir (default: --out's directory).  The card's name, power limit and largest SM clock are read in the same run."""
import argparse
import contextlib
import copy
import gzip
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_split_train import AMPS, N_CONCEPT, N_NODE, R, SENT_DIM, T, make_decoder  # noqa: E402
from bench_stream_split import gpu_info  # noqa: E402

SHAPES = {"bs64_mbs2_nc5": (64, 2, 5), "bs128_mbs1_nc4": (128, 1, 4)}
BRANCHES = (1, 2, 4, 8, 16, 32)


def make_split(n_q, nc, seed, dev):
    from qagnn_b200 import data as Dt
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_q * nc, seed=seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, nc)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), nc,
                           N_NODE)
    cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)
    labels = torch.from_numpy(np.random.default_rng(seed).integers(0, nc, n_q))
    return flat, Dt.DeviceSplit(flat, cids, ntypes, scores, lens, dev, T, R, labels=labels)


class Loop:
    """One decoder copy, its optimiser and scaler, run through a SplitTrainBatch (branches S) or the plain loop (None)."""

    def __init__(self, base, split, flat, mbs, amp, branches):
        from qagnn_b200 import optim
        from qagnn_b200.pipeline import SplitTrainBatch, SplitTrainStep
        self.dec = copy.deepcopy(base)
        kw = dict(edge_capacity=flat.max_batch_edges(mbs), max_edges=flat.max_graph_edges(), autocast_dtype=amp)
        self.mbs, self.branches = mbs, branches
        self.tb = SplitTrainBatch(self.dec, split, mbs, branches=branches, **kw) if branches else None
        self.step = None if branches else SplitTrainStep(self.dec, split, mbs, **kw)
        self.params = [p for p in self.dec.parameters() if p.requires_grad]
        self.opt = optim.RAdam(self.params, lr=1e-5)
        self.scaler = torch.amp.GradScaler("cuda") if amp == torch.float16 else None
        self.optim = optim

    def _backward(self, x):
        (self.scaler.scale(x) if self.scaler is not None else x).backward()

    def chunks(self, batch):
        from qagnn_b200.pipeline import train_chunks
        return train_chunks(batch, self.mbs, self.branches or 1)

    def chunk(self, chunk, svs, w):
        if self.tb is not None:
            self._backward((self.tb(chunk, svs) * w[:len(chunk)]).sum())
        else:
            for j, (q, sv) in enumerate(zip(chunk, svs)):
                self._backward(self.step(q, sv) * w[j])

    def micro_steps(self, batch, svs, w, around_chunk=None):
        self.opt.zero_grad()
        at = 0
        for c, chunk in enumerate(self.chunks(batch)):
            with around_chunk(c) if around_chunk is not None else contextlib.nullcontext():
                self.chunk(chunk, [svs[(at + j) % len(svs)] for j in range(len(chunk))], w)
            at += len(chunk)

    def batch(self, batch, svs, w):
        self.micro_steps(batch, svs, w)
        if self.scaler is not None:
            self.scaler.unscale_(self.opt)
        self.optim.clip_grad_norm_(self.params, 1.0)
        if self.scaler is not None:
            self.scaler.step(self.opt)
            self.scaler.update()
        else:
            self.opt.step()

    def window(self, batches, svs, w):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in batches:
            self.batch(b, svs, w)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / len(batches), (t1 - t0) / len(batches)


def chunk_overlap(loop, batch, svs, w, trace_path):
    """The micro-steps of one optimiser batch under torch.profiler, each chunk in a record_function range that ends in a
    device synchronise, so that every kernel of a chunk starts inside its range: per chunk, the sum of its kernels'
    durations and its span on the device, first kernel start to last kernel end (µs); and the chunk's device time between
two CUDA events in a pass without the profiler, whose tracing may serialise what runs concurrently without it."""
    from torch.profiler import ProfilerActivity, profile, record_function

    @contextlib.contextmanager
    def around(c):
        with record_function(f"chunk {c}"):
            yield
            torch.cuda.synchronize()

    walls = []

    @contextlib.contextmanager
    def timed(c):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        yield
        ev[1].record()
        walls.append(ev)

    loop.micro_steps(batch, svs, w, around_chunk=timed)  # the device time of every chunk without the profiler
    torch.cuda.synchronize()
    walls = [a.elapsed_time(b) * 1e3 for a, b in walls]
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        loop.micro_steps(batch, svs, w, around_chunk=around)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace_path)  # gzip-compressed, by its name
    with gzip.open(trace_path, "rt") as f:
        events = json.load(f)["traceEvents"]
    kernels = [(e["ts"], e["ts"] + e["dur"]) for e in events if e.get("cat") == "kernel"]
    ranges = sorted((e["ts"], e["ts"] + e["dur"]) for e in events
                    if e.get("cat") == "user_annotation" and str(e.get("name", "")).startswith("chunk "))
    out = []
    for (lo, hi), wall in zip(ranges, walls):
        g = [k for k in kernels if lo <= k[0] <= hi]
        ksum = sum(b - a for a, b in g)
        span = max(b for _, b in g) - min(a for a, _ in g)
        out.append({"kernels": len(g), "kernel_sum_us": ksum, "traced_span_us": span, "untraced_wall_us": wall,
                    "kernel_sum_over_untraced_wall": ksum / wall, "kernel_sum_over_traced_span": ksum / span})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=list(SHAPES), choices=list(SHAPES))
    ap.add_argument("--amps", nargs="+", default=list(AMPS), choices=list(AMPS))
    ap.add_argument("--branches", type=int, nargs="+", default=list(BRANCHES))
    ap.add_argument("--batches", type=int, default=2, help="optimiser batches per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None)
    ap.add_argument("--profile-amps", nargs="*", default=["fp16"], choices=list(AMPS),
                    help="precisions that get the profiler pass and its trace")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_split_train_batch.py: needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = gpu_info()
    trace_dir = args.trace_dir or os.path.dirname(os.path.abspath(args.out or "profiles/x"))
    os.makedirs(trace_dir, exist_ok=True)
    lines = []
    for shape in args.shapes:
        bs, mbs, nc = SHAPES[shape]
        n_q = 4 * bs
        flat, split = make_split(n_q, nc, args.seed, dev)
        perm = np.random.default_rng(args.seed).permutation(n_q)
        batches = [perm[a:a + bs] for a in range(0, n_q, bs)]
        M = bs // mbs
        w = torch.full((max(args.branches + [M]),), mbs / bs, device=dev)
        for amp_name in args.amps:
            amp = AMPS[amp_name]
            base = make_decoder(dev, 0.2)
            plain = Loop(base, split, flat, mbs, amp, None)
            for S in args.branches:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                before = torch.cuda.memory_allocated(dev)  # the split, the plain loop's decoder and graphs
                loop = Loop(base, split, flat, mbs, amp, S)
                res = {}
                for frozen in (False, True):
                    g = torch.Generator(device=dev).manual_seed(mbs)
                    svs = [torch.randn(mbs * nc, SENT_DIM, device=dev, generator=g).requires_grad_(not frozen)
                           for _ in range(8)]
                    for lp in (loop, plain):  # warm-up: capture, optimiser state
                        lp.window(batches[:1], svs, w)
                    t, tp = [], []
                    for r in range(args.reps):
                        t.append(loop.window(batches[r % 2 * 2:r % 2 * 2 + args.batches], svs, w))
                        tp.append(plain.window(batches[r % 2 * 2:r % 2 * 2 + args.batches], svs, w))
                    wall, host = [x[0] * 1e3 for x in t], [x[1] * 1e3 for x in t]
                    pwall, phost = [x[0] * 1e3 for x in tp], [x[1] * 1e3 for x in tp]
                    key = "sent_vecs_requires_grad" if not frozen else "sent_vecs_frozen"
                    res[key] = {"ms_per_optimiser_batch": statistics.median(wall), "spread_ms": [min(wall), max(wall)],
                                "host_ms_per_optimiser_batch": statistics.median(host),
                                "plain_ms_per_optimiser_batch": statistics.median(pwall),
                                "plain_spread_ms": [min(pwall), max(pwall)],
                                "plain_host_ms_per_optimiser_batch": statistics.median(phost),
                                "speedup_vs_plain": statistics.median(pwall) / statistics.median(wall)}
                peak = torch.cuda.max_memory_allocated(dev)
                profiled = None
                if amp_name in args.profile_amps:
                    trace = os.path.join(trace_dir, f"split_train_batch_{shape}_{amp_name}_S{S}.pt.trace.json.gz")
                    overlap = chunk_overlap(loop, batches[0], svs, w, trace)
                    profiled = {"trace": os.path.basename(trace), "n": len(overlap), "first": overlap[0],
                                **{"median_" + k: statistics.median(c[k] for c in overlap) for k in overlap[0] if k != "kernels"}}
                line = {"gpu": gpu, "shape": shape, "batch_size": bs, "micro_batch_size": mbs, "num_choice": nc,
                        "micro_batches": M, "autocast": amp_name, "loss": "cross_entropy", "n_node": N_NODE, "D": 200,
                        "k": 5, "dropout": 0.2, "branches": S, "chunks_per_batch": -(-M // S),
                        "batches_per_window": args.batches, "reps": args.reps, **res,
                        "peak_memory_allocated_bytes": peak, "memory_allocated_before_bytes": before,
                        "profiled_chunks": profiled}
                print(json.dumps(line), flush=True)
                lines.append(line)
                del loop
                torch.cuda.empty_cache()
            del plain, base
            torch.cuda.empty_cache()
        del split
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
