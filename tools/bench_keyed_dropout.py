"""Times keyed dropout (training.keyed_dropout, csrc/dropout.cu) against torch's dropout:

    python tools/bench_keyed_dropout.py --out profiles/h100_keyed_dropout.jsonl

Kernel lines: forward and backward of one site's layout at [64000, 200] elements (12.8 M), fp16 and fp32, keyed against
torch.native_dropout / native_dropout_backward: --iters calls captured in one CUDA graph after a warm-up, CUDA events
around its replay.  The layouts are the
node sites' [1, B, n D] (B = 320, n D = 40000), the graph-level sites' [1, B, F] (B = 64000, F = 200) and the pooler
attention's [n_head, B, n] (2, 32000, 200).  Bytes are counted from the shapes: x read and y written, plus the mask, which
is 1 bit per element for the keyed op and 1 byte (a bool) for torch's; the rate is reported against 3.35 TB/s.

Optimiser-batch lines: tools/bench_split_train.py's decoder and tools/bench_split_train_batch.py's split at -bs 64 -mbs 2
with 5 choices, fp16 autocast with a GradScaler, every dropout site at the recipe's rate (0.2, the pooler's 0.1), through
SplitTrainBatch at 8 branches and through the plain SplitTrainStep loop, each with a DropoutKey (advanced after every
optimiser step) and without one.  The four loops' windows of --batches optimiser batches alternate, each ending in a
device synchronise; medians and spreads over --reps windows.  The card's name, power limit and largest SM clock are read
in the same run."""
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

from bench_split_train import make_decoder  # noqa: E402
from bench_split_train_batch import make_split  # noqa: E402
from bench_stream_split import gpu_info  # noqa: E402

LAYOUTS = {"node [1, 320, 40000]": (1, 320, 40000, 0), "graph [1, 64000, 200]": (1, 64000, 200, 0),
           "pool_attn [2, 32000, 200]": (2, 32000, 200, 1)}
DTYPES = {"fp16": torch.float16, "fp32": torch.float32}


def _events_ms(fn, iters):
    """Device ms per call of fn: `iters` calls captured in one CUDA graph, so the host's per-call cost is not timed."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_lines(dev, iters, info):
    from qagnn_b200 import _lib, training
    p, nc = 0.2, 5
    out = []
    for lname, (A, G, L, gdim) in LAYOUTS.items():
        for dname, dt in DTYPES.items():
            shape = (G, L) if A == 1 else (A, G, L)
            n, es = A * G * L, torch.finfo(dt).bits // 8
            x = torch.randn(shape, device=dev, dtype=dt, requires_grad=True)
            dy = torch.randn(shape, device=dev, dtype=dt)
            key = training.DropoutKey(1, dev)
            qids = torch.arange(G // nc, device=dev)
            with training.keyed_dropout(key, qids, nc):
                y = training.dropout(x, p, True, training.SITE_FC_IN, graph_dim=gdim)

            def keyed_fwd():
                with training.keyed_dropout(key, qids, nc):
                    training.dropout(x.detach(), p, True, training.SITE_FC_IN, graph_dim=gdim)

            lib, mask_bits, dx = _lib.load(), y.grad_fn.saved_tensors[0], torch.empty_like(dy)

            def keyed_bwd():  # the entry _KeyedDropout.backward calls, without autograd's engine
                _lib.check(lib.qagnn_keyed_dropout_backward_typed(_lib.DTYPE_CODES[dt], n, p, _lib.ptr(mask_bits), _lib.ptr(dy),
                                                                  _lib.ptr(dx), _lib.stream_ptr(dev)), "keyed backward")

            _, mask = torch.native_dropout(x.detach(), p, True)

            def torch_fwd():
                torch.native_dropout(x.detach(), p, True)

            def torch_bwd():
                torch.ops.aten.native_dropout_backward(dy, mask, 1.0 / (1.0 - p))

            for impl, fwd, bwd, mask_bytes in (("keyed", keyed_fwd, keyed_bwd, n / 8), ("torch", torch_fwd, torch_bwd, n)):
                for pas, fn in (("forward", fwd), ("backward", bwd)):
                    ms = _events_ms(fn, iters)
                    nbytes = 2 * n * es + mask_bytes
                    rec = {"bench": "keyed_dropout_kernel", "layout": lname, "dtype": dname, "impl": impl, "pass": pas,
                           "elements": n, "p": p, "ms": round(ms, 4), "bytes": int(nbytes),
                           "tb_per_s": round(nbytes / ms / 1e9, 3), "of_3.35_tb_per_s": round(nbytes / ms / 1e9 / 3.35, 3),
                           "gpu": info}
                    print(json.dumps(rec), flush=True)
                    out.append(rec)
            del x, dy, y, mask, mask_bits, dx
    return out


class Loop:
    """One decoder copy trained at -mbs `mbs` through SplitTrainBatch (branches) or the plain loop (None), keyed or not."""

    def __init__(self, base, split, flat, mbs, branches, keyed, dev):
        from qagnn_b200 import optim, training
        from qagnn_b200.pipeline import SplitTrainBatch, SplitTrainStep
        self.dec = copy.deepcopy(base)
        self.key = training.DropoutKey(7, dev) if keyed else None
        kw = dict(edge_capacity=flat.max_batch_edges(mbs), max_edges=flat.max_graph_edges(), autocast_dtype=torch.float16,
                  dropout_key=self.key)
        self.mbs, self.branches = mbs, branches
        self.tb = SplitTrainBatch(self.dec, split, mbs, branches=branches, **kw) if branches else None
        self.step = None if branches else SplitTrainStep(self.dec, split, mbs, **kw)
        self.params = [p for p in self.dec.parameters() if p.requires_grad]
        self.opt = optim.RAdam(self.params, lr=1e-5)
        self.scaler = torch.amp.GradScaler("cuda")
        self.optim = optim

    def batch(self, batch, svs, w):
        from qagnn_b200.pipeline import train_chunks
        self.opt.zero_grad()
        at = 0
        for chunk in train_chunks(batch, self.mbs, self.branches or 1):
            cs = [svs[(at + j) % len(svs)] for j in range(len(chunk))]
            if self.tb is not None:
                self.scaler.scale((self.tb(chunk, cs) * w[:len(chunk)]).sum()).backward()
            else:
                for j, (q, sv) in enumerate(zip(chunk, cs)):
                    self.scaler.scale(self.step(q, sv) * w[j]).backward()
            at += len(chunk)
        self.scaler.unscale_(self.opt)
        self.optim.clip_grad_norm_(self.params, 1.0)
        self.scaler.step(self.opt)
        self.scaler.update()
        if self.key is not None:
            self.key.advance_()

    def window(self, batches, svs, w):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in batches:
            self.batch(b, svs, w)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / len(batches) * 1e3


def batch_lines(dev, n_batches, reps, seed, info):
    from bench_split_train import SENT_DIM
    bs, mbs, nc = 64, 2, 5
    n_q = bs * n_batches
    flat, split = make_split(n_q, nc, seed, dev)
    base = make_decoder(dev, 0.2)
    base.pooler.attn_dropout.p = base.pooler.dropout.p = 0.1
    order = np.random.default_rng(seed).permutation(n_q)
    batches = [order[i * bs:(i + 1) * bs] for i in range(n_batches)]
    g = torch.Generator(device=dev).manual_seed(seed)
    svs = [torch.randn(mbs * nc, SENT_DIM, device=dev, generator=g).requires_grad_(True) for _ in range(bs // mbs)]
    w = torch.full((8,), mbs / bs, device=dev)
    loops = {(route, keyed): Loop(base, split, flat, mbs, 8 if route == "batch8" else None, keyed, dev)
             for route in ("batch8", "plain") for keyed in (True, False)}
    for loop in loops.values():  # capture and warm up
        loop.window(batches[:1], svs, w)
    times = {k: [] for k in loops}
    for _ in range(reps):
        for k, loop in loops.items():
            times[k].append(loop.window(batches, svs, w))
    out = []
    for (route, keyed), t in times.items():
        rec = {"bench": "keyed_dropout_batch", "shape": "bs64_mbs2_nc5", "amp": "fp16",
               "route": "SplitTrainBatch(branches=8)" if route == "batch8" else "SplitTrainStep loop",
               "dropout": "keyed" if keyed else "torch", "ms_per_batch_median": round(statistics.median(t), 3),
               "ms_per_batch_min": round(min(t), 3), "ms_per_batch_max": round(max(t), 3), "windows": reps,
               "batches_per_window": n_batches, "gpu": info}
        print(json.dumps(rec), flush=True)
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--batches", type=int, default=4, help="optimiser batches per timed window")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--skip-batches", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyed_dropout: needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    info = gpu_info()
    recs = kernel_lines(dev, args.iters, info)
    if not args.skip_batches:
        recs += batch_lines(dev, args.batches, args.reps, args.seed, info)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in recs:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
