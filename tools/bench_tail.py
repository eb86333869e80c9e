"""Times the recipe's optimiser tail two ways, alternated in one process, with --optim radam (the default), adamw, adam or
sgd (qagnn_b200.optim.DEVICE_OPTIMIZER_CLASSES, constructed as the reference constructs them):

  eager     scaler.unscale_(opt); qagnn_b200.optim.clip_grad_norm_(params, max_norm); scheduler.step(); scaler.step(opt);
            scaler.update(), with qagnn_b200.optim's optimiser
  captured  qagnn_b200.optim.CapturedTail: one graph replay of two launches

Cases:
  decoder   the decoder's trainable tensors (k = 5, D = 200, sent_dim 1024), fp16 with a GradScaler, clipping at 1.0
  encoder   a RoBERTa-large-shaped set plus the decoder, fp16, at a max_norm that clips (half the norm) and with no clip
            (max_grad_norm 0, so no unscale_ either)
  batch     one optimiser batch of 64 questions at -mbs 2 under fp16 autocast through SplitTrainBatch(branches=8), then
            each tail
Each line: wall ms (ending in a synchronise), host ms (the enqueue before it), launches and synchronisations from a
torch.profiler pass of its own, and, for the tensor sets, the kernels' summed device time with its share of 3.35 TB/s at
the bytes each route moves per parameter (traffic()).  Medians with the spread (min, max) over --reps repetitions.

    python tools/bench_tail.py --out profiles/h100_tail.jsonl
    python tools/bench_tail.py --optim adamw --out profiles/h100_tail.jsonl --append
    python tools/bench_tail.py --optim sgd --cases decoder encoder --out profiles/h100_optim_sgd.jsonl --append
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_optim import HBM_TBS, kernel_ms, profile_counts, recipe_groups, roberta_large_shapes, stats  # noqa: E402
from bench_split_train import N_CONCEPT, N_NODE, NC, R, SENT_DIM, T, make_decoder  # noqa: E402
from bench_stream_split import gpu_info  # noqa: E402

ROUTES = ("eager", "captured")


def traffic(route, clip, scaler, optim="radam"):
    """Compulsory bytes per fp32 parameter of one tail, from shapes alone.  The step alone reads g, p, m, v and writes p, m,
    v (28; SGD without momentum reads g, p and writes p: 12).  eager: unscale_ reads and writes g (8), the clip reads g for
    the norm (4) and reads and writes it to scale it (8), then the step, which also writes g (4) when it unscales.
    captured: pass 1 reads g (4, when it runs), pass 2 is the step and writes g back (4) whenever it unscales or clips."""
    step = 12 if optim == "sgd" else 28
    if route == "eager":
        if clip:
            return (8 if scaler else 0) + 4 + 8 + step
        return step + 4 if scaler else step
    return (4 if clip or scaler else 0) + (step + 4 if clip or scaler else step)


class Run:
    def __init__(self, optim, route, named, max_norm, dev):
        from qagnn_b200 import optim as O
        self.ps = [torch.nn.Parameter(p.detach().clone()) for _, p in named]
        groups = recipe_groups(list(zip([n for n, _ in named], self.ps)), 1e-3)
        self.opt = O.DEVICE_OPTIMIZER_CLASSES[optim](groups)
        self.scaler = torch.amp.GradScaler("cuda")
        self.scaler.scale(torch.ones((), device=dev))
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda s: min(1.0, (s + 1) / 100))
        self.max_norm = max_norm
        self.tail = O.CapturedTail(self.opt, self.scaler, self.sched, max_norm, self.ps) if route == "captured" else None

    def __call__(self):
        from qagnn_b200 import optim as O
        if self.tail is not None:
            return self.tail()
        if self.max_norm > 0:
            self.scaler.unscale_(self.opt)
            O.clip_grad_norm_(self.ps, self.max_norm)
        self.sched.step()
        self.scaler.step(self.opt)
        self.scaler.update()


def case_set(name, named, dev, reps, optim, clipping):
    g = torch.Generator(device=dev).manual_seed(0)
    grads = [torch.randn(p.shape, device=dev, generator=g) * 1e-3 for _, p in named]
    norm = float(torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(x) for x in grads])))
    max_norm = {"clips": 0.5 * norm, "no_clip": 0.0, "recipe": 1.0}[clipping]
    runs = {r: Run(optim, r, named, max_norm, dev) for r in ROUTES}
    for r in ROUTES:
        for p, x in zip(runs[r].ps, grads):
            p.grad = x.clone()

    def load(r):
        sc = runs[r].scaler._scale
        for p, x in zip(runs[r].ps, grads):
            torch.mul(x, sc, out=p.grad)

    for r in ROUTES:  # state, capture and the rectified branch (step >= 6) before timing
        for _ in range(7):
            load(r)
            runs[r]()
    wall, host, kern = ({r: [] for r in ROUTES} for _ in range(3))
    for _ in range(reps):
        for r in ROUTES:
            load(r)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            runs[r]()
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            wall[r].append((time.perf_counter() - t0) * 1e3)
            host[r].append((t1 - t0) * 1e3)
    for _ in range(5):
        for r in ROUTES:
            load(r)
            torch.cuda.synchronize()
            kern[r].append(kernel_ms(runs[r]))
    n_params = sum(p.numel() for _, p in named)
    out = []
    for r in ROUTES:
        load(r)
        launches, syncs = profile_counts(runs[r])
        k = stats(kern[r])
        nbytes = traffic(r, max_norm > 0, True, optim)
        out.append({"case": name, "route": r, "max_norm": clipping, "tensors": len(named), "params": n_params,
                    "wall_ms": stats(wall[r]), "host_ms": stats(host[r]), "launches": launches, "syncs": syncs,
                    "kernel_ms": k, "bytes_per_param": nbytes,
                    "hbm_fraction": nbytes * n_params / (k["median"] * 1e-3) / (HBM_TBS * 1e12),
                    "captures": runs[r].tail.captures if runs[r].tail else None})
    return out


def case_batch(dev, reps, seed, optim):
    from qagnn_b200 import data as Dt
    from qagnn_b200.pipeline import SplitTrainBatch, train_chunks
    n_q, mbs, branches = 64, 2, 8
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_q * NC, seed=seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC, N_NODE)
    cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)
    labels = torch.from_numpy(np.random.default_rng(seed).integers(0, NC, n_q))
    split = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, dev, T, R, labels=labels)
    K, M = flat.max_batch_edges(mbs), flat.max_graph_edges()
    g = torch.Generator(device=dev).manual_seed(seed)
    svs = [torch.randn(mbs * NC, SENT_DIM, device=dev, generator=g).requires_grad_(True) for _ in range(n_q // mbs)]
    qids = np.random.default_rng(seed).permutation(n_q)
    runs = {}
    for r in ROUTES:
        dec = make_decoder(dev, 0.2)
        named = [(n, p) for n, p in dec.named_parameters() if p.requires_grad]
        run = Run(optim, r, named, 1.0, dev)
        run.ps = [p for _, p in named]  # train the decoder's own parameters
        from qagnn_b200 import optim as O
        run.opt = O.DEVICE_OPTIMIZER_CLASSES[optim](recipe_groups(named, 1e-3))
        run.sched = torch.optim.lr_scheduler.LambdaLR(run.opt, lambda s: min(1.0, (s + 1) / 100))
        if r == "captured":
            run.tail = O.CapturedTail(run.opt, run.scaler, run.sched, 1.0, run.ps)
        tb = SplitTrainBatch(dec, split, mbs, branches=branches, edge_capacity=K, max_edges=M, autocast_dtype=torch.float16)
        runs[r] = (run, tb)

    def batch(r):
        run, tb = runs[r]
        run.opt.zero_grad(set_to_none=False)
        j = 0
        for chunk in train_chunks(qids, mbs, branches):
            w = torch.full((len(chunk),), mbs / n_q, device=dev)
            run.scaler.scale((tb(chunk, svs[j:j + len(chunk)]) * w).sum()).backward()
            j += len(chunk)
        run()

    for r in ROUTES:
        for _ in range(3):
            batch(r)
    wall = {r: [] for r in ROUTES}
    for _ in range(reps):
        for r in ROUTES:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batch(r)
            torch.cuda.synchronize()
            wall[r].append((time.perf_counter() - t0) * 1e3)
    return [{"case": "batch", "route": r, "questions": n_q, "mbs": mbs, "branches": branches, "amp": "fp16",
             "wall_ms": stats(wall[r])} for r in ROUTES]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--optim", choices=("radam", "adamw", "adam", "sgd"), default="radam")
    ap.add_argument("--cases", nargs="+", default=["decoder", "encoder", "batch"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--append", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tail.py measures on a GPU; none is visible")
    dev = torch.device("cuda:0")
    info = gpu_info()
    dec = make_decoder(dev, 0.2)
    named_dec = [("decoder." + n, p) for n, p in dec.named_parameters() if p.requires_grad]
    lines = []
    if "decoder" in args.cases:
        lines += case_set("decoder", named_dec, dev, args.reps, args.optim, "recipe")
    if "encoder" in args.cases:
        torch.manual_seed(0)
        enc = [(n, torch.randn(s, device=dev) * 0.02) for n, s in roberta_large_shapes()] + named_dec
        for clipping in ("clips", "no_clip"):
            lines += case_set("encoder", enc, dev, args.reps, args.optim, clipping)
            torch.cuda.empty_cache()
        del enc
    if "batch" in args.cases:
        lines += case_batch(dev, args.reps, args.seed, args.optim)
    out = open(args.out, "a" if args.append else "w") if args.out else sys.stdout
    for line in lines:
        line.update(gpu=info, optim=args.optim)
        out.write(json.dumps(line) + "\n")
    if args.out:
        out.close()


if __name__ == "__main__":
    main()
