"""Times the RAdam optimiser step three ways, alternated in one process:

  oracle       the reference's RAdam restated as eager torch ops (tests/radam_oracle.py): about ten ops per tensor, and
               GradScaler.step reads found_inf on the host before it calls step()
  torch_radam  torch.optim.RAdam(foreach=True, decoupled_weight_decay=True): the nearest stock optimiser (a different decay)
  qagnn        qagnn_b200.optim.RAdam: one launch per device, GradScaler's skip taken on the device

Cases:
  1. tail     the recipes' fp16 optimiser tail (unscale_, clip_grad_norm_(1.0), scaler.step, scaler.update) over the
              decoder's trainable tensors (k = 5, D = 200, sent_dim 1024): wall ms (ending in a synchronise), host ms (the
              enqueue before it), CUDA launches and synchronisations per tail from a separate torch.profiler pass
  2. encoder  optimizer.step() alone over a RoBERTa-large-shaped random parameter set (391 tensors, 355 M parameters) plus
              the decoder: kernel ms from CUDA events and, for qagnn, the fraction of 3.35 TB/s at 28 bytes per parameter
  3. batch    one optimiser batch of 64 questions at -mbs 2 under fp16 autocast through SplitTrainStep (32 micro-steps) and
              the tail of case 1 with each optimiser
Medians with the spread (min, max) over --reps alternated repetitions.  Everything it writes goes to --out.

    python tools/bench_optim.py --out profiles/h100_optim.jsonl
"""
import argparse
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

from bench_split_train import N_CONCEPT, N_NODE, NC, R, SENT_DIM, T, make_decoder  # noqa: E402
from bench_stream_split import gpu_info  # noqa: E402
from tests.radam_oracle import RAdamOracle  # noqa: E402

NO_DECAY = ("bias", "LayerNorm.bias", "LayerNorm.weight")
ROUTES = ("oracle", "torch_radam", "qagnn")
HBM_TBS = 3.35  # H100 SXM data-sheet HBM3 bandwidth


def make_opt(route, groups):
    from qagnn_b200.optim import RAdam
    if route == "oracle":
        return RAdamOracle(groups)
    if route == "torch_radam":
        return torch.optim.RAdam(groups, foreach=True, decoupled_weight_decay=True)
    return RAdam(groups)


def recipe_groups(named, lr):
    return [{"params": [p for n, p in named if not any(nd in n for nd in NO_DECAY)], "weight_decay": 0.01, "lr": lr},
            {"params": [p for n, p in named if any(nd in n for nd in NO_DECAY)], "weight_decay": 0.0, "lr": lr}]


def roberta_large_shapes():
    H, F, V = 1024, 4096, 50265
    shapes = [("embeddings.word_embeddings.weight", (V, H)), ("embeddings.position_embeddings.weight", (514, H)),
              ("embeddings.token_type_embeddings.weight", (1, H)), ("embeddings.LayerNorm.weight", (H,)),
              ("embeddings.LayerNorm.bias", (H,))]
    for i in range(24):
        L = f"encoder.layer.{i}."
        for n in ("query", "key", "value"):
            shapes += [(L + f"attention.self.{n}.weight", (H, H)), (L + f"attention.self.{n}.bias", (H,))]
        shapes += [(L + "attention.output.dense.weight", (H, H)), (L + "attention.output.dense.bias", (H,)),
                   (L + "attention.output.LayerNorm.weight", (H,)), (L + "attention.output.LayerNorm.bias", (H,)),
                   (L + "intermediate.dense.weight", (F, H)), (L + "intermediate.dense.bias", (F,)),
                   (L + "output.dense.weight", (H, F)), (L + "output.dense.bias", (H,)),
                   (L + "output.LayerNorm.weight", (H,)), (L + "output.LayerNorm.bias", (H,))]
    return shapes + [("pooler.dense.weight", (H, H)), ("pooler.dense.bias", (H,))]


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def profile_counts(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    launches = sum(n.startswith("cudaLaunchKernel") or n == "cuLaunchKernel" or n.startswith("cudaLaunchCooperative") for n in names)
    syncs = sum("Synchronize" in n for n in names) - 1  # less the closing torch.cuda.synchronize()
    return launches, syncs


def case_tail(dec, dev, reps):
    named = [(n, p) for n, p in dec.named_parameters() if p.requires_grad]
    g = torch.Generator(device=dev).manual_seed(0)
    grads = [torch.randn(p.shape, device=dev, generator=g) * 1e-3 for _, p in named]
    runs = {}
    for route in ROUTES:
        ps = [(n, torch.nn.Parameter(p.detach().clone())) for n, p in named]
        runs[route] = ([p for _, p in ps], make_opt(route, recipe_groups(ps, 1e-3)), torch.amp.GradScaler("cuda"))

    def load(route):
        ps, _, sc = runs[route]
        for p, gr in zip(ps, grads):
            p.grad = sc.scale(gr)

    def tail(route):
        ps, opt, sc = runs[route]
        sc.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(ps, 1.0)
        sc.step(opt)
        sc.update()

    for route in ROUTES:  # state allocation and the rectified branch (step >= 6) before timing
        for _ in range(7):
            load(route)
            tail(route)
    wall, host = {r: [] for r in ROUTES}, {r: [] for r in ROUTES}
    for _ in range(reps):
        for route in ROUTES:
            load(route)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tail(route)
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            wall[route].append((t2 - t0) * 1e3)
            host[route].append((t1 - t0) * 1e3)
    out = []
    for route in ROUTES:
        load(route)
        launches, syncs = profile_counts(lambda: tail(route))
        out.append({"case": "tail", "route": route, "tensors": len(named), "params": sum(p.numel() for _, p in named),
                    "wall_ms": stats(wall[route]), "host_ms": stats(host[route]), "launches": launches, "syncs": syncs})
    return out


def case_encoder(dec, dev, reps):
    named_dec = [("decoder." + n, p) for n, p in dec.named_parameters() if p.requires_grad]
    torch.manual_seed(0)
    base = [(n, torch.randn(s, device=dev) * 0.02) for n, s in roberta_large_shapes()] + [(n, p.detach()) for n, p in named_dec]
    n_params = sum(p.numel() for _, p in base)
    opts = {}
    for route in ROUTES:
        ps = [(n, torch.nn.Parameter(p.clone())) for n, p in base]
        for _, p in ps:
            p.grad = torch.randn_like(p) * 1e-3
        enc = [x for x in ps if not x[0].startswith("decoder.")]
        opts[route] = make_opt(route, recipe_groups(enc, 1e-5) + recipe_groups([x for x in ps if x[0].startswith("decoder.")], 1e-3))
        for _ in range(7):
            opts[route].step()
    del base
    ms = {r: [] for r in ROUTES}
    for _ in range(reps):
        for route in ROUTES:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            opts[route].step()
            e1.record()
            torch.cuda.synchronize()
            ms[route].append(e0.elapsed_time(e1))
    from torch.profiler import ProfilerActivity, profile
    kernel_us = []
    for _ in range(3):  # the kernel's own duration, without the host's enqueue in front of it
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            opts["qagnn"].step()
            torch.cuda.synchronize()
        kernel_us += [e.time_range.elapsed_us() for e in prof.events() if "radam_kernel" in e.name]
    out = []
    for route in ROUTES:
        line = {"case": "encoder", "route": route, "tensors": len(roberta_large_shapes()) + len(named_dec), "params": n_params,
                "step_ms": stats(ms[route])}
        if route == "qagnn":
            line["kernel_ms"] = stats([u * 1e-3 for u in kernel_us])
            line["hbm_fraction"] = 28 * n_params / (line["kernel_ms"]["median"] * 1e-3) / (HBM_TBS * 1e12)
            line["datasheet_ms"] = 28 * n_params / (HBM_TBS * 1e12) * 1e3
        out.append(line)
    del opts
    torch.cuda.empty_cache()
    return out


def case_batch(dev, reps, seed):
    from qagnn_b200 import data as Dt
    from qagnn_b200.pipeline import SplitTrainStep
    n_q, mbs = 64, 2
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
    svs = [torch.randn(mbs * NC, SENT_DIM, device=dev, generator=g).requires_grad_(True) for _ in range(4)]
    qids = np.random.default_rng(seed).permutation(n_q)
    runs = {}
    for route in ROUTES:
        dec = make_decoder(dev, 0.2)
        named = [(n, p) for n, p in dec.named_parameters() if p.requires_grad]
        step = SplitTrainStep(dec, split, mbs, edge_capacity=K, max_edges=M, autocast_dtype=torch.float16)
        runs[route] = (dec, step, make_opt(route, recipe_groups(named, 1e-3)), torch.amp.GradScaler("cuda"))

    def batch(route):
        dec, step, opt, sc = runs[route]
        opt.zero_grad()
        for j, a in enumerate(range(0, n_q, mbs)):
            sc.scale(step(qids[a:a + mbs], svs[j % len(svs)]) * (mbs / n_q)).backward()
        sc.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(dec.parameters(), 1.0)
        sc.step(opt)
        sc.update()

    for route in ROUTES:
        for _ in range(3):
            batch(route)
    wall = {r: [] for r in ROUTES}
    for _ in range(reps):
        for route in ROUTES:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batch(route)
            torch.cuda.synchronize()
            wall[route].append((time.perf_counter() - t0) * 1e3)
    return [{"case": "batch", "route": r, "questions": n_q, "mbs": mbs, "amp": "fp16", "wall_ms": stats(wall[r])} for r in ROUTES]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--cases", nargs="+", default=["tail", "encoder", "batch"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = gpu_info()
    dec = make_decoder(dev, 0.2)
    lines = []
    if "tail" in args.cases:
        lines += case_tail(dec, dev, args.reps)
    if "encoder" in args.cases:
        lines += case_encoder(dec, dev, max(5, args.reps // 3))
    if "batch" in args.cases:
        lines += case_batch(dev, max(3, args.reps // 6), args.seed)
    for line in lines:
        line["gpu"] = gpu
        print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
