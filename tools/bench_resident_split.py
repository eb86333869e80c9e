"""Times the evaluation of a whole split held on the GPU (data.DeviceSplit + pipeline.SplitEvalStep) against today's route
(a pinned FlatAdjCache.pack and upload per batch, then the eager decoder), padded and ragged.

The split is built as tools/bench_ragged.py builds it (data.synth_adj_pickle -> load_flat_adj_cache: max_node_num 200, 38
relations; 64 questions x 5 choices = 320 graphs per batch).  A real QAGNN decoder in .eval() (k = 5, D = 200, sent_dim 1024,
a fixed 50 000-concept table with concept_in_dim 1024, 2 pooling heads) runs every full batch; the sent_vecs are made on the
device once and shared by every route.  Routes, each timed over the whole split with a host clock that ends in a device
synchronise, alternated over --reps repetitions:

  host_padded / host_ragged          flat.pack (pinned) + node rows sliced on the host, uploaded, eager decoder(...)
  resident_padded / resident_ragged  SplitEvalStep(question ids, sent_vecs): one CUDA graph per batch
  resident_*_item                    the same step on a split without labels, scored as evaluate_accuracy (qagnn.py:30-38)
                                     scores: argmax, compare with the batch's labels (on the device) and .item() per batch
  resident_*_scored                  a step on the same split built with labels: scored inside its graph, reset_scores()
                                     before the split and accuracy() (one read) after it

It also reports the host pack time alone (per batch), the assembly kernel alone (qagnn_assemble_batch: CUDA events around a
CUDA graph of 200 calls, so that the host's enqueue is not what is timed), max |d logits| and |d pool_attn| between every route
and host_padded, and the card's name, power limit and max SM clock, and appends one JSON line to --out.

    python tools/bench_resident_split.py --batches 16 --reps 5 --out profiles/h100_resident_split.jsonl
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

N_NODE, NC, D, K_LAYERS, T, R, SENT_DIM = 200, 5, 200, 5, 4, 38, 1024
N_CONCEPT, CONCEPT_IN = 50000, 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=64, help="questions per batch (x5 choices)")
    ap.add_argument("--batches", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resident_split.py: needs a CUDA device")

    import qagnn_b200
    from bench_stream_split import gpu_info
    from oracle import qagnn_oracle as O
    from qagnn_b200 import _lib
    from qagnn_b200 import data as Dt
    from qagnn_b200.pipeline import SplitEvalStep

    dev = torch.device("cuda:0")
    bs, nb = args.batch_size, args.batches
    B = bs * NC
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, bs * nb * NC, seed=args.seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
        flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC, N_NODE)
    cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)  # ids of the fixed table; the context node keeps 0
    K, M = flat.max_batch_edges(bs), flat.max_graph_edges()
    N_cap = Dt.split_node_capacity(lens, bs)  # the split is read in order
    batches = [np.arange(b * bs, (b + 1) * bs) for b in range(nb)]

    torch.manual_seed(args.seed)
    table = torch.randn(N_CONCEPT, CONCEPT_IN) * 0.5
    dec = qagnn_b200.QAGNN(None, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, D, CONCEPT_IN, 2, D, 0, 0.2, 0.2, 0.2,
                           pretrained_concept_emb=table)
    dec.gnn.load_state_dict(O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=args.seed))
    dec = dec.to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(args.seed)
    svs = [torch.randn(B, SENT_DIM, device=dev, generator=g) * 0.5 for _ in batches]

    split = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, dev, T, R)
    labels = torch.from_numpy(np.random.default_rng(args.seed).integers(0, NC, bs * nb))
    labelled = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, dev, T, R, labels=labels)
    batch_labels = [labels[q].to(dev) for q in batches]  # what the reference's loader hands evaluate_accuracy per batch
    caps = {"padded": None, "ragged": N_cap}
    steps = {name: SplitEvalStep(dec, split, bs, edge_capacity=K, max_edges=M, node_capacity=nc_) for name, nc_ in caps.items()}
    scored = {name: SplitEvalStep(dec, labelled, bs, edge_capacity=K, max_edges=M, node_capacity=nc_)
              for name, nc_ in caps.items()}
    accuracy = {}

    def up(t):
        return t.contiguous().pin_memory().to(dev, non_blocking=True)

    @torch.no_grad()
    def host_route(layout, keep=False):
        out = []
        for q, sv in zip(batches, svs):
            al = lens[q]
            adj = flat.pack(q, edge_capacity=K, adj_lengths=al if layout == "ragged" else None, node_capacity=caps[layout])
            logits, attn = dec(sv, up(cids[q].reshape(B, N_NODE)), up(ntypes[q].reshape(B, N_NODE)),
                               up(scores[q].reshape(B, N_NODE, 1)), up(al.reshape(B)), adj.to(dev))
            if keep:
                out.append((logits.clone(), attn.clone()))
        return out

    def resident_route(layout, keep=False):
        out = []
        for q, sv in zip(batches, svs):
            logits, attn = steps[layout](q, sv)
            if keep:
                out.append((logits.clone(), attn.clone()))
        return out

    def item_route(layout, keep=False):
        out, n_correct = [], 0
        for q, sv, lab in zip(batches, svs, batch_labels):
            logits, attn = steps[layout](q, sv)
            n_correct += (logits.view(bs, NC).argmax(1) == lab).sum().item()
            if keep:
                out.append((logits.clone(), attn.clone()))
        accuracy[f"resident_{layout}_item"] = n_correct / (bs * nb)
        return out

    def scored_route(layout, keep=False):
        out, step = [], scored[layout]
        step.reset_scores()
        for q, sv in zip(batches, svs):
            logits, attn = step(q, sv)
            if keep:
                out.append((logits.clone(), attn.clone()))
        accuracy[f"resident_{layout}_scored"] = step.accuracy()
        return out

    routes = {f"host_{l}": (lambda l=l, keep=False: host_route(l, keep)) for l in caps}
    routes.update({f"resident_{l}": (lambda l=l, keep=False: resident_route(l, keep)) for l in caps})
    routes.update({f"resident_{l}_item": (lambda l=l, keep=False: item_route(l, keep)) for l in caps})
    routes.update({f"resident_{l}_scored": (lambda l=l, keep=False: scored_route(l, keep)) for l in caps})
    results = {name: fn(keep=True) for name, fn in routes.items()}  # also warms every route up (and captures the steps)
    torch.cuda.synchronize()
    if len(set(accuracy.values())) != 1:
        raise SystemExit(f"bench_resident_split.py: the scoring routes disagree: {accuracy}")
    ref = results["host_padded"]
    deltas = {name: {"max_abs_d_logits": max((a[0] - b[0]).abs().max().item() for a, b in zip(res, ref)),
                     "max_abs_d_pool_attn": max((a[1] - b[1]).abs().max().item() for a, b in zip(res, ref))}
              for name, res in results.items() if name != "host_padded"}

    times = {name: [] for name in routes}
    for _ in range(args.reps):
        for name, fn in routes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / nb)

    pack_ms = {}
    for layout in caps:
        ts = []
        for _ in range(args.reps):
            for q in batches:
                t0 = time.perf_counter()
                flat.pack(q, edge_capacity=K, adj_lengths=lens[q] if layout == "ragged" else None, node_capacity=caps[layout])
                ts.append((time.perf_counter() - t0) * 1e3)
        pack_ms[layout] = {"median_ms": statistics.median(ts), "spread_ms": [min(ts), max(ts)]}

    lib = _lib.load()
    qd = torch.from_numpy(batches[0]).to(dev)
    kernel_us = {}
    for layout, nc_ in caps.items():
        bufs = split.buffers(bs, K, nc_)

        def assemble():
            st = lib.qagnn_assemble_batch(_lib.ptr(split.src), _lib.ptr(split.tgt), _lib.ptr(split.etype), _lib.ptr(split.graph_ptr),
                                          _lib.ptr(split.adj_lengths), split.lens.numel(), NC, N_NODE, _lib.ptr(qd), bs, K,
                                          -1 if nc_ is None else nc_, _lib.ptr(bufs["edges"]), _lib.ptr(bufs["graph_ptr"]),
                                          _lib.ptr(bufs.get("node_ptr")), _lib.stream_ptr(dev))
            _lib.check(st, "qagnn_assemble_batch")

        # 200 calls captured into one CUDA graph: a Python loop of ctypes calls would time the host's enqueue instead
        for _ in range(3):
            assemble()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(200):
                assemble()
        graph.replay()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(args.reps):
            ev0.record()
            graph.replay()
            ev1.record()
            ev1.synchronize()
            ts.append(ev0.elapsed_time(ev1) * 1e3 / 200)
        kernel_us[layout] = {"median_us": statistics.median(ts), "spread_us": [min(ts), max(ts)]}

    def stats(ts):
        return {"ms_per_batch": statistics.median(ts), "spread_ms": [min(ts), max(ts)]}

    res = {"gpu": gpu_info(), "batch_questions": bs, "batch_graphs": B, "batches": nb, "reps": args.reps, "n_node": N_NODE,
           "D": D, "k": K_LAYERS, "sent_dim": SENT_DIM, "edge_capacity": K, "node_capacity": N_cap,
           "split_edges": int(flat.graph_ptr[-1]), "routes": {name: stats(ts) for name, ts in times.items()},
           "host_pack": pack_ms, "assemble_kernel_us": kernel_us, "vs_host_padded": deltas,
           "captures": {name: s.captures for name, s in steps.items()},
           "captures_scored": {name: s.captures for name, s in scored.items()}, "accuracy": accuracy}
    res["speedup"] = {l: res["routes"][f"host_{l}"]["ms_per_batch"] / res["routes"][f"resident_{l}"]["ms_per_batch"] for l in caps}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
