"""Streams a loader-shaped synthetic split through the decoder step and reports batches/s and edge-layers/s.

The split has the graph statistics of the CommonsenseQA-shaped config (data.synth_adj_pickle -> load_flat_adj_cache:
~120-concept sub-graphs, max_node_num 200, 38 relations) and the batch size of the 1xH100 config (64 questions x 5
choices = 320 graphs per batch).  Two ways to run it are timed, alternated in one process:

  captured  PackedAdjBatchGenerator-style batches packed at the split's edge capacity, streamed by StreamedRunner through
            ONE captured DecoderStep per buffer set (copies on their own streams);
  eager     every batch packed exactly, uploaded, run through a per-batch DecoderStep without a CUDA graph, downloaded.

edge-layers/s = k * (real edges of the batches) / time.  Both paths must return the same logits and pooling attention,
bit for bit, or the run aborts.  Everything it writes goes to a temporary directory and to --out.

    python tools/bench_stream_split.py --batches 8 --reps 3 --out /tmp/stream_split.jsonl
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_NODE, NC, D, K_LAYERS, T, R, SENT_DIM = 200, 5, 200, 5, 4, 38, 1024


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=64, help="questions per batch (x5 choices)")
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_split.py: needs a CUDA device")

    import qagnn_b200
    from oracle import qagnn_oracle as O
    from qagnn_b200 import data as Dt
    from qagnn_b200.layers import MLP, MultiheadAttPoolLayer
    from qagnn_b200.pipeline import DecoderStep, StreamedRunner, packed_host_batch

    dev = torch.device("cuda:0")
    bs, nb = args.batch_size, args.batches
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, bs * nb * NC, seed=args.seed)
        _, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    K, M = flat.max_batch_edges(bs), flat.max_graph_edges()
    order = np.random.default_rng(args.seed).permutation(flat.n_questions())
    g = torch.Generator().manual_seed(args.seed)
    cap_hosts, exact_hosts = [], []
    for b in range(nb):
        qs = np.sort(order[b * bs:(b + 1) * bs])
        B = bs * NC
        H = torch.randn(B, N_NODE, D, generator=g) * 0.5
        sv = torch.randn(B, SENT_DIM, generator=g) * 0.5
        cap_hosts.append(packed_host_batch(flat.pack(qs, edge_capacity=K), H, ntypes[qs], scores[qs], sv, lens[qs]))
        exact_hosts.append(packed_host_batch(flat.pack(qs), H, ntypes[qs], scores[qs], sv, lens[qs]))
    edges = [int(h["graph_ptr"][-1]) for h in cap_hosts]

    sd = O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, K_LAYERS, T, R, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(dev)
    torch.manual_seed(1)
    pooler = MultiheadAttPoolLayer(2, SENT_DIM, D).eval().to(dev)
    fc = MLP(D + SENT_DIM + D, D, 1, 0, 0.2, layer_norm=True).eval().to(dev)

    runner = StreamedRunner(mod, cap_hosts[0], dev, depth=2, fields=DecoderStep.PACKED_FIELDS, download=(0, 1),
                            make_step=lambda d: DecoderStep(mod, pooler, fc, d, use_cuda_graph=True, max_edges=M))

    def captured():
        results = [None] * nb
        for i, hb in enumerate(cap_hosts):
            runner.submit(hb)
            if i >= 1:
                prev = (i - 1) % 2
                runner.ev_down[prev].synchronize()
                results[i - 1] = [t.clone() for t in runner.host_out[prev]]
        runner.drain()
        torch.cuda.synchronize()
        results[nb - 1] = [t.clone() for t in runner.host_out[(nb - 1) % 2]]
        return results

    def eager():
        results = []
        for hb in exact_hosts:
            d = {k: v.to(dev, non_blocking=True) for k, v in hb.items()}
            gp = hb["graph_ptr"]
            step = DecoderStep(mod, pooler, fc, d, use_cuda_graph=False, max_edges=int((gp[1:] - gp[:-1]).max()))
            logits, attn, _ = step.run()
            results.append([logits.to("cpu"), attn.to("cpu")])
        torch.cuda.synchronize()
        return results

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fn()
        return time.perf_counter() - t0, res

    timed(captured)
    timed(eager)  # warm-up: module loads, workspaces, one capture per buffer set
    t_cap, t_eag = [], []
    for _ in range(args.reps):
        t, rc = timed(captured)
        t_cap.append(t)
        t, re_ = timed(eager)
        t_eag.append(t)
    for i, (a, b) in enumerate(zip(rc, re_)):
        for x, y in zip(a, b):
            if not torch.equal(x, y):
                raise SystemExit(f"bench_stream_split.py: batch {i}: captured and eager results differ")

    def rates(ts):
        t = statistics.median(ts)
        return {"s_per_pass": t, "spread_s": [min(ts), max(ts)], "batches_per_s": nb / t,
                "edge_layers_per_s": K_LAYERS * sum(edges) / t}

    res = {"gpu": gpu_info(), "batch_graphs": bs * NC, "n_node": N_NODE, "D": D, "k": K_LAYERS, "batches": nb,
           "reps": args.reps, "edge_capacity": K, "max_graph_edges": M, "edges_per_batch": [min(edges), max(edges)],
           "mean_fill": sum(edges) / (nb * K), "captured": rates(t_cap), "eager": rates(t_eag),
           "outputs_identical": True}
    res["speedup"] = res["captured"]["batches_per_s"] / res["eager"]["batches_per_s"]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
