"""Times one training micro-step of the QAGNN decoder (forward + backward(), ending in a device synchronise), eager and as
pipeline.TrainStep's two CUDA graphs, alternated in one process.

Workloads: the batch of the reference's training recipes (run_qagnn__*.sh: -mbs 2, so 2 questions x 5 choices = 10 sub-graphs
per backward) and the whole -bs 64 batch (320 sub-graphs), each under fp16 autocast (--fp16 true), under bf16 autocast and in
fp32.  Sub-graphs
come from the loader-shaped synthetic split of tools/bench_stream_split.py (n = 200, 38 relations), packed at the split's
edge capacity; decoder k = 5, D = 200, sent_dim 1024, dropout 0.2 (the recipes' values).  The text encoder and the
optimiser are not part of the step (sent_vecs is a leaf tensor standing in for the encoder's output).

Paths, each timed over --steps micro-steps, --reps rounds in alternation, medians reported:
  eager          the decoder called eagerly with index validation (GraphPrep synchronises once per micro-step to check)
  eager_nocheck  the same after one check_batch with check_indices off: the eager path with no host synchronisation
  graphs         TrainStep (index checks through the deferred status word, no host synchronisation)
Per path: wall ms per micro-step, host ms per micro-step (the enqueue loop before the final synchronise), library kernel
launches per micro-step (qagnn_launch_count), and in a separate profiled pass the CUDA kernels and the kernel / graph
launch calls per micro-step (torch.profiler).  Everything it writes goes to --out.

    python tools/bench_train_step.py --steps 20 --reps 5 --out /tmp/train_step.jsonl
"""
import argparse
import copy
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

N_NODE, NC, D, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, DROPOUT = 200, 5, 200, 5, 4, 38, 1024, 2000, 0.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, nargs="+", default=[2, 64], help="questions per micro-batch (x5 choices)")
    ap.add_argument("--steps", type=int, default=20, help="micro-steps per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_step.py: needs a CUDA device")

    import qagnn_b200
    from bench_stream_split import gpu_info
    from oracle import qagnn_oracle as O
    from qagnn_b200 import _lib
    from qagnn_b200 import data as Dt
    from qagnn_b200.pipeline import TrainStep

    dev = torch.device("cuda:0")
    lib = _lib.load()
    gpu = gpu_info()
    n_batches = 4
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, max(args.questions) * n_batches * NC, seed=args.seed)
        _, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    M = flat.max_graph_edges()
    lines = []
    for bs in args.questions:
        K = flat.max_batch_edges(bs)
        g = torch.Generator().manual_seed(args.seed + bs)
        batches = []
        for b in range(n_batches):
            qs = np.arange(b * bs, (b + 1) * bs)
            B = bs * NC
            cid = torch.randint(1, N_CONCEPT + 1, (B, N_NODE), generator=g)
            cid[:, 0] = 0
            d = {"sent_vecs": torch.randn(B, SENT_DIM, generator=g) * 0.5, "concept_ids": cid,
                 "node_type_ids": ntypes[qs].reshape(B, N_NODE), "node_scores": scores[qs].reshape(B, N_NODE, 1),
                 "adj_lengths": lens[qs].reshape(B), "labels": torch.randint(0, NC, (bs,), generator=g)}
            d = {k: v.to(dev) for k, v in d.items()}
            d["adj"] = flat.pack(qs, edge_capacity=K).to(dev)
            d["sent_vecs"].requires_grad_(True)
            batches.append(d)
        edges = [d["adj"].n_edges for d in batches]
        for amp in (torch.float16, torch.bfloat16, None):
            torch.manual_seed(1)
            base = qagnn_b200.QAGNN(None, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, D, D, 2, D, 0, DROPOUT, DROPOUT, DROPOUT)
            base.gnn.load_state_dict(O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=0))
            base = base.to(dev).train()
            dec_e, dec_n, dec_g = base, copy.deepcopy(base), copy.deepcopy(base)
            dec_n.gnn.check_batch(batches[0]["adj"], batches[0]["node_type_ids"])
            dec_n.gnn.check_indices = False
            b0 = batches[0]
            step = TrainStep(dec_g, b0["sent_vecs"], b0["concept_ids"], b0["node_type_ids"], b0["node_scores"], b0["adj_lengths"],
                             b0["adj"], max_edges=M, edge_capacity=K, autocast_dtype=amp)
            ac = (lambda: torch.autocast("cuda", dtype=amp, cache_enabled=False)) if amp else torch.enable_grad

            def eager_fn(dec):
                def run(d):
                    with ac():
                        logits, _ = dec(d["sent_vecs"], d["concept_ids"], d["node_type_ids"], d["node_scores"], d["adj_lengths"],
                                        d["adj"])
                        loss = torch.nn.functional.cross_entropy(logits.float().view(-1, NC), d["labels"])
                    loss.backward()
                return run

            def graph_run(d):
                logits, _ = step(d["sent_vecs"], d["concept_ids"], d["node_type_ids"], d["node_scores"], d["adj_lengths"], d["adj"])
                loss = torch.nn.functional.cross_entropy(logits.float().view(-1, NC), d["labels"])
                loss.backward()

            paths = {"eager": eager_fn(dec_e), "eager_nocheck": eager_fn(dec_n), "graphs": graph_run}

            def window(fn):
                torch.cuda.synchronize()
                l0 = lib.qagnn_launch_count()
                t0 = time.perf_counter()
                for i in range(args.steps):
                    fn(batches[i % n_batches])
                t1 = time.perf_counter()
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                return (t2 - t0) / args.steps, (t1 - t0) / args.steps, (lib.qagnn_launch_count() - l0) / args.steps

            for fn in paths.values():  # warm-up
                window(fn)
            samples = {k: [] for k in paths}
            for _ in range(args.reps):
                for k, fn in paths.items():
                    samples[k].append(window(fn))
            res = {}
            for k, fn in paths.items():
                wall = [s[0] for s in samples[k]]
                res[k] = {"ms_per_step": 1e3 * statistics.median(wall), "spread_ms": [1e3 * min(wall), 1e3 * max(wall)],
                          "host_ms_per_step": 1e3 * statistics.median(s[1] for s in samples[k]),
                          "lib_launches_per_step": samples[k][0][2]}
                from torch.profiler import ProfilerActivity, profile
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    for i in range(args.steps):
                        fn(batches[i % n_batches])
                    torch.cuda.synchronize()
                kernels = launches = 0
                for e in prof.events():
                    if e.device_type == torch.autograd.DeviceType.CUDA:
                        kernels += 1
                    elif e.name.startswith(("cudaLaunchKernel", "cuLaunchKernel", "cudaGraphLaunch")):
                        launches += 1
                res[k]["profiler_gpu_ops_per_step"] = kernels / args.steps
                res[k]["profiler_launch_calls_per_step"] = launches / args.steps
            for d in batches:
                d["sent_vecs"].grad = None
            line = {"gpu": gpu, "questions": bs, "graphs": bs * NC, "n_node": N_NODE, "D": D, "k": K_LAYERS,
                    "autocast": {torch.float16: "fp16", torch.bfloat16: "bf16", None: "fp32"}[amp], "edge_capacity": K, "max_graph_edges": M,
                    "edges_per_batch": [min(edges), max(edges)], "steps": args.steps, "reps": args.reps, **res,
                    "speedup_vs_eager": res["eager"]["ms_per_step"] / res["graphs"]["ms_per_step"],
                    "speedup_vs_eager_nocheck": res["eager_nocheck"]["ms_per_step"] / res["graphs"]["ms_per_step"],
                    "parent_eager": "not measured"}
            print(json.dumps(line), flush=True)
            lines.append(line)
            del step, dec_e, dec_n, dec_g, base
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
