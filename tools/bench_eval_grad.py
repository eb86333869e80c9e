"""Times the eval-mode QAGNN decoder forward + backward (gradients wanted, as when the encoder is fine-tuned under a frozen
decoder), on padded against ragged batches, in fp32 and under bf16 autocast.

The split is tools/bench_ragged.py's: data.synth_adj_pickle -> load_flat_adj_cache (cfg3 graph statistics, max_node_num
200, 38 relations), 64 questions x 5 choices = 320 graphs per batch, k = 5, D = 200.  The decoder runs in .eval() with
sent_vecs requiring grad; one timed unit is forward + loss.backward() over every batch of the window, bracketed by CUDA
events.  The four configurations run in one process, alternated in every repetition.  One JSON line per configuration is
appended to --out, with the card's name and power limit read in the same run.

    python tools/bench_eval_grad.py --batches 4 --reps 5 --out profiles/h100_eval_grad.jsonl
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N_NODE, NC, D, K_LAYERS, T, R, SENT_DIM, N_CONCEPT = 200, 5, 200, 5, 4, 38, 1024, 5000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=64, help="questions per batch (x5 choices)")
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_grad.py: needs a CUDA device")

    import qagnn_b200
    from bench_stream_split import gpu_info
    from qagnn_b200 import data as Dt

    dev = torch.device("cuda:0")
    bs, nb = args.batch_size, args.batches
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, bs * nb * NC, seed=args.seed)
        _, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    N_cap = Dt.split_node_capacity(lens, bs)
    B = bs * NC
    g = torch.Generator().manual_seed(args.seed)
    batches = []
    for b in range(nb):
        qs = np.arange(b * bs, (b + 1) * bs)
        al = lens[qs].reshape(-1)
        cids = torch.randint(1, N_CONCEPT + 1, (B, N_NODE), generator=g)
        cids[:, 0] = 0
        common = {"sent_vecs": torch.randn(B, SENT_DIM, generator=g) * 0.5, "concept_ids": cids,
                  "node_type": ntypes[qs].reshape(B, N_NODE), "node_scores": scores[qs].reshape(B, N_NODE, 1).float(),
                  "adj_lengths": al}
        common = {k: v.to(dev) for k, v in common.items()}
        batches.append({"common": common, "padded": flat.pack(qs, pin=False).to(dev),
                        "ragged": flat.pack(qs, pin=False, adj_lengths=al, node_capacity=N_cap).to(dev)})
    pad_fraction = 1.0 - int(lens[:bs * nb].sum()) / (bs * nb * NC * N_NODE)

    torch.manual_seed(1)
    dec = qagnn_b200.QAGNN(None, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, D, D, 2, D, 0, 0.2, 0.2, 0.2).to(dev).eval()

    def window(layout, amp):
        for bt in batches:
            c = bt["common"]
            sv = c["sent_vecs"].detach().requires_grad_(True)
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                logits, _ = dec(sv, c["concept_ids"], c["node_type"], c["node_scores"], c["adj_lengths"], bt[layout])
            logits.float().sum().backward()

    def timed(layout, amp):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        window(layout, amp)
        ev1.record()
        ev1.synchronize()
        return ev0.elapsed_time(ev1) / len(batches)

    configs = [(layout, amp) for amp in (False, True) for layout in ("padded", "ragged")]
    for cfg in configs:  # warm-up: every shape, library algorithm choice and module load
        window(*cfg)
    times = {cfg: [] for cfg in configs}
    for _ in range(args.reps):
        for cfg in configs:
            times[cfg].append(timed(*cfg))
    gpu = gpu_info()
    for (layout, amp), ts in times.items():
        res = {"gpu": gpu, "what": "QAGNN.eval() forward + backward, sent_vecs.requires_grad", "layout": layout,
               "precision": "bf16 autocast" if amp else "fp32", "batch_graphs": B, "n_node": N_NODE, "D": D, "k": K_LAYERS,
               "batches": nb, "reps": args.reps, "node_capacity": N_cap, "padded_row_fraction": pad_fraction,
               "ms_per_batch": statistics.median(ts), "spread_ms": [min(ts), max(ts)]}
        line = json.dumps(res)
        print(line)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
