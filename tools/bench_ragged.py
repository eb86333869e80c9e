"""Times the eval decoder step on ragged batches against padded ones, on a loader-shaped synthetic split.

The split is built as tools/bench_stream_split.py builds it (data.synth_adj_pickle -> load_flat_adj_cache: cfg3 graph
statistics, max_node_num 200, 38 relations; 64 questions x 5 choices = 320 graphs per batch, k = 5, D = 200).  Two captured
DecoderSteps run the same batches, in alternated windows, from batches already on the device (each run copies its batch into
the step's buffers, as a streamed split does):

  padded  every graph padded to 200 rows, edges at the split's edge capacity K (DecoderStep.PACKED_FIELDS);
  ragged  the same graphs without padding rows, node arrays at the split's node capacity N_cap (data.split_node_capacity)
          and the same K (DecoderStep.RAGGED_FIELDS).

It reports the median and spread of the time per batch, the padded-row fraction of the split (computed from adj_lengths) and
max |logits_ragged - logits_padded| and max |pool_attn_ragged - pool_attn_padded| over every batch, and appends one JSON line
to --out.

    python tools/bench_ragged.py --batches 8 --reps 5 --out profiles/h100_ragged.jsonl
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

N_NODE, NC, D, K_LAYERS, T, R, SENT_DIM = 200, 5, 200, 5, 4, 38, 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=64, help="questions per batch (x5 choices)")
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged.py: needs a CUDA device")

    import qagnn_b200
    from bench_stream_split import gpu_info
    from oracle import qagnn_oracle as O
    from qagnn_b200 import data as Dt
    from qagnn_b200.layers import MLP, MultiheadAttPoolLayer
    from qagnn_b200.pipeline import DecoderStep

    dev = torch.device("cuda:0")
    bs, nb = args.batch_size, args.batches
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, bs * nb * NC, seed=args.seed)
        _, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    K, M = flat.max_batch_edges(bs), flat.max_graph_edges()
    N_cap = Dt.split_node_capacity(lens, bs)  # dev / test splits are read in order
    B = bs * NC
    g = torch.Generator().manual_seed(args.seed)
    padded, ragged = [], []
    for b in range(nb):
        qs = np.arange(b * bs, (b + 1) * bs)
        H = torch.randn(B, N_NODE, D, generator=g) * 0.5
        sv = torch.randn(B, SENT_DIM, generator=g) * 0.5
        al = lens[qs].reshape(-1)
        pa = flat.pack(qs, pin=False, edge_capacity=K)
        padded.append({"H": H, "edge_index": pa.edge_index, "edge_type": pa.edge_type, "node_type": ntypes[qs].reshape(B, N_NODE),
                       "node_score": scores[qs].reshape(B, N_NODE, 1), "sent_vecs": sv, "adj_lengths": al,
                       "graph_ptr": pa.graph_ptr})
        ra = flat.pack(qs, pin=False, edge_capacity=K, adj_lengths=al, node_capacity=N_cap)
        rows = torch.cat([i * N_NODE + torch.arange(int(l)) for i, l in enumerate(al)])
        Hp = torch.zeros(N_cap, D)
        Hp[:rows.numel()] = H.reshape(-1, D)[rows]
        ntp = torch.full((N_cap,), 2, dtype=torch.long)
        ntp[:rows.numel()] = ntypes[qs].reshape(-1)[rows]
        nsp = torch.zeros(N_cap, 1)
        nsp[:rows.numel()] = scores[qs].reshape(-1, 1)[rows]
        ragged.append({"H": Hp, "edge_index": ra.edge_index, "edge_type": ra.edge_type, "node_type": ntp, "node_score": nsp,
                       "sent_vecs": sv, "adj_lengths": al, "graph_ptr": ra.graph_ptr})
    padded = [{k: v.to(dev) for k, v in h.items()} for h in padded]
    ragged = [{k: v.to(dev) for k, v in h.items()} for h in ragged]
    valid = int(lens[:bs * nb].sum())
    pad_fraction = 1.0 - valid / (bs * nb * NC * N_NODE)

    sd = O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, K_LAYERS, T, R, D, D, D).eval()
    mod.load_state_dict(sd)
    mod = mod.to(dev)
    torch.manual_seed(1)
    pooler = MultiheadAttPoolLayer(2, SENT_DIM, D).eval().to(dev)
    fc = MLP(D + SENT_DIM + D, D, 1, 0, 0.2, layer_norm=True).eval().to(dev)

    dp = {k: v.clone() for k, v in padded[0].items()}
    dr = {k: v.clone() for k, v in ragged[0].items()}
    step_p = DecoderStep(mod, pooler, fc, dp, use_cuda_graph=True, max_edges=M)
    step_r = DecoderStep(mod, pooler, fc, dr, use_cuda_graph=True, max_edges=M, max_nodes=N_NODE)

    def window(step, bufs, batches, keep=False):
        out = []
        for h in batches:
            for k in bufs:
                bufs[k].copy_(h[k], non_blocking=True)
            logits, attn, _ = step.run()
            if keep:
                out.append((logits.clone(), attn.clone()))
        return out

    def timed(step, bufs, batches):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        window(step, bufs, batches)
        ev1.record()
        ev1.synchronize()
        return ev0.elapsed_time(ev1) / len(batches)

    res_p = window(step_p, dp, padded, keep=True)
    res_r = window(step_r, dr, ragged, keep=True)
    torch.cuda.synchronize()
    d_logits = max((a[0] - b[0]).abs().max().item() for a, b in zip(res_p, res_r))
    d_attn = max((a[1] - b[1]).abs().max().item() for a, b in zip(res_p, res_r))
    t_p, t_r = [], []
    for _ in range(args.reps):
        t_p.append(timed(step_p, dp, padded))
        t_r.append(timed(step_r, dr, ragged))

    def stats(ts):
        return {"ms_per_batch": statistics.median(ts), "spread_ms": [min(ts), max(ts)]}

    res = {"gpu": gpu_info(), "batch_graphs": B, "n_node": N_NODE, "D": D, "k": K_LAYERS, "batches": nb, "reps": args.reps,
           "edge_capacity": K, "node_capacity": N_cap, "padded_rows": B * N_NODE, "padded_row_fraction": pad_fraction,
           "padded": stats(t_p), "ragged": stats(t_r), "max_abs_d_logits": d_logits, "max_abs_d_pool_attn": d_attn}
    res["speedup"] = res["padded"]["ms_per_batch"] / res["ragged"]["ms_per_batch"]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
