"""Times data-parallel training of a split (qagnn_b200.distributed.DataParallelSplitTrain) across the GPUs of one box:

    torchrun --nproc-per-node N tools/bench_dp_train.py --out profiles/h100_dp_train.jsonl     # N = 1, 2, 4, 8
    python tools/bench_dp_train.py --out ...                                                  # N = 1, no process group

Workload: tools/bench_split_train.py's loader-shaped synthetic split and decoder (k = 5, D = 200, sent_dim 1024, dropout
0.2) with the recipe's frozen 1024-wide concept table, fp16 autocast with a GradScaler, optimiser batches of 64 questions in micro-batches of 2 (the recipes' -bs 64 -mbs 2)
and --loss cross_entropy.  The encoder is a frozen stand-in: each micro-batch's sent_vecs is a fixed random tensor, so
the encoder bucket is empty and every number is the decoder's.

Per N, rank 0 appends one line: the optimiser-batch wall time (zero_grad, this rank's micro-steps, reduce_, unscale_,
clip_grad_norm_, the RAdam step and the scaler update; each window of --batches batches ends in a device synchronise), median
and spread over --reps windows; reduce_'s parts from CUDA events around each (the slot all-gather, the ordered-sum kernel, the
encoder bucket and the BatchNorm fold), medians over the timed batches; the ordered-sum kernel's time alone (50 launches of
the C entry back to back between two events, argument arrays built once) and its compulsory bytes (M P 4 read of the slots plus P 4 read and written of .grad) over
that time, against 3.35 TB/s; with one rank, the plain SplitTrainStep loop on
an identical model with the same tail, its windows alternated with the wrapper's; the card's name, power limit and largest SM
clock, read in the same run."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_split_train import D, K_LAYERS, N_CONCEPT, N_NODE, NC, OPT_BATCH, R, SENT_DIM, T  # noqa: E402
from bench_stream_split import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
MBS = 2


def make_decoder(dev, dropout):
    """bench_split_train.make_decoder with the recipe's 1024-wide concept table, frozen: 86 trainable tensors, 2,845,025
    elements."""
    import qagnn_b200
    from oracle import qagnn_oracle as O
    torch.manual_seed(1)
    dec = qagnn_b200.QAGNN(None, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, D, 1024, 2, D, 0, dropout, dropout, dropout,
                           pretrained_concept_emb=torch.randn(N_CONCEPT, 1024), freeze_ent_emb=True)
    dec.gnn.load_state_dict(O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=0))
    for m in dec.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = dropout
    return dec.to(dev).train()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4, help="optimiser batches per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dp_train.py: needs a CUDA device")

    from qagnn_b200 import data as Dt
    from qagnn_b200 import distributed as D
    from qagnn_b200 import optim
    from qagnn_b200.pipeline import SplitTrainStep

    rank = int(os.environ.get("RANK", 0))
    if "WORLD_SIZE" in os.environ:
        local = int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local)
        dev = torch.device(f"cuda:{local}")
        dist.init_process_group("nccl", device_id=dev)
    else:
        dev = torch.device("cuda:0")
    world = dist.get_world_size() if dist.is_initialized() else 1
    try:
        n_q = OPT_BATCH * 4
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "split.graph.adj.pk")
            Dt.synth_adj_pickle(path, n_q * NC, seed=args.seed)
            cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
        flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC,
                               N_NODE)
        cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)
        labels = torch.from_numpy(np.random.default_rng(args.seed).integers(0, NC, n_q))
        split = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, dev, T, R, labels=labels)
        dec = make_decoder(dev, 0.2)
        torch.manual_seed(1000 + rank)  # each rank its own dropout stream
        step = SplitTrainStep(dec, split, MBS, edge_capacity=flat.max_batch_edges(MBS), max_edges=flat.max_graph_edges(),
                              autocast_dtype=torch.float16)
        dp = D.DataParallelSplitTrain(step, split, batch_size=OPT_BATCH, micro_batch_size=MBS)
        params = [p for p in dec.parameters() if p.requires_grad]
        opt = optim.RAdam(params, lr=1e-5)
        scaler = torch.amp.GradScaler("cuda")
        g = torch.Generator(device=dev).manual_seed(args.seed)
        svs = [torch.randn(MBS * NC, SENT_DIM, device=dev, generator=g) for _ in range(4)]
        perm = np.random.default_rng(args.seed).permutation(n_q)
        batches = [perm[a:a + OPT_BATCH] for a in range(0, n_q, OPT_BATCH)]

        def micro_steps(batch):
            opt.zero_grad()
            for j, q in enumerate(dp.micro_batches(batch)):
                with dp.micro_step():
                    scaler.scale(dp.loss(q, svs[j % len(svs)]) * len(q) / len(batch)).backward()

        def tail():
            scaler.unscale_(opt)
            optim.clip_grad_norm_(params, 1.0)
            scaler.step(opt)
            scaler.update()

        def window(n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(n):
                batch = batches[i % len(batches)]
                micro_steps(batch)
                dp.reduce_(len(batch))
                tail()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / n

        # with one rank, the plain SplitTrainStep loop on its own copy of the same model, with the same tail, alternated
        plain = None
        if world == 1:
            pdec = make_decoder(dev, 0.2)
            pstep = SplitTrainStep(pdec, split, MBS, edge_capacity=flat.max_batch_edges(MBS),
                                   max_edges=flat.max_graph_edges(), autocast_dtype=torch.float16)
            pparams = [p for p in pdec.parameters() if p.requires_grad]
            popt, pscaler = optim.RAdam(pparams, lr=1e-5), torch.amp.GradScaler("cuda")

            def plain(n):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(n):
                    batch = batches[i % len(batches)]
                    popt.zero_grad()
                    for j, a in enumerate(range(0, len(batch), MBS)):
                        q = batch[a:a + MBS]
                        pscaler.scale(pstep(q, svs[j % len(svs)]) * len(q) / len(batch)).backward()
                    pscaler.unscale_(popt)
                    optim.clip_grad_norm_(pparams, 1.0)
                    pscaler.step(popt)
                    pscaler.update()
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) / n

        window(2)  # capture, optimiser state, NCCL communicators
        walls, plain_walls = [], []
        if plain is not None:
            plain(2)
        for _ in range(args.reps):
            walls.append(window(args.batches))
            if plain is not None:
                plain_walls.append(plain(args.batches))

        parts = {k: [] for k in ("all_gather", "ordered_sum", "encoder_bucket", "bn_fold", "reduce_total")}
        for i in range(args.reps * 2):
            batch = batches[i % len(batches)]
            micro_steps(batch)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            if dp._pattern != dp._other_pattern:
                dp._exchange_reached()
            ev[0].record()
            dp._gather_slots()
            ev[1].record()
            dp._sum_slots()
            ev[2].record()
            dp._reduce_other()
            ev[3].record()
            dp._fold_bn()
            ev[4].record()
            dp._batch = None
            tail()
            torch.cuda.synchronize()
            for k, (a, b) in zip(parts, [(0, 1), (1, 2), (2, 3), (3, 4), (0, 4)]):
                parts[k].append(ev[a].elapsed_time(ev[b]))
        med = {k: statistics.median(v) for k, v in parts.items()}
        M = -(-OPT_BATCH // MBS)
        P = sum(params[i].numel() for i in dp._reached)
        kernel_bytes = M * P * 4 + 2 * P * 4
        # the kernel alone: 50 launches of the C entry back to back on the gathered slots, its argument arrays built once so
        # that the host keeps ahead of the device (reduce_'s event pair also holds ordered_grad_sum_'s Python checks)
        import ctypes as C
        from qagnn_b200 import _lib
        outs = [torch.empty_like(params[i]) for i in dp._reached]
        n = len(outs)
        cargs = (n, (C.c_void_p * n)(*[o.data_ptr() for o in outs]), (C.c_int64 * n)(*[o.numel() for o in outs]),
                 (C.c_int64 * n)(*D.slot_columns([o.numel() for o in outs])[0]), (C.c_int32 * n)(*([0] * n)),
                 _lib.ptr(dp._grad_slots.slots), dp._grad_slots.slots.stride(0), M, _lib.stream_ptr(dev))
        lib = _lib.load()
        _lib.check(lib.qagnn_ordered_grad_sum(*cargs), "qagnn_ordered_grad_sum")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            lib.qagnn_ordered_grad_sum(*cargs)
        e1.record()
        torch.cuda.synchronize()
        kernel_ms = e0.elapsed_time(e1) / 50
        line = {"gpu": gpu_info(), "world_size": world, "batch_size": OPT_BATCH, "micro_batch_size": MBS, "autocast": "fp16",
                "loss": "cross_entropy", "encoder": "frozen stand-in", "n_node": N_NODE, "k": 5, "D": 200,
                "micro_batches": M, "micro_batches_per_rank": -(-M // world), "decoder_grad_tensors": len(dp._reached),
                "decoder_grad_elements": P, "batches_per_window": args.batches, "reps": args.reps,
                "ms_per_optimiser_batch": 1e3 * statistics.median(walls),
                "optimiser_batch_spread_ms": [1e3 * min(walls), 1e3 * max(walls)],
                "reduce_ms": {k: v for k, v in med.items()},
                "plain_split_train_step_ms_per_optimiser_batch": 1e3 * statistics.median(plain_walls) if plain_walls else None,
                "plain_spread_ms": [1e3 * min(plain_walls), 1e3 * max(plain_walls)] if plain_walls else None,
                "ordered_sum_kernel_ms": kernel_ms, "ordered_sum_bytes": kernel_bytes,
                "ordered_sum_hbm_share": kernel_bytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S}
        if rank == 0:
            print(json.dumps(line), flush=True)
            if args.out:
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "a") as f:
                    f.write(json.dumps(line) + "\n")
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
