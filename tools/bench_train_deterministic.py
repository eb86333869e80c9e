"""Cost of deterministic training: the message-passing core's backward with atomic edge-table sums (the default,
qagnn_mp_core_backward_typed) against the deterministic one (qagnn_mp_core_backward_det), and a TrainStep micro-step built
with and without torch.use_deterministic_algorithms(True).

Workloads: loader-shaped batches of 2 and 64 questions x 5 choices (10 and 320 sub-graphs of n = 200 nodes, 38 relations;
the split of tools/bench_stream_split.py) packed at the split's edge capacity, D = 200, H = 2 (the decoder's values).

  core        one backward call per launch, timed with CUDA events around --launches back-to-back calls, default and
              deterministic alternated --reps times, fp32 and bf16 operands; median microseconds per call
  train_step  TrainStep (decoder k = 5, sent_dim 1024, dropout 0.2) forward + backward() ending in a synchronise, one step
              per mode, the two alternated over --steps micro-steps x --reps windows; median ms per micro-step

CUBLAS_WORKSPACE_CONFIG=:4096:8 (which PyTorch requires for cuBLAS under the flag) is set for both modes.  The card's name,
power limit and maximum SM clock are read in the same run.  Prints one JSON line per measurement and appends them to --out.

    python tools/bench_train_deterministic.py --out /tmp/train_det.jsonl
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import tempfile
import time

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N_NODE, NC, D, H, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, DROPOUT = 200, 5, 200, 2, 5, 4, 38, 1024, 2000, 0.2


def bench_core(lib, _lib, prep, N, dt, launches, reps, dev):
    """(median us per default call, median us per deterministic call, bitwise-equal d_qkm, max |d_ke| difference)."""
    E = prep.E
    shape = _lib.Shape(N, E, D, H, T, R, 1, 0)
    g = torch.Generator(device=dev).manual_seed(N)
    Cn = R * T * T + T
    qkm = (torch.randn(N, 3 * D, generator=g, device=dev) * 0.5).to(dt)
    ke, me = (torch.randn(Cn, D, generator=g, device=dev).to(dt) for _ in range(2))
    d_aggr = torch.randn(N, D, generator=g, device=dev).to(dt)
    code = _lib.DTYPE_CODES[dt]
    aggr = torch.empty(N, D, dtype=dt, device=dev)
    alpha_s = torch.empty(N + E, H, dtype=torch.float32, device=dev)
    fscratch = torch.empty(N + E, H, dtype=torch.float32, device=dev)
    st = lib.qagnn_mp_core_forward_typed(C.byref(shape), code, _lib.ptr(prep.buf), _lib.ptr(qkm), _lib.ptr(ke), _lib.ptr(me),
                                         _lib.ptr(aggr), _lib.ptr(alpha_s), None, _lib.ptr(fscratch), _lib.stream_ptr(dev))
    _lib.check(st, "qagnn_mp_core_forward_typed")
    count, order = prep.combo_sort()
    outs = {m: (torch.empty_like(qkm), torch.empty_like(ke), torch.empty_like(me)) for m in ("default", "det")}
    nb = {"default": lib.qagnn_mp_core_scratch_bytes(C.byref(shape), code),
          "det": lib.qagnn_mp_core_backward_det_scratch_bytes(C.byref(shape), code)}
    scratch = {m: torch.empty(nb[m] // 4, dtype=torch.float32, device=dev) for m in nb}
    s = _lib.stream_ptr(dev)
    common = (_lib.ptr(qkm), _lib.ptr(ke), _lib.ptr(me), _lib.ptr(alpha_s), _lib.ptr(d_aggr))

    def call(m):
        dq, dk, dm = (_lib.ptr(t) for t in outs[m])
        if m == "default":
            st = lib.qagnn_mp_core_backward_typed(C.byref(shape), code, _lib.ptr(prep.buf), _lib.ptr(order), *common, dq, dk, dm,
                                                  _lib.ptr(scratch[m]), s)
        else:
            st = lib.qagnn_mp_core_backward_det(C.byref(shape), code, _lib.ptr(prep.buf), _lib.ptr(order), _lib.ptr(count), *common,
                                                dq, dk, dm, _lib.ptr(scratch[m]), nb[m], s)
        if st != 0:
            _lib.check(st, m)

    def window(m):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            call(m)
        b.record()
        b.synchronize()
        return 1e3 * a.elapsed_time(b) / launches

    for m in outs:
        window(m)
    t = {m: [] for m in outs}
    for _ in range(reps):
        for m in outs:
            t[m].append(window(m))
    torch.cuda.synchronize()
    same_dqkm = torch.equal(outs["default"][0], outs["det"][0])
    diff = float((outs["default"][1].float() - outs["det"][1].float()).abs().max())
    return ({m: statistics.median(v) for m, v in t.items()}, {m: [min(v), max(v)] for m, v in t.items()}, same_dqkm, diff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, nargs="+", default=[2, 64], help="questions per micro-batch (x5 choices)")
    ap.add_argument("--launches", type=int, default=200, help="core backward calls per timed window")
    ap.add_argument("--steps", type=int, default=20, help="TrainStep micro-steps per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_deterministic.py: needs a CUDA device")

    import qagnn_b200
    from bench_stream_split import gpu_info
    from oracle import qagnn_oracle as O
    from qagnn_b200 import _lib
    from qagnn_b200 import data as Dt
    from qagnn_b200.modeling_qagnn import GraphPrep
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

    def emit(line):
        print(json.dumps(line), flush=True)
        lines.append(line)

    for bs in args.questions:
        K = flat.max_batch_edges(bs)
        qs = np.arange(bs)
        adj = flat.pack(qs, edge_capacity=K).to(dev)
        nt = ntypes[qs].reshape(-1).to(dev)
        prep = GraphPrep(adj.edge_index, adj.edge_type, nt, T, R, N_NODE, graph_ptr=adj.graph_ptr_dev, max_edges=adj.max_edges)
        for dt in (torch.float32, torch.bfloat16):
            med, spread, same, diff = bench_core(lib, _lib, prep, nt.numel(), dt, args.launches, args.reps, dev)
            emit({"gpu": gpu, "what": "core_backward", "questions": bs, "graphs": bs * NC, "positions": adj.n_edges + nt.numel(),
                  "edge_capacity": K, "D": D, "H": H, "dtype": str(dt).replace("torch.", ""), "launches": args.launches,
                  "reps": args.reps, "default_us": med["default"], "deterministic_us": med["det"],
                  "spread_us": spread, "ratio": med["det"] / med["default"], "d_qkm_bitwise_equal": same,
                  "d_ke_max_abs_diff": diff})
        del prep

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
        steps = {}
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            torch.manual_seed(1)
            dec = qagnn_b200.QAGNN(None, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, D, D, H, D, 0, DROPOUT, DROPOUT, DROPOUT)
            dec.gnn.load_state_dict(O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=0))
            dec = dec.to(dev).train()
            b0 = batches[0]
            steps[det] = TrainStep(dec, b0["sent_vecs"], b0["concept_ids"], b0["node_type_ids"], b0["node_scores"],
                                   b0["adj_lengths"], b0["adj"], max_edges=M, edge_capacity=K)

        def window(det):
            torch.use_deterministic_algorithms(det)
            step = steps[det]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.steps):
                d = batches[i % n_batches]
                logits, _ = step(d["sent_vecs"], d["concept_ids"], d["node_type_ids"], d["node_scores"], d["adj_lengths"], d["adj"])
                torch.nn.functional.cross_entropy(logits.float().view(-1, NC), d["labels"]).backward()
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0) / args.steps

        for det in steps:
            window(det)
        t = {det: [] for det in steps}
        for _ in range(args.reps):
            for det in steps:
                t[det].append(window(det))
        torch.use_deterministic_algorithms(False)
        emit({"gpu": gpu, "what": "train_step", "questions": bs, "graphs": bs * NC, "edge_capacity": K, "D": D, "H": H, "k": K_LAYERS,
              "autocast": "fp32", "steps": args.steps, "reps": args.reps, "default_ms": statistics.median(t[False]),
              "deterministic_ms": statistics.median(t[True]), "spread_ms": {"default": [min(t[False]), max(t[False])],
                                                                          "deterministic": [min(t[True]), max(t[True])]},
              "ratio": statistics.median(t[True]) / statistics.median(t[False])})
        del steps, batches
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
