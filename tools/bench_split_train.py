"""Times a training micro-step of the QAGNN decoder fed three ways, alternated in one process:

  a_host_pack   FlatAdjCache.pack + pinned uploads of the micro-batch on the host, pipeline.TrainStep, then the eager
                loss and backward(): the loop INTEGRATION §1 documents for TrainStep
  b_split_batch DeviceSplit.batch (assembly on the device from the question ids) + TrainStep + eager loss / backward:
                (a) without the host packing
  c_split_step  pipeline.SplitTrainStep: assembly, labels, forward and loss in one graph; backward and the .grad adds in
                another

--loss picks the loss of qagnn.py:208-224.  Routes (a) and (b) take it eagerly in the reference's own form
(tests/answer_oracle.py: nn.CrossEntropyLoss, or the margin-rank loss selected with boolean masks, which reads the device
twice per micro-step); route (c) captures training.answer_loss, which reads nothing.  With margin_rank a fourth route,
d_split_step_ce, runs route (c) with the cross entropy in the same alternation, so the two losses' steps are compared
within one process.

Workload: the loader-shaped synthetic split of tools/bench_train_step.py (n = 200, 38 relations), decoder k = 5, D = 200,
sent_dim 1024, dropout 0.2 (the recipes' values); micro-batches of 2 questions (the recipes' -mbs 2) and 64, under fp16
autocast with a GradScaler (--fp16 true), bf16 autocast and fp32.  sent_vecs is a leaf standing in for the encoder's
output, once requiring grad (encoder unfrozen) and once not (frozen).  Every micro-step's loss is weighted and
back-propagated as qagnn.py:261-265 does.

Per route: wall ms per micro-step (ending in a device synchronise), host ms per micro-step (the enqueue loop before that
synchronise), --reps windows of --steps micro-steps in alternation with medians and spreads, the CUDA launch, copy and
synchronise calls per micro-step from a separate torch.profiler pass, and at -mbs 2 the ms per optimiser batch of 64 questions (32
micro-steps + clip_grad_norm_ + an Adam step + zero_grad).  Before timing, one optimiser batch per precision runs through
the three routes under torch.use_deterministic_algorithms(True) with dropout 0; the script fails when their .grad differ.
Everything it writes goes to --out.

    python tools/bench_split_train.py --out profiles/h100_split_train.jsonl
    python tools/bench_split_train.py --loss margin_rank --out profiles/h100_split_loss.jsonl
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

from tests import answer_oracle as A  # noqa: E402

N_NODE, NC, D, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, DROPOUT = 200, 5, 200, 5, 4, 38, 1024, 2000, 0.2
OPT_BATCH = 64  # questions per optimiser batch (the recipes' -bs 64)
AMPS = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": None}


class Routes:
    """The three ways of running one micro-step on one decoder copy each; `run(route, qids, sv, weight)`."""

    def __init__(self, base, split, host, labels, mbs, K, M, amp, dev, loss):
        from qagnn_b200.pipeline import SplitTrainStep, TrainStep
        self.split, self.host, self.labels, self.K, self.amp, self.dev = split, host, labels, K, amp, dev
        self.loss = loss
        self.dec_ab, self.dec_c = copy.deepcopy(base), copy.deepcopy(base)
        self.scaler = torch.amp.GradScaler("cuda") if amp == torch.float16 else None
        q0 = np.arange(mbs)
        ex = self._host_batch(q0)
        self.train_step = TrainStep(self.dec_ab, torch.zeros(mbs * NC, SENT_DIM, device=dev), *ex[:4], ex[4], max_edges=M,
                                    edge_capacity=K, autocast_dtype=amp)
        self.split_step = SplitTrainStep(self.dec_c, split, mbs, edge_capacity=K, max_edges=M, autocast_dtype=amp,
                                         loss=loss)
        self.decs = {"a_host_pack": self.dec_ab, "b_split_batch": self.dec_ab, "c_split_step": self.dec_c}
        if loss != "cross_entropy":
            self.decs["d_split_step_ce"] = copy.deepcopy(base)
            self.ce_step = SplitTrainStep(self.decs["d_split_step_ce"], split, mbs, edge_capacity=K, max_edges=M,
                                          autocast_dtype=amp)
        self.names = tuple(self.decs)

    def _ac(self):
        return torch.autocast("cuda", dtype=self.amp, cache_enabled=False) if self.amp else torch.autocast("cuda", enabled=False)

    def _host_batch(self, q):
        """Route (a)'s batch: sliced, packed and pinned on the host, uploaded with non-blocking copies."""
        cids, ntypes, scores, lens, flat = self.host
        B = len(q) * NC
        qt = torch.from_numpy(q)
        adj = flat.pack(q, edge_capacity=self.K).to(self.dev, non_blocking=True)
        arrs = [cids[qt].reshape(B, N_NODE), ntypes[qt].reshape(B, N_NODE), scores[qt].reshape(B, N_NODE, 1),
                lens[qt].reshape(B), self.labels[qt]]
        arrs = [a.pin_memory().to(self.dev, non_blocking=True) for a in arrs]
        return arrs[0], arrs[1], arrs[2], arrs[3], adj, arrs[4]

    def _backward(self, loss):
        (self.scaler.scale(loss) if self.scaler is not None else loss).backward()

    def run(self, route, q, sv, weight):
        if route in ("c_split_step", "d_split_step_ce"):
            step = self.split_step if route == "c_split_step" else self.ce_step
            self._backward(step(q, sv) * weight)
            return
        if route == "a_host_pack":
            cid, nt, ns, al, adj, labels = self._host_batch(q)
        else:
            cid, nt, ns, al, adj = self.split.batch(q, self.K)
            labels = self.split.labels[torch.from_numpy(q).to(self.dev, non_blocking=True)]
        logits, _ = self.train_step(sv, cid, nt, ns, al, adj)
        with self._ac():
            loss = A.compute_loss(logits.view(-1, NC), labels, self.loss)
        self._backward(loss * weight)

    def decoder(self, route):
        return self.decs[route]

    def optimiser_batch(self, route, opt, qids, svs, mbs):
        """One optimiser batch of qagnn.py:249-278: micro-steps, clip_grad_norm_, the Adam step, zero_grad."""
        for j, a in enumerate(range(0, len(qids), mbs)):
            self.run(route, qids[a:a + mbs], svs[j % len(svs)], mbs / len(qids))
        params = [p for p in self.decoder(route).parameters() if p.requires_grad]
        if self.scaler is not None:
            self.scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        if self.scaler is not None:
            self.scaler.step(opt)
            self.scaler.update()
        else:
            opt.step()
        opt.zero_grad()


ROUTES = ("a_host_pack", "b_split_batch", "c_split_step")


def make_decoder(dev, dropout):
    import qagnn_b200
    from oracle import qagnn_oracle as O
    torch.manual_seed(1)
    dec = qagnn_b200.QAGNN(None, K_LAYERS, T, R, SENT_DIM, N_CONCEPT, D, D, 2, D, 0, dropout, dropout, dropout)
    dec.gnn.load_state_dict(O.random_state_dict(K_LAYERS, D, T, R, "prod", seed=0))
    for m in dec.modules():  # the pooler's attention dropout included, which the constructor does not set
        if isinstance(m, torch.nn.Dropout):
            m.p = dropout
    return dec.to(dev).train()


def check_equal_grads(split, host, labels, K2, M, dev, loss):
    """One optimiser batch at -mbs 2 through every route under torch.use_deterministic_algorithms(True), dropout 0: the
    routes' .grad must be equal bit for bit.  Returns one result line per precision."""
    lines = []
    was = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    try:
        for name, amp in AMPS.items():
            routes = Routes(make_decoder(dev, 0.0), split, host, labels, 2, K2, M, amp, dev, loss)
            qids = np.random.default_rng(5).permutation(split.n_questions)[:OPT_BATCH]
            g = torch.Generator(device=dev).manual_seed(6)
            grads = {}
            for route in ROUTES:
                routes.scaler = torch.amp.GradScaler("cuda") if amp == torch.float16 else None
                for p in routes.decoder(route).parameters():  # (a) and (b) share a decoder
                    p.grad = None
                for j, a in enumerate(range(0, OPT_BATCH, 2)):
                    g.manual_seed(j)
                    sv = torch.randn(2 * NC, SENT_DIM, device=dev, generator=g).requires_grad_(True)
                    routes.run(route, qids[a:a + 2], sv, 2 / OPT_BATCH)
                grads[route] = {k: p.grad.clone() for k, p in routes.decoder(route).named_parameters() if p.grad is not None}
            ref = grads["a_host_pack"]
            differ = {r: sorted(k for k in ref if k not in grads[r] or not torch.equal(grads[r][k], ref[k])) +
                      sorted(set(grads[r]) - set(ref)) for r in ROUTES[1:]}
            line = {"check": "grad after one optimiser batch, deterministic, dropout 0", "loss": loss, "autocast": name,
                    "params_with_grad": len(ref), "differing": differ, "equal": not any(differ.values())}
            print(json.dumps(line), flush=True)
            lines.append(line)
            del routes
    finally:
        torch.use_deterministic_algorithms(False)
        if was is None:
            os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
        else:
            os.environ["CUBLAS_WORKSPACE_CONFIG"] = was
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, nargs="+", default=[2, 64], help="questions per micro-batch (x5 choices)")
    ap.add_argument("--steps", type=int, default=32, help="micro-steps per timed window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--loss", choices=("cross_entropy", "margin_rank"), default="cross_entropy")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_split_train.py: needs a CUDA device")

    from bench_stream_split import gpu_info
    from qagnn_b200 import data as Dt

    dev = torch.device("cuda:0")
    gpu = gpu_info()
    n_q = max(max(args.questions) * 4, OPT_BATCH)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "split.graph.adj.pk")
        Dt.synth_adj_pickle(path, n_q * NC, seed=args.seed)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N_NODE, NC)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC, N_NODE)
    cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)
    labels = torch.from_numpy(np.random.default_rng(args.seed).integers(0, NC, n_q))
    split = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, dev, T, R, labels=labels)
    host = (cids, ntypes, scores, lens, flat)
    M = flat.max_graph_edges()
    lines = check_equal_grads(split, host, labels, flat.max_batch_edges(2), M, dev, args.loss)
    if not all(line["equal"] for line in lines):
        raise SystemExit("bench_split_train.py: the routes' .grad differ under deterministic mode")

    from torch.profiler import ProfilerActivity, profile
    for mbs in args.questions:
        K = flat.max_batch_edges(mbs)
        order = np.random.default_rng(args.seed + mbs).permutation(n_q)
        micro = [order[i * mbs:(i + 1) * mbs] for i in range(len(order) // mbs)]
        for name, amp in AMPS.items():
            base = make_decoder(dev, DROPOUT)
            routes = Routes(base, split, host, labels, mbs, K, M, amp, dev, args.loss)
            for frozen in (False, True):
                g = torch.Generator(device=dev).manual_seed(mbs)
                svs = [torch.randn(mbs * NC, SENT_DIM, device=dev, generator=g).requires_grad_(not frozen) for _ in range(4)]

                def window(route):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for i in range(args.steps):
                        routes.run(route, micro[i % len(micro)], svs[i % len(svs)], 0.5)
                    t1 = time.perf_counter()
                    torch.cuda.synchronize()
                    return (time.perf_counter() - t0) / args.steps, (t1 - t0) / args.steps

                for route in routes.names:  # warm-up
                    window(route)
                samples = {r: [] for r in routes.names}
                for _ in range(args.reps):
                    for route in routes.names:
                        samples[route].append(window(route))
                res = {}
                for route in routes.names:
                    wall = [s[0] for s in samples[route]]
                    res[route] = {"ms_per_step": 1e3 * statistics.median(wall), "spread_ms": [1e3 * min(wall), 1e3 * max(wall)],
                                  "host_ms_per_step": 1e3 * statistics.median(s[1] for s in samples[route])}
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                        for i in range(args.steps):
                            routes.run(route, micro[i % len(micro)], svs[i % len(svs)], 0.5)
                        torch.cuda.synchronize()
                    launches = copies = syncs = 0
                    for e in prof.events():
                        if e.device_type == torch.autograd.DeviceType.CUDA:
                            continue
                        if e.name.startswith(("cudaLaunchKernel", "cuLaunchKernel", "cudaGraphLaunch", "cudaLaunchKernelExC")):
                            launches += 1
                        elif e.name.startswith("cudaMemcpy"):
                            copies += 1
                        elif e.name.startswith(("cudaStreamSynchronize", "cudaDeviceSynchronize")):
                            syncs += 1
                    res[route]["launch_calls_per_step"] = launches / args.steps
                    res[route]["copy_calls_per_step"] = copies / args.steps
                    # the one device synchronise that ends the profiled window is not a micro-step's
                    res[route]["sync_calls_per_step"] = max(syncs - 1, 0) / args.steps
                if mbs == 2:  # an optimiser batch of the recipes: 32 micro-steps of 2 questions
                    opts = {r: torch.optim.Adam([p for p in routes.decoder(r).parameters() if p.requires_grad], lr=1e-5)
                            for r in routes.names}
                    qids = order[:OPT_BATCH]
                    for route in routes.names:  # warm-up (the optimiser state)
                        routes.optimiser_batch(route, opts[route], qids, svs, mbs)
                    times = {r: [] for r in routes.names}
                    for _ in range(args.reps):
                        for route in routes.names:
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            routes.optimiser_batch(route, opts[route], qids, svs, mbs)
                            torch.cuda.synchronize()
                            times[route].append(time.perf_counter() - t0)
                    for route in routes.names:
                        t = times[route]
                        res[route]["ms_per_optimiser_batch"] = 1e3 * statistics.median(t)
                        res[route]["optimiser_batch_spread_ms"] = [1e3 * min(t), 1e3 * max(t)]
                line = {"gpu": gpu, "loss": args.loss, "questions": mbs, "graphs": mbs * NC, "n_node": N_NODE, "D": D, "k": K_LAYERS,
                        "autocast": name, "sent_vecs_requires_grad": not frozen, "edge_capacity": K, "max_graph_edges": M,
                        "steps": args.steps, "reps": args.reps, **res,
                        "speedup_c_vs_a": res["a_host_pack"]["ms_per_step"] / res["c_split_step"]["ms_per_step"],
                        "speedup_c_vs_b": res["b_split_batch"]["ms_per_step"] / res["c_split_step"]["ms_per_step"]}
                print(json.dumps(line), flush=True)
                lines.append(line)
            del routes, base
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
