#!/usr/bin/env python
"""The eval step in fp32 against the same step under bf16 autocast (single-pass bf16 GEMMs), on the benchmark's workload.

    python tools/bench_eval_bf16.py [--windows 7] [--steps 50] [--out FILE]

Workload: bench.py's cfg2 step (320 graphs x 200 nodes x 1000 edges, D = 200, H = 4, k = 5, pooling and answer MLP) with
its generator, seeds and production-init weights.  Both forms run as captured DecoderSteps over the same device buffers and
are timed alternately in one process: per window, each form replays `--steps` steps between two CUDA events; the result is
the median over the windows.  Accuracy: the largest |logit difference| between the two forms and the fraction of the 64
questions (5 choices each) whose argmax agrees.  The card's name, power limit and maximum SM clock are read in the same run.
Prints one JSON line (also appended to --out when given).  Per-call GEMM kernel times: tools/profile_gemm.py --bf16.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from profile_gemm import card  # noqa: E402  (the card's name, power limit and maximum SM clock)


def time_window(step, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step.run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=50, help="replays per window and form")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="append the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_bf16.py: needs a CUDA device")

    import bench
    import qagnn_b200
    from qagnn_b200.pipeline import DecoderStep
    from oracle import qagnn_oracle as O

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    C = bench.CFG
    inp = bench.synth_step_inputs(0)
    sd = O.random_state_dict(C["k"], C["D"], C["T"], C["R"], "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, C["k"], C["T"], C["R"], C["D"], C["D"], C["D"]).eval()
    mod.load_state_dict(sd)
    mod = mod.to(dev)
    pooler, fc = bench.build_decoder_tail(C["D"], bench.SENT_DIM, dev)
    d = {k: inp[k].to(dev) for k in DecoderStep.PACKED_FIELDS}
    max_edges = int((inp["graph_ptr"][1:] - inp["graph_ptr"][:-1]).max())
    steps = {"fp32": DecoderStep(mod, pooler, fc, d, 1, None, max_edges=max_edges),
             "bf16": DecoderStep(mod, pooler, fc, d, 1, None, max_edges=max_edges, autocast_dtype=torch.bfloat16)}
    assert all(s.graph is not None for s in steps.values()), "both forms must be captured"

    logits = {}
    for name, s in steps.items():
        lg, _, out = s.run()
        torch.cuda.synchronize()
        logits[name] = lg.float().view(-1, 5).cpu()  # 64 questions x 5 choices
        assert out.dtype == (torch.float32 if name == "fp32" else torch.bfloat16)
    diff = (logits["fp32"] - logits["bf16"]).abs().max().item()
    agree = (logits["fp32"].argmax(1) == logits["bf16"].argmax(1)).double().mean().item()

    for s in steps.values():
        for _ in range(args.warmup):
            s.run()
    torch.cuda.synchronize()
    ms = {name: [] for name in steps}
    for w in range(args.windows):  # alternate the forms, and which goes first
        order = list(steps) if w % 2 == 0 else list(steps)[::-1]
        for name in order:
            ms[name].append(time_window(steps[name], args.steps))
    med = {name: sorted(v)[len(v) // 2] for name, v in ms.items()}
    res = {"what": "eval DecoderStep (captured), cfg2: fp32 vs bf16 autocast", "card": card(),
           "windows": args.windows, "steps_per_window": args.steps,
           "ms_per_step_median": med, "ms_per_step_windows": ms,
           "speedup_fp32_over_bf16": med["fp32"] / med["bf16"],
           "max_abs_logit_diff": diff, "argmax_agreement": agree, "questions": logits["fp32"].size(0)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
