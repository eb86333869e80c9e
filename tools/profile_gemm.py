#!/usr/bin/env python
"""Kernel time of every split-bf16 GEMM (`gemm_tc_kernel`, `mlp_tc_kernel`, `proj_resident_kernel`) of one cfg2 step, beside
its bounds.

    python tools/profile_gemm.py --out DIR [--steps 5]

Runs the benchmark's step (bench.py: cfg2, 320 graphs x 200 nodes x 1000 edges, D = 200, H = 4, k = 5) eagerly under
torch.profiler with CUDA activities, writes the trace to DIR/gemm_trace.json and prints, per GEMM call of a step:
the median kernel time over the profiled steps, the data-sheet tensor and HBM bounds computed from the shapes, and the time
of three cuBLAS BF16 `torch.mm` calls at the same M, N, K (the card's practical tensor ceiling for the three passes).
The calls are told apart by the template arguments <ACT, BN, CTAS> and, for mlp.3 and Vh/Vx (both <2, 208, CTAS>), by
launch order.  The step is profiled twice: with the fused node MLP (`mlp_tc_kernel`, one launch per layer) and with
QAGNN_MLP_FUSED=0 (mlp.0 + mlp.3), so the fused kernel is timed beside the pair at the same shape; the "mlp.0+mlp.3" row
sums the pair's medians and bounds (the pair also writes and reads back the hidden planes).  The projection runs on
`proj_resident_kernel` (<ACT, BN, CTAS> shown as <0, 104, CTAS>); a third profile with QAGNN_PROJ_RESIDENT=0 times it on
`gemm_tc_kernel` as well, in the "proj.gemm_tc" row.  One JSON line with everything follows the table.

    python tools/profile_gemm.py --out DIR --bf16

also profiles the same step under bf16 autocast (DecoderStep(autocast_dtype=torch.bfloat16): the single-pass
`gemm_bf16_kernel` / `mlp_bf16_kernel`) and prints each call's median kernel time in both forms side by side; the JSON line
then carries them under "bf16".
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BF16 = 989e12  # H100 SXM data sheet, dense BF16 (700 W card)
PEAK_HBM = 3.35e12  # H100 SXM data sheet, HBM3

# (M, N, K, output bytes per element) per call of the cfg2 step; K is the GEMM's K (both A segments for Vh/Vx)
N_NODES, D, H, DP = 64000, 200, 4, 52
SHAPES = {
    "emb_score": (N_NODES, D // 2, D // 2, 4),       # bf16 hi + lo planes out
    "projection": (N_NODES, 3 * H * DP, D + D // 2, 4),  # fp32 head-major [3][H][N][DP] out
    "proj.gemm_tc": (N_NODES, 3 * H * DP, D + D // 2, 4),  # the same call on gemm_tc_kernel (QAGNN_PROJ_RESIDENT=0)
    "mlp.0": (N_NODES, D, D, 4),                     # bf16 hi + lo planes out
    "mlp.3": (N_NODES, D, D, 4),                     # bf16 hi + lo planes out
    "Vh/Vx": (N_NODES, D, 2 * D, 4),                 # fp32 out
}
ORDER = ["emb_score", "projection", "proj.gemm_tc", "mlp.0", "mlp.3", "mlp.0+mlp.3", "mlp fused", "Vh/Vx"]


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        info["nvidia_smi"] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        info["nvidia_smi"] = f"unavailable: {exc}"
    return info


def label_calls(kernels):
    """kernels: [(template args, µs)] of one step in launch order -> [(label, µs)]."""
    out, prev = [], None
    for (act, bn, _ctas), us in kernels:
        if bn is None:
            lab = "mlp fused"
        elif act == 0:
            lab = "projection"
        elif act == 1:
            lab = "mlp.0"
        elif bn == 208 and prev == "mlp.0":
            lab = "mlp.3"
        elif bn == 208:
            lab = "Vh/Vx"
        else:
            lab = "emb_score"
        out.append((lab, us))
        prev = lab
    return out


def cublas_ceiling_us(M, N, K, reps=20):
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    c = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        torch.mm(a, b, out=c)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        for _ in range(3):
            torch.mm(a, b, out=c)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def profile_gemms(step, steps, trace, kind="tc"):
    """[(start, (ACT, BN or None for the fused MLP, CTAS), µs)] of the GEMM launches of `steps` eager steps, in launch
    order, and the launches per step.  kind "tc": the split-bf16 kernels; "bf16": the single-pass ones."""
    from torch.profiler import ProfilerActivity, profile
    pat = re.compile(r"gemm_%s_kernel<(\d+), *(\d+), *(\d+)>" % kind)
    pat_mlp = re.compile(r"mlp_%s_kernel<(\d+), *(\d+)>" % kind)
    pat_res = re.compile(r"proj_resident_kernel<(\d+)>") if kind == "tc" else None
    for _ in range(3):
        step.run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step.run()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    kern = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        m, mm = pat.search(e.name), pat_mlp.search(e.name)
        mr = pat_res.search(e.name) if pat_res else None
        if mr:  # the projection (ACT_NONE) on a 104-column resident W slice
            kern.append((e.time_range.start, (0, 104, int(mr.group(1))), e.time_range.elapsed_us()))
        elif m:
            kern.append((e.time_range.start, tuple(int(x) for x in m.groups()), e.time_range.elapsed_us()))
        elif mm:
            act, ctas = (int(x) for x in mm.groups())
            kern.append((e.time_range.start, (act, None, ctas), e.time_range.elapsed_us()))
    kern.sort()
    n = len(kern) // steps
    if n == 0 or len(kern) % steps:
        raise SystemExit(f"profile_gemm.py: {len(kern)} GEMM launches over {steps} steps")
    return kern, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the trace")
    ap.add_argument("--steps", type=int, default=5, help="profiled eager steps")
    ap.add_argument("--bf16", action="store_true", help="also profile the step under bf16 autocast (single-pass GEMMs)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_gemm.py: needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)

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
    step = DecoderStep(mod, pooler, fc, d, 1, None, use_cuda_graph=False, max_edges=max_edges)
    times, templ, per_step = {}, {}, {}
    for fused in ("1", "0"):
        os.environ["QAGNN_MLP_FUSED"] = fused
        kern, n = profile_gemms(step, args.steps, os.path.join(args.out, f"gemm_trace_fused{fused}.json"))
        per_step[fused] = n
        for s in range(args.steps):
            one = kern[s * n:(s + 1) * n]
            for (lab, us), (_, t, _) in zip(label_calls([(t, us) for _, t, us in one]), one):
                if fused == "0" and lab not in ("mlp.0", "mlp.3"):
                    continue  # the other calls are the same kernels in both runs: keep the default run's times
                times.setdefault(lab, []).append(us)
                templ[lab] = t
    os.environ.pop("QAGNN_MLP_FUSED", None)
    os.environ["QAGNN_PROJ_RESIDENT"] = "0"  # the projection on gemm_tc_kernel, in the same process
    kern, n = profile_gemms(step, args.steps, os.path.join(args.out, "gemm_trace_proj_gemm_tc.json"))
    per_step["proj.gemm_tc"] = n
    for s in range(args.steps):
        one = kern[s * n:(s + 1) * n]
        for (lab, us), (_, t, _) in zip(label_calls([(t, us) for _, t, us in one]), one):
            if lab == "projection":
                times.setdefault("proj.gemm_tc", []).append(us)
                templ["proj.gemm_tc"] = t
    os.environ.pop("QAGNN_PROJ_RESIDENT", None)
    if "mlp.0" in times and "mlp.3" in times:  # the pair, call by call
        times["mlp.0+mlp.3"] = [a + b for a, b in zip(times["mlp.0"], times["mlp.3"])]
        templ["mlp.0+mlp.3"] = templ["mlp.0"]

    rows = []
    info = card()
    print(f"card: {info['name']} | nvidia-smi name, power limit, max SM clock: {info['nvidia_smi']}")
    print(f"{'call':<12} {'<ACT,BN,CTAS>':<14} {'calls/step':>10} {'median µs':>10} {'tensor µs':>10} {'HBM µs':>8} "
          f"{'cuBLAS 3x µs':>12} {'TFLOP/s-eq':>10}")
    for lab in ORDER:
        if lab not in times:
            continue
        ts = sorted(times[lab])
        med = ts[len(ts) // 2]
        if lab in ("mlp.0+mlp.3", "mlp fused"):
            M, N, K, ob = SHAPES["mlp.0"]
            flops = 2 * 3 * 2 * M * N * K
            # the pair moves the hidden planes out and back in; the fused kernel reads aggr and writes x only
            hbm = 2 * (M * K * 4 + M * N * ob) if lab == "mlp.0+mlp.3" else M * K * 4 + M * N * ob
            cub = 2 * cublas_ceiling_us(M, N, K)
        else:
            M, N, K, ob = SHAPES[lab]
            flops = 3 * 2 * M * N * K
            hbm = M * K * 4 + M * N * ob
            cub = cublas_ceiling_us(M, N, K)
        row = dict(call=lab, template=list(templ[lab]), calls_per_step=len(ts) // args.steps, median_us=med,
                   min_us=ts[0], max_us=ts[-1], M=M, N=N, K=K, flop_equiv=flops, hbm_bytes=hbm,
                   tensor_bound_us=flops / PEAK_BF16 * 1e6, hbm_bound_us=hbm / PEAK_HBM * 1e6, cublas_3x_us=cub,
                   tflops_equiv=flops / med / 1e6)
        rows.append(row)
        print(f"{lab:<12} {str(tuple(templ[lab])):<14} {row['calls_per_step']:>10} {med:>10.1f} {row['tensor_bound_us']:>10.1f} "
              f"{row['hbm_bound_us']:>8.1f} {cub:>12.1f} {row['tflops_equiv']:>10.1f}")
    total = sum(sum(times[k]) for k in ORDER if k in times and k not in ("mlp.0", "mlp.3", "mlp.0+mlp.3", "proj.gemm_tc")) / args.steps
    print(f"all GEMM launches of the default (fused) step: {total:.1f} µs per step ({per_step['1']} launches; "
          f"{per_step['0']} with QAGNN_MLP_FUSED=0)")
    res = {"card": info, "gemm_us_per_step": total, "launches_per_step": per_step, "calls": rows, "trace_dir": args.out}
    if args.bf16:
        step16 = DecoderStep(mod, pooler, fc, d, 1, None, use_cuda_graph=False, max_edges=max_edges,
                             autocast_dtype=torch.bfloat16)
        kern, n = profile_gemms(step16, args.steps, os.path.join(args.out, "gemm_trace_bf16.json"), "bf16")
        t16 = {}
        for s_ in range(args.steps):
            one = kern[s_ * n:(s_ + 1) * n]
            for lab, us in label_calls([(t, us) for _, t, us in one]):
                t16.setdefault(lab, []).append(us)
        print(f"\nunder bf16 autocast (gemm_bf16_kernel / mlp_bf16_kernel), same card, {n} launches per step")
        print(f"{'call':<11} {'fp32 µs':>10} {'bf16 µs':>10} {'fp32/bf16':>10}")
        cmp_rows = []
        for lab in ORDER:
            if lab not in t16 or lab not in times:
                continue
            m32 = sorted(times[lab])[len(times[lab]) // 2]
            m16 = sorted(t16[lab])[len(t16[lab]) // 2]
            cmp_rows.append(dict(call=lab, fp32_median_us=m32, bf16_median_us=m16, ratio=m32 / m16,
                                 calls_per_step=len(t16[lab]) // args.steps))
            print(f"{lab:<11} {m32:>10.1f} {m16:>10.1f} {m32 / m16:>10.2f}")
        total16 = sum(sum(v) for v in t16.values()) / args.steps
        print(f"all GEMM launches of the bf16 step: {total16:.1f} µs per step (fp32: {total:.1f})")
        res["bf16"] = {"gemm_us_per_step": total16, "launches_per_step": n, "calls": cmp_rows}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
