#!/usr/bin/env python
"""Times the wgmma split-bf16 GEMM on the hot-path shapes and checks it against an fp64 matmul."""
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qagnn_b200 import ops  # noqa: E402

dev = "cuda:0"
torch.manual_seed(0)
for (M, K1, K2, N, act) in [(64000, 200, 200, 600, "none"), (64000, 200, 0, 200, "relu"), (64000, 200, 200, 200, "gelu"),
                            (1000, 64, 64, 192, "none"), (333, 72, 0, 40, "gelu")]:
    a1 = torch.randn(M, K1, device=dev) * 0.5
    a2 = torch.randn(M, K2, device=dev) * 0.5 if K2 else None
    w = torch.randn(N, K1 + K2, device=dev) / (K1 + K2) ** 0.5
    b = torch.randn(N, device=dev) * 0.1
    out = ops.linear_bf16x3(a1, w, b, a2, act)
    A = torch.cat([a1, a2], 1) if K2 else a1
    ref = A.double() @ w.double().t() + b.double()
    if act == "relu":
        ref = ref.relu()
    if act == "gelu":
        ref = torch.nn.functional.gelu(ref, approximate="tanh")
    err = (out.double() - ref).abs().max().item()
    err32 = ((A @ w.t() + b).double() - (A.double() @ w.double().t() + b.double())).abs().max().item()
    for _ in range(3):
        ops.linear_bf16x3(a1, w, b, a2, act)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        ops.linear_bf16x3(a1, w, b, a2, act)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print(f"M={M} K={K1}+{K2} N={N} act={act}: max|err| {err:.2e} (torch fp32 matmul: {err32:.2e}); {ms*1e3:.1f} us incl. operand split "
          f"({2*M*(K1+K2)*N/ms/1e9:.1f} TFLOP/s effective)")
