"""Thin Python wrappers over stand-alone C-ABI ops (diagnostics and tests)."""
import torch

from . import _lib


def linear_bf16x3(a1, weight, bias=None, a2=None, act="none"):
    """act([a1 | a2] @ weight^T + bias) through the wgmma split-bf16 (3-pass) GEMM.  fp32 CUDA tensors."""
    lib = _lib.load()
    a1 = _lib.f32c(a1, "a1")
    w = _lib.f32c(weight, "weight")
    a2c = _lib.f32c(a2, "a2") if a2 is not None else None
    b = _lib.f32c(bias, "bias") if bias is not None else None
    M, K1 = a1.shape
    K2 = a2c.shape[1] if a2c is not None else 0
    N = w.shape[0]
    if w.shape[1] != K1 + K2:
        raise ValueError("weight must be [N, K1+K2]")
    out = torch.empty(M, N, dtype=torch.float32, device=a1.device)
    nbytes = lib.qagnn_linear_workspace_bytes(M, N, K1, K2)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=a1.device)
    code = {"none": 0, "relu": 1, "gelu": 2}[act]
    with torch.cuda.device(a1.device):
        st = lib.qagnn_linear_bf16x3(_lib.ptr(a1), K1, K1, _lib.ptr(a2c), K2, K2, _lib.ptr(w), K1 + K2, _lib.ptr(b),
                                     _lib.ptr(out), N, M, N, code, _lib.ptr(ws), nbytes, _lib.stream_ptr(a1.device))
    _lib.check(st, "qagnn_linear_bf16x3")
    return out


def _bf16c(t, name):
    _lib.require_cuda(t, name)
    if t.dtype != torch.bfloat16:
        raise TypeError(f"qagnn_b200: `{name}` must be bfloat16 (got {t.dtype})")
    return t.detach().contiguous()


def linear_bf16(a1, weight, bias=None, a2=None, act="none", out_dtype=torch.float32):
    """act([a1 | a2] @ weight^T + bias) through the single-pass bf16 wgmma GEMM of the bf16 eval forward: bf16 a1 / a2 /
    weight, fp32 bias, fp32 accumulation.  Returns fp32, or with out_dtype=torch.bfloat16 that value rounded to nearest
    even (the GEMM's bf16 plane output)."""
    lib = _lib.load()
    a1 = _bf16c(a1, "a1")
    w = _bf16c(weight, "weight")
    a2c = _bf16c(a2, "a2") if a2 is not None else None
    b = _lib.f32c(bias, "bias") if bias is not None else None
    M, K1 = a1.shape
    K2 = a2c.shape[1] if a2c is not None else 0
    N = w.shape[0]
    if w.shape[1] != K1 + K2:
        raise ValueError("weight must be [N, K1+K2]")
    if out_dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("out_dtype must be torch.float32 or torch.bfloat16")
    out = torch.empty(M, N, dtype=out_dtype, device=a1.device)
    f32, pl = (out, None) if out_dtype == torch.float32 else (None, out)
    code = {"none": 0, "relu": 1, "gelu": 2}[act]
    with torch.cuda.device(a1.device):
        st = lib.qagnn_linear_bf16(_lib.ptr(a1), K1, K1, _lib.ptr(a2c), K2, K2, _lib.ptr(w), K1 + K2, _lib.ptr(b), _lib.ptr(f32),
                                   N, _lib.ptr(pl), N, M, N, code, _lib.stream_ptr(a1.device))
    _lib.check(st, "qagnn_linear_bf16")
    return out
