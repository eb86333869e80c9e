"""ctypes binding of libqagnn_b200.so (include/qagnn_b200.h).

The product path has no CPU or eager-PyTorch fallback: if the shared library is missing this
module raises, it never degrades silently.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libqagnn_b200.so")

OK = 0
STATUS = {0: "ok", -1: "invalid argument", -2: "CUDA error", -3: "index out of range",
          -4: "workspace too small", -5: "unsupported shape"}


class Shape(C.Structure):
    _fields_ = [("N", C.c_int64), ("E", C.c_int64), ("D", C.c_int32), ("H", C.c_int32), ("T", C.c_int32),
                ("R", C.c_int32), ("k", C.c_int32), ("n_per_graph", C.c_int32)]


_P = C.c_void_p


class EdgeEncoderParams(C.Structure):
    _fields_ = [(n, _P) for n in ("lin0_w", "lin0_b", "bn_w", "bn_b", "bn_mean", "bn_var", "lin3_w", "lin3_b")]


class LayerParams(C.Structure):
    _fields_ = [(n, _P) for n in ("key_w", "key_b", "msg_w", "msg_b", "query_w", "query_b", "mlp0_w", "mlp0_b",
                                  "bn_w", "bn_b", "bn_mean", "bn_var", "mlp3_w", "mlp3_b")]


class MPParams(C.Structure):
    _fields_ = [(n, _P) for n in ("emb_node_type_w", "emb_node_type_b", "emb_score_w", "emb_score_b", "vh_w", "vh_b",
                                  "vx_w", "vx_b", "score_basis")]


class PrepLayout(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("total_bytes", "src", "tgt", "combo", "rowptr_src", "rowptr_tgt", "perm_src",
                                          "perm_tgt", "csr_src_tgt", "csr_src_combo", "csr_tgt_src", "csr_tgt_combo",
                                          "csr_tgt_apos", "pk_src", "pk_tgt", "csr_src_tpos", "order_src", "order_tgt", "ninfo_src", "ninfo_tgt",
                                          "status", "scratch")]


EXPORTS = {
    "qagnn_abi_version": (C.c_int32, []),
    "qagnn_status_string": (C.c_char_p, [C.c_int32]),
    "qagnn_last_cuda_error": (C.c_char_p, []),
    "qagnn_graph_prep_layout": (C.c_int32, [C.c_int64, C.c_int64, C.POINTER(PrepLayout)]),
    "qagnn_graph_prep_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "qagnn_graph_prep": (C.c_int32, [_P, _P, _P, C.POINTER(Shape), _P, C.c_size_t, C.c_int32, _P]),
    "qagnn_graph_prep_packed": (C.c_int32, [_P, _P, _P, _P, C.c_int32, C.POINTER(Shape), _P, C.c_size_t, C.c_int32, _P]),
    "qagnn_graph_prep_ragged": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.POINTER(Shape), _P, C.c_size_t,
                                            C.c_int32, _P]),
    "qagnn_fold_bytes": (C.c_size_t, [C.POINTER(Shape)]),
    "qagnn_fold_weights": (C.c_int32, [C.POINTER(Shape), C.POINTER(EdgeEncoderParams), C.POINTER(LayerParams),
                                       C.POINTER(MPParams), _P, C.c_size_t, _P]),
    "qagnn_forward_workspace_bytes": (C.c_size_t, [C.POINTER(Shape)]),
    "qagnn_gatconve_forward": (C.c_int32, [C.POINTER(Shape), C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "qagnn_gatconve_forward_typed": (C.c_int32, [C.POINTER(Shape), C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P,
                                                 _P, _P, C.c_size_t, _P]),
    "qagnn_mp_path": (C.c_int32, [C.POINTER(Shape)]),
    "qagnn_node_feature_extra": (C.c_int32, [C.POINTER(Shape), _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "qagnn_mp_forward": (C.c_int32, [C.POINTER(Shape), _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "qagnn_mp_forward_typed": (C.c_int32, [C.POINTER(Shape), C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t,
                                           _P]),
    "qagnn_gatconve_forward_ragged": (C.c_int32, [C.POINTER(Shape), C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P,
                                                  _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "qagnn_mp_forward_ragged": (C.c_int32, [C.POINTER(Shape), C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                            C.c_size_t, _P]),
    "qagnn_mp_core_forward": (C.c_int32, [C.POINTER(Shape), _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_mp_core_backward": (C.c_int32, [C.POINTER(Shape), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_mp_core_scratch_bytes": (C.c_size_t, [C.POINTER(Shape), C.c_int32]),
    "qagnn_mp_core_forward_typed": (C.c_int32, [C.POINTER(Shape), C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_mp_core_backward_typed": (C.c_int32, [C.POINTER(Shape), C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_mp_core_backward_det_scratch_bytes": (C.c_size_t, [C.POINTER(Shape), C.c_int32]),
    "qagnn_mp_core_backward_det": (C.c_int32, [C.POINTER(Shape), C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                               C.c_size_t, _P]),
    "qagnn_combo_sort_bytes": (C.c_size_t, [C.POINTER(Shape)]),
    "qagnn_combo_sort": (C.c_int32, [C.POINTER(Shape), _P, _P, _P, _P, C.c_size_t, _P]),
    "qagnn_linear_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    "qagnn_linear_bf16x3": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, C.c_int32,
                                        C.c_int64, C.c_int32, C.c_int32, _P, C.c_size_t, _P]),
    "qagnn_linear_bf16": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, C.c_int32, _P,
                                      C.c_int32, C.c_int64, C.c_int32, C.c_int32, _P]),
    "qagnn_attention_pool": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_attention_pool_typed": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P,
                                               _P, _P, _P, _P]),
    "qagnn_decoder_tail": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                       _P, _P]),
    "qagnn_decoder_tail_typed": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P,
                                             _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_decoder_head": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_decoder_head_ragged": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int64, _P, C.c_int64, _P, _P, _P, _P, _P, _P,
                                              _P, _P, _P, _P]),
    "qagnn_decoder_tail_ragged": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int64, _P, _P,
                                              _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_attention_pool_backward_ragged_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "qagnn_attention_pool_backward_ragged": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                         C.c_int64] + [_P] * 16 + [C.c_size_t, _P]),
    "qagnn_assemble_batch": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int64, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int64,
                                         C.c_int64, _P, _P, _P, _P]),
    "qagnn_optim_step": (C.c_int32, [C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_int32, _P, _P, _P, _P, _P, _P, _P,
                                     C.c_int64, _P, _P, _P, _P]),
    "qagnn_clip_grad_norm_slots": (C.c_int64, [C.c_int32, _P]),
    "qagnn_clip_grad_norm": (C.c_int32, [C.c_int32, _P, _P, C.c_double, _P, C.c_int64, _P, _P, _P, _P]),
    "qagnn_step_tail_block_bytes": (C.c_int64, [C.c_int32]),
    "qagnn_step_tail_fill": (C.c_int32, [C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_int64, C.c_double, C.c_double,
                                         C.c_double, C.c_int32, _P, C.c_int64]),
    "qagnn_step_tail": (C.c_int32, [C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P,
                                    _P, C.c_int64, _P, _P, _P, _P, _P, _P, _P]),
    "qagnn_ordered_grad_sum":(C.c_int32, [C.c_int32, _P, _P, _P, _P, _P, C.c_int64, C.c_int32, _P]),
    "qagnn_keyed_dropout_forward_typed": (C.c_int32, [C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_int64, _P, _P,
                                                      C.c_int32, C.c_int32, _P, _P, _P, _P]),
    "qagnn_keyed_dropout_backward_typed": (C.c_int32, [C.c_int32, C.c_int64, C.c_double, _P, _P, _P, _P]),
    "qagnn_schedule_batch": (C.c_int32, [_P, C.c_int64, _P, C.c_int64, C.c_int32, C.c_int64, _P, _P, _P]),
    "qagnn_batch_log": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P]),
    "qagnn_graph_add_child": (C.c_int32, [_P, _P]),
    "qagnn_graph_node_count": (C.c_int64, [_P, C.c_int32]),
    "qagnn_launch_count": (C.c_int64, []),
    "qagnn_profile_enable": (C.c_int32, [C.c_int32]),
    "qagnn_profile_read": (C.c_int32, [C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
}

_lib = None


def load():
    """Loads the C-ABI library (built in-tree by `python -m qagnn_b200.build` / __graft_entry__.build)."""
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build
    if not _build.is_current():
        # library missing (fresh checkout: built artefacts are not in the history) or older than qagnn_b200/csrc: build it
        # when a compiler is around, never run stale code.  Under torchrun every rank gets here at once: one builds under an
        # exclusive file lock, the others wait and re-check.
        import fcntl
        stale = os.path.exists(LIB_PATH)
        try:
            _build._nvcc()
        except RuntimeError:
            raise RuntimeError(
                f"{LIB_PATH} is {'older than qagnn_b200/csrc' if stale else 'missing'} and there is no nvcc to build it. Run "
                f"`python -c 'import __graft_entry__ as g; g.build()'` on a machine with the CUDA toolkit. There is no CPU fallback.") from None
        os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
        with open(LIB_PATH + ".lock", "w") as lock:
            fcntl.flock(lock, fcntl.LOCK_EX)
            try:
                if not _build.is_current():
                    _build.build()
            except Exception as e:  # noqa: BLE001
                raise RuntimeError(f"{LIB_PATH} is {'older than qagnn_b200/csrc' if stale else 'missing'} and could not be "
                                   f"built: {e}. There is no CPU fallback.") from e
            finally:
                fcntl.flock(lock, fcntl.LOCK_UN)
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing after a build. There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype, fn.argtypes = res, args
    if lib.qagnn_abi_version() != 3:
        raise RuntimeError("libqagnn_b200.so ABI version mismatch")
    _lib = lib
    return lib


PROF_STAGES = ("graph_prep", "projection", "message_passing", "node_mlp", "pro_epilogue")


def profile_read():
    """{stage: (ms, intervals)} since the last qagnn_profile_enable(1)."""
    lib = load()
    ms = (C.c_double * len(PROF_STAGES))()
    cnt = (C.c_int64 * len(PROF_STAGES))()
    check(lib.qagnn_profile_read(ms, cnt), "qagnn_profile_read")
    return {n: (ms[i], cnt[i]) for i, n in enumerate(PROF_STAGES)}


class QagnnError(RuntimeError):
    """A library call failed; `status` is its return code (a key of STATUS) when there is one."""

    def __init__(self, msg, status=None):
        super().__init__(msg)
        self.status = status


def check(status, what):
    if status != OK:
        lib = load()
        msg = lib.qagnn_status_string(status).decode()
        if status == -2:
            msg += ": " + lib.qagnn_last_cuda_error().decode()
        if status == -3:
            raise IndexError(f"{what}: {msg}")
        raise QagnnError(f"{what}: {msg} (status {status})", status)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"qagnn_b200: `{name}` must live on a CUDA device (got {t.device}); "
                           f"this implementation has no CPU path")


def f32c(t, name):
    require_cuda(t, name)
    if t.dtype != torch.float32:
        raise TypeError(f"qagnn_b200: `{name}` must be float32 (got {t.dtype})")
    return t.detach().contiguous()


# dtype codes of the *_typed entry points (QAGNN_DTYPE_* in include/qagnn_b200.h)
DTYPE_CODES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def autocast_dtype():
    """The CUDA autocast dtype when autocast is on, else None."""
    return torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else None


def eval_dtype(t, name):
    """(tensor, forward dtype) for an eval forward's input.  Under bf16 autocast: an fp32 or bf16 CUDA tensor as it is (the
    library rounds an fp32 one to bf16 as it writes the GEMM operand, as autocast's cast would) and torch.bfloat16; otherwise
    an fp32 tensor (f32c) and torch.float32.  Any other autocast dtype runs the fp32 kernels."""
    if autocast_dtype() == torch.bfloat16:
        require_cuda(t, name)
        if t.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"qagnn_b200: `{name}` must be float32 or bfloat16 under bf16 autocast (got {t.dtype})")
        return t.detach().contiguous(), torch.bfloat16
    return f32c(t, name), torch.float32


def i64c(t, name):
    require_cuda(t, name)
    if t.dtype != torch.int64:
        raise TypeError(f"qagnn_b200: `{name}` must be int64 (got {t.dtype})")
    return t.contiguous()
