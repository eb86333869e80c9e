"""CPU-side checks of training in the autocast dtype: the dtype-carrying core entry points refuse bad arguments before any
CUDA call and size their scratch, the core picks its storage dtype from its operands, and TrainStep takes bf16."""
import ctypes as C

import pytest
import torch

from qagnn_b200 import _lib
from qagnn_b200 import training as TR
from qagnn_b200.pipeline import TrainStep


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_dtype_codes_match_the_header():
    import os
    import re
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "qagnn_b200.h")).read()
    codes = dict((n, int(v)) for n, v in re.findall(r"QAGNN_DTYPE_(F32|F16|BF16) = (\d+)", header))
    assert codes == {"F32": _lib.DTYPE_CODES[torch.float32], "F16": _lib.DTYPE_CODES[torch.float16],
                     "BF16": _lib.DTYPE_CODES[torch.bfloat16]}


def test_scratch_bytes_cover_ds_and_the_fp32_table_accumulators(lib):
    N, E, D, H, T, R = 64000, 250000, 200, 4, 4, 38
    s = _lib.Shape(N, E, D, H, T, R, 1, 0)
    ds = (N + E) * H * 4
    f32 = lib.qagnn_mp_core_scratch_bytes(C.byref(s), 0)
    assert ds <= f32 < ds + 256 and f32 % 256 == 0
    Cn = R * T * T + T
    for code in (1, 2):
        assert lib.qagnn_mp_core_scratch_bytes(C.byref(s), code) == f32 + 2 * Cn * D * 4
    assert lib.qagnn_mp_core_scratch_bytes(C.byref(s), 3) == 0
    assert lib.qagnn_mp_core_scratch_bytes(C.byref(_lib.Shape(N, E, D, 3, T, R, 1, 0)), 1) == 0  # D % H != 0


def test_typed_entry_points_refuse_before_any_cuda_call(lib):
    s = _lib.Shape(100, 300, 64, 4, 4, 38, 1, 0)
    p = C.c_void_p(256)  # never dereferenced: every refusal comes before a launch
    assert lib.qagnn_mp_core_forward_typed(C.byref(s), 3, p, p, p, p, p, p, None, p, None) == -1
    assert lib.qagnn_mp_core_forward_typed(C.byref(s), -1, p, p, p, p, p, p, None, p, None) == -1
    assert lib.qagnn_mp_core_forward_typed(C.byref(s), 2, p, None, p, p, p, p, None, p, None) == -1
    assert lib.qagnn_mp_core_backward_typed(C.byref(s), 7, p, p, p, p, p, p, p, p, p, p, p, None) == -1
    assert lib.qagnn_mp_core_backward_typed(C.byref(s), 1, p, p, p, p, p, p, p, p, p, None, p, None) == -1
    bad = _lib.Shape(100, 300, 64, 3, 4, 38, 1, 0)
    assert lib.qagnn_mp_core_forward_typed(C.byref(bad), 1, p, p, p, p, p, p, None, p, None) == -1


def test_core_storage_dtype_is_the_widest_operand_dtype():
    h, b, f = (torch.zeros(2, dtype=dt) for dt in (torch.float16, torch.bfloat16, torch.float32))
    assert TR._core_dtype(h, h, h) == torch.float16
    assert TR._core_dtype(b, b, b) == torch.bfloat16
    assert TR._core_dtype(h, f, h) == torch.float32
    assert TR._core_dtype(h, b, h) == torch.float32  # neither 16-bit type holds the other
    with pytest.raises(TypeError, match="float32, float16 or bfloat16"):
        TR._core_dtype(torch.zeros(2, dtype=torch.float64), f, f)


def test_train_step_accepts_bf16_and_refuses_other_autocast_dtypes():
    with pytest.raises(ValueError, match="None, torch.float16 or torch.bfloat16"):
        TrainStep(None, None, None, None, None, None, None, max_edges=1, autocast_dtype=torch.float64)
    # bf16 passes the dtype check and reaches the decoder (None here)
    with pytest.raises(AttributeError):
        TrainStep(None, None, None, None, None, None, None, max_edges=1, autocast_dtype=torch.bfloat16)
