"""Host-side contract of qagnn_mp_core_backward_det: the scratch query and the argument checks, which return before any
device work (so no GPU is needed)."""
import ctypes as C

import pytest

from qagnn_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _shape(N=64000, E=320000, D=200, H=4):
    return _lib.Shape(N, E, D, H, 4, 38, 1, 0)


def test_scratch_bytes_cover_the_default_scratch_and_the_run_slots(lib):
    s = _shape()
    for code in (0, 1, 2):
        default = lib.qagnn_mp_core_scratch_bytes(C.byref(s), code)
        det = lib.qagnn_mp_core_backward_det_scratch_bytes(C.byref(s), code)
        runs = (s.N + s.E + 63) // 64
        assert det >= default + 4 * (612 + 2 * runs * 2 * s.D)
    assert lib.qagnn_mp_core_backward_det_scratch_bytes(C.byref(s), 3) == 0
    assert lib.qagnn_mp_core_backward_det_scratch_bytes(C.byref(_shape(D=202, H=4)), 0) == 0  # D % H != 0


def test_too_small_scratch_and_bad_arguments_are_refused(lib):
    s = _shape(N=300, E=1200)
    need = lib.qagnn_mp_core_backward_det_scratch_bytes(C.byref(s), 0)
    p = C.c_void_p(256)  # never dereferenced: every check below returns first
    args = [p] * 12

    def call(dtype, scratch_bytes, ptrs=args):
        return lib.qagnn_mp_core_backward_det(C.byref(s), dtype, *ptrs, scratch_bytes, None)

    assert call(0, need - 1) == -4  # QAGNN_ERR_WORKSPACE
    assert call(5, need) == -1      # unknown dtype
    assert call(0, need, [p] * 3 + [None] + [p] * 8) == -1  # combo_count missing
