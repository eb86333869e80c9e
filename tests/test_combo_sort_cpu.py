"""CPU-side checks of the combo sort entry points (qagnn_combo_sort): the scratch-size query through ctypes, argument checks
that return before any CUDA call, and the compiler's report for its kernels."""
import ctypes as C
import os
import re

import pytest

from qagnn_b200 import _lib, build

TILE = 4096  # positions per tile of csrc/combo_sort.cu


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_scratch_query_sizes_one_histogram_row_per_tile(lib):
    s = _lib.Shape(64000, 320000, 200, 4, 4, 38, 5, 200)  # cfg2: C = 38*4*4 + 4 = 612 combos
    tiles = -(-(64000 + 320000) // TILE)
    nbytes = lib.qagnn_combo_sort_bytes(C.byref(s))
    assert nbytes % 256 == 0 and tiles * 612 * 4 <= nbytes < tiles * 612 * 4 + 256
    small = _lib.Shape(2000, 0, 200, 4, 4, 38, 5, 200)  # zero edges: one tile
    assert lib.qagnn_combo_sort_bytes(C.byref(small)) == 2560
    assert lib.qagnn_combo_sort_bytes(C.byref(_lib.Shape(0, 10, 200, 4, 4, 38, 5, 0))) == 0
    assert lib.qagnn_combo_sort_bytes(C.byref(_lib.Shape(100, 10, 200, 4, 0, 38, 5, 0))) == 0
    assert lib.qagnn_combo_sort_bytes(C.byref(_lib.Shape(100, 10, 200, 4, 8, 100, 5, 0))) == 0  # C = 6408 > 6144
    assert lib.qagnn_combo_sort_bytes(None) == 0


def test_combo_sort_rejects_bad_arguments_before_touching_the_device(lib):
    s = _lib.Shape(64000, 320000, 200, 4, 4, 38, 5, 200)
    assert lib.qagnn_combo_sort(C.byref(s), None, None, None, None, 0, None) == -1
    p = C.c_void_p(256)  # never dereferenced: the checks below return first
    assert lib.qagnn_combo_sort(C.byref(s), p, p, p, p, 0, None) == -4  # scratch too small
    wide = _lib.Shape(100, 10, 200, 4, 8, 100, 5, 0)
    assert lib.qagnn_combo_sort(C.byref(wide), p, p, p, p, 1 << 20, None) == -5


def test_combo_sort_kernels_do_not_spill(lib):
    log = open(os.path.join(build.LIBDIR, "build.log")).read()
    section = log.split("== combo_sort.cu\n", 1)[1].split("\n== ", 1)[0]
    kernels = re.findall(r"Function properties for \S*(combo_\w+?_kernel)\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", section)
    assert {k for k, *_ in kernels} == {"combo_hist_kernel", "combo_scan_kernel", "combo_scatter_kernel"}, kernels
    for name, stack, st, ld in kernels:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name
