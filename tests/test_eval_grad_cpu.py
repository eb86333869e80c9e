"""CPU-side checks of the eval-mode gradient path: which calls take it, the ragged pooling backward's C entry points refusing
what the kernels do not take, and ptxas's report on the new kernels.  No GPU needed."""
import ctypes as C
import os
import re

import pytest
import torch

import qagnn_b200
from qagnn_b200 import _lib
from qagnn_b200.modeling_qagnn import _refuse_ragged_training, _wants_autograd


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        from qagnn_b200 import build
        build.build()
    return _lib.load()


def test_eval_calls_take_the_autograd_path_only_when_an_input_wants_a_gradient():
    mod = qagnn_b200.QAGNN_Message_Passing(None, 1, 4, 38, 16, 16, 16).eval()
    x, y = torch.zeros(2, 16), torch.zeros(2, 16, requires_grad=True)
    assert not _wants_autograd(mod, x, None)
    assert _wants_autograd(mod, x, y)
    with torch.no_grad():
        assert not _wants_autograd(mod, x, y)
    assert _wants_autograd(mod.train(), x, None)


def test_a_ragged_batch_is_refused_in_training_only():
    mod = qagnn_b200.QAGNN_Message_Passing(None, 1, 4, 38, 16, 16, 16)
    _refuse_ragged_training(mod.eval(), "QAGNN_Message_Passing")
    with pytest.raises(ValueError, match="eval"):
        _refuse_ragged_training(mod.train(), "QAGNN_Message_Passing")


def test_pool_backward_scratch_and_argument_refusals(lib):
    B, n, D, nh = 320, 200, 200, 2
    assert lib.qagnn_attention_pool_backward_ragged_scratch_bytes(B, n, D, nh) == 4 * (4 * B * nh * D + nh * B * n + B * nh)
    assert lib.qagnn_attention_pool_backward_ragged_scratch_bytes(B, n, 10, 4) == 0  # D % n_head != 0
    assert lib.qagnn_attention_pool_backward_ragged_scratch_bytes(0, n, D, nh) == 0
    p = [C.c_void_p(64)] * 16
    nbytes = lib.qagnn_attention_pool_backward_ragged_scratch_bytes(B, n, D, nh)
    # the pointers are never dereferenced on the host: every refusal comes before a CUDA call
    assert lib.qagnn_attention_pool_backward_ragged(0, B, n, 216, 9, 8, 1000, *p, nbytes, None) == -5  # > 8 heads
    assert lib.qagnn_attention_pool_backward_ragged(0, B, n, 10, 4, 8, 1000, *p, nbytes, None) == -1  # D % n_head
    assert lib.qagnn_attention_pool_backward_ragged(1, B, n, D, nh, 8, 1000, *p, nbytes, None) == -1  # fp16 X
    assert lib.qagnn_attention_pool_backward_ragged(0, B, n, D, nh, 8, 0, *p, nbytes, None) == -1     # no rows
    assert lib.qagnn_attention_pool_backward_ragged(0, B, n, D, nh, 8, 1000, *p[:15], None, nbytes, None) == -1
    assert lib.qagnn_attention_pool_backward_ragged(0, B, n, D, nh, 8, 1000, *p, nbytes - 4, None) == -4


def test_pool_backward_kernels_do_not_spill():
    log = os.path.join(os.path.dirname(_lib.LIB_PATH), "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log")
    text = open(log).read()
    props = re.findall(r"Function properties for \S*pool_backward_\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", text)
    assert len(props) == 4, "expected the head kernel (fp32 and bf16 X), the rows kernel and the weights kernel"
    assert all(int(s) == 0 and int(st) == 0 and int(ld) == 0 for s, st, ld in props), props
