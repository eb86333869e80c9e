"""Host-side contracts of pipeline.SplitTrainBatchGraph and csrc/schedule.cu, no GPU needed: a numpy restatement of
qagnn_schedule_batch's id layout and status bits against the chunks SplitTrainBatch takes, the fp64 order of qagnn_batch_log
against Python's `total_loss += loss.item()`, the refusals raised before anything reaches a device, and the SASS listing
of schedule.cu's kernels for sm_90a."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from qagnn_b200 import _lib, optim, pipeline
from qagnn_b200.pipeline import SplitTrainBatchGraph, train_chunks
from tests.test_split_train_batch_cpu import _decoder, _tb, split  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def schedule(order, counter, bs, mbs, n_questions):
    """qagnn_schedule_batch restated: (ids [n_full], status bits)."""
    n_full = bs // mbs * mbs
    in_epoch = 0 <= counter < len(order) // bs
    status = 0 if in_epoch else pipeline.SCHEDULE_PAST_EPOCH
    ids = np.asarray(order[counter * bs:counter * bs + n_full] if in_epoch else np.zeros(n_full), dtype=np.int64).copy()
    bad = (ids < 0) | (ids >= n_questions)
    if bad.any():
        status |= pipeline.SCHEDULE_BAD_ID
        ids[bad] = 0
    return ids, status


@pytest.mark.parametrize("bs,mbs,branches", [(64, 2, 8), (128, 1, 32), (6, 1, 4), (2, 2, 2), (12, 3, 3)])
def test_the_schedules_rows_are_the_chunks_of_split_train_batch(bs, mbs, branches):
    order = np.random.default_rng(bs).permutation(5 * bs)
    for counter in range(5):
        ids, status = schedule(order, counter, bs, mbs, 5 * bs)
        assert status == 0
        n_chunks = -(-(bs // mbs) // branches)
        block = np.zeros((n_chunks * branches, mbs), dtype=np.int64)  # the graph's [chunks * branches, mbs] id rows
        block.reshape(-1)[:ids.size] = ids
        chunks = train_chunks(order[counter * bs:(counter + 1) * bs], mbs, branches)
        assert len(chunks) == n_chunks
        for c, chunk in enumerate(chunks):  # chunk c's copy into the branches' rows reads block[c * S : c * S + n]
            assert np.array_equal(block[c * branches:c * branches + len(chunk)], np.stack(chunk))


def test_the_status_bits_flag_a_bad_id_and_a_counter_past_the_epoch():
    order = np.arange(10)
    order[6] = 99
    assert schedule(order, 0, 4, 2, 10)[1] == 0
    ids, st = schedule(order, 1, 4, 2, 10)
    assert st == pipeline.SCHEDULE_BAD_ID and list(ids) == [4, 5, 0, 7]
    ids, st = schedule(order, 2, 4, 2, 10)  # 10 // 4 = 2 full batches
    assert st == pipeline.SCHEDULE_PAST_EPOCH and not ids.any()
    assert schedule(order, -1, 4, 2, 10)[1] == pipeline.SCHEDULE_PAST_EPOCH


def test_the_status_bits_are_the_headers_and_above_graph_preps():
    text = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    bits = {m.group(1): 1 << int(m.group(2)) for m in re.finditer(r"QAGNN_SCHEDULE_(\w+) = 1 << (\d+)", text)}
    assert bits == {"BAD_ID": pipeline.SCHEDULE_BAD_ID, "PAST_EPOCH": pipeline.SCHEDULE_PAST_EPOCH}
    assert min(bits.values()) > 1 << 8  # graph prep's status bits are the low ones


def batch_log(losses, mbs, bs, total=0.0):
    """qagnn_batch_log restated: fp32 (loss * mbs) * (1 / bs), each product rounded, added in order in fp64."""
    inv = np.float32(1.0) / np.float32(bs)
    for x in np.asarray(losses, dtype=np.float32):
        total += float(np.float32(np.float32(x * np.float32(mbs)) * inv))
    return total


@pytest.mark.parametrize("mbs,bs", [(2, 64), (1, 128), (1, 6), (3, 12)])
def test_the_log_adds_in_micro_batch_order_as_python_does(mbs, bs):
    losses = np.random.default_rng(bs).uniform(0.1, 3.0, bs // mbs).astype(np.float32)
    weighted = [float(np.float32(np.float32(x * np.float32(mbs)) * (np.float32(1) / np.float32(bs)))) for x in losses]
    total = 0.0
    for w in weighted:  # total_loss += loss.item()
        total += w
    assert batch_log(losses, mbs, bs) == total


def test_the_log_order_is_observable():
    """Python's left-to-right double sum differs from other orders for some inputs, so the order is part of the contract."""
    rng = np.random.default_rng(0)
    for _ in range(1000):
        losses = rng.uniform(0, 1e4, 8).astype(np.float32) * rng.choice([1e-6, 1.0, 1e3], 8).astype(np.float32)
        if batch_log(losses, 1, 8) != batch_log(losses[::-1], 1, 8):
            return
    pytest.fail("no input showed the order")


def test_construction_refusals(split):
    flat, s = split
    with pytest.raises(ValueError, match="SplitTrainBatch"):
        SplitTrainBatchGraph(object(), 4)
    quiet = _decoder()
    for m in quiet.modules():  # the pooler's attention dropout included, which the constructor sets to 0.1
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    tb = _tb(split, dec=quiet)
    with pytest.raises(ValueError, match="multiple"):
        SplitTrainBatchGraph(tb, 5)
    with pytest.raises(ValueError, match="multiple"):
        SplitTrainBatchGraph(tb, 1)
    with pytest.raises(ValueError, match="edge capacity"):
        SplitTrainBatchGraph(_tb(split, edge_capacity=flat.max_batch_edges(2) - 1), 4)
    with pytest.raises(ValueError, match="DropoutKey"):
        SplitTrainBatchGraph(_tb(split), 4)
    params = [p for p in tb.decoder.parameters() if p.requires_grad]
    tail = optim.CapturedTail(optim.RAdam(params), torch.amp.GradScaler("cpu"))
    with pytest.raises(ValueError, match="scaler"):
        SplitTrainBatchGraph(tb, 4, tail=tail)


def test_the_split_and_the_flat_cache_agree_on_the_edge_capacity(split):
    flat, s = split
    for mbs in (1, 2, 3, 100):
        assert s.max_batch_edges(mbs) == flat.max_batch_edges(mbs)


def test_the_c_entries_refuse_bad_arguments_without_a_device():
    lib = _lib.load()
    buf = (C.c_int64 * 4)()
    st = (C.c_int32 * 1)()
    p, s = C.cast(buf, C.c_void_p), C.cast(st, C.c_void_p)
    bad = -1  # QAGNN_ERR_INVALID_ARGUMENT
    assert lib.qagnn_schedule_batch(None, 4, p, 4, 2, 10, p, s, None) == bad
    assert lib.qagnn_schedule_batch(p, 4, p, 4, 5, 10, p, s, None) == bad  # mbs > bs
    assert lib.qagnn_schedule_batch(p, 4, p, 0, 1, 10, p, s, None) == bad
    assert lib.qagnn_schedule_batch(p, 4, p, 4, 2, 0, p, s, None) == bad
    assert lib.qagnn_batch_log(p, 0, 1, 4, p, p, None) == bad
    assert lib.qagnn_batch_log(None, 2, 1, 4, p, p, None) == bad
    assert lib.qagnn_graph_add_child(None, None) == bad
    assert lib.qagnn_graph_node_count(None, 0) == -1


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_the_schedule_kernels_are_built_for_sm_90a():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    _lib.load()  # builds the library when it is missing or stale
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = {}
    for section in re.split(r"Fatbin elf code:", sass)[1:]:
        arch = re.search(r"arch = (\w+)", section).group(1)
        for name in re.findall(r"Function : (\S+)", section):
            for k in ("schedule_batch_kernel", "batch_log_kernel"):
                if k in name:
                    found.setdefault(k, set()).add(arch)
    assert found == {"schedule_batch_kernel": {"sm_90a"}, "batch_log_kernel": {"sm_90a"}}
