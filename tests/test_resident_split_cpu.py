"""CPU-side checks of a split held on the device (qagnn_b200.data.DeviceSplit, qagnn_assemble_batch): the host batch checks
against FlatAdjCache.pack, the validation at upload, the C entry's argument refusals and what ptxas and cuobjdump report for
the assembly kernels.  A DeviceSplit on the CPU runs the same host code; no GPU needed."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from qagnn_b200 import _lib
from qagnn_b200 import data as Dt

T, R, N, NC = 4, 38, 200, 5


@pytest.fixture(scope="module")
def split():
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        Dt.synth_adj_pickle(path, 10 * NC, seed=21)
        cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N, NC)
    flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr), NC, N)
    return cids, ntypes, scores, lens, flat


def _totals(flat, lens, q):
    gids = (np.asarray(q)[:, None] * NC + np.arange(NC)).reshape(-1)
    return int(np.diff(flat.graph_ptr)[gids].sum()), int(lens.reshape(-1)[gids].sum())


def _outcome(fn):
    try:
        fn()
        return None
    except (IndexError, ValueError) as e:
        return type(e)


@pytest.mark.parametrize("q", [[0, 1, 2], [9, 3, 3], [4], [2, 10], [12], [0, 9, 10 ** 6]])
@pytest.mark.parametrize("k_slack", [None, 0, -1, 25])
@pytest.mark.parametrize("n_slack", [None, 0, -1, 7])
def test_host_checks_accept_and_refuse_as_pack_does(split, q, k_slack, n_slack):
    cids, ntypes, scores, lens, flat = split
    dev = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, "cpu", T, R)
    ok = [i for i in q if i < flat.n_questions()]
    e, rows = _totals(flat, lens, ok) if ok else (0, 0)
    K = None if k_slack is None else e + k_slack
    N_cap = None if n_slack is None else rows + n_slack

    def pack():
        qs = np.asarray(q)
        al = lens[torch.from_numpy(qs)] if n_slack is not None else None  # IndexError for an id past Q, as pack's own gather
        flat.pack(qs, pin=False, edge_capacity=K, adj_lengths=al, node_capacity=N_cap)

    got, ref = _outcome(lambda: dev.check(q, K, N_cap)), _outcome(pack)
    assert got == ref, (got, ref)
    if got is None:
        _, ptr, node_ptr, k, n_cap = dev.check(q, K, N_cap)
        p = flat.pack(np.asarray(q), pin=False, edge_capacity=K, adj_lengths=lens[torch.tensor(q)] if N_cap is not None else None,
                      node_capacity=N_cap)
        assert torch.equal(ptr, p.graph_ptr) and k == p.edge_capacity and n_cap == p.node_capacity
        assert (node_ptr is None) == (p.node_ptr is None)
        if node_ptr is not None:
            assert torch.equal(node_ptr, p.node_ptr)


def test_negative_question_ids_are_refused(split):
    cids, ntypes, scores, lens, flat = split
    dev = Dt.DeviceSplit(flat, cids, ntypes, scores, lens, "cpu", T, R)
    with pytest.raises(IndexError, match="-1"):
        dev.check([0, -1], None)


def _corrupt(split, what, g):
    cids, ntypes, scores, lens, flat = split
    src, tgt, et, lens, ntypes = flat.src.copy(), flat.tgt.copy(), flat.etype.copy(), lens.clone(), ntypes.clone()
    e = int(flat.graph_ptr[g])
    if what == "src":
        src[e] = int(lens.reshape(-1)[g])
    elif what == "tgt":
        tgt[e] = -1
    elif what == "etype":
        et[e] = R
    elif what == "node_type":
        ntypes.reshape(-1, N)[g, 5] = T
    elif what == "adj_length":
        lens.reshape(-1)[g] = 0
    return Dt.FlatAdjCache(src, tgt, et, flat.graph_ptr, NC, N), cids, ntypes, scores, lens


@pytest.mark.parametrize("what", ["src", "tgt", "etype", "node_type", "adj_length"])
def test_a_bad_split_is_refused_at_upload_naming_its_question(split, what):
    g = 23
    with pytest.raises(IndexError, match=f"question {g // NC} "):
        Dt.DeviceSplit(*_corrupt(split, what, g), "cpu", T, R)


def test_assemble_refuses_bad_arguments_before_any_cuda_call():
    lib = _lib.load()
    p = C.c_void_p(64)  # never dereferenced on the host
    args = lambda **kw: [kw.get(k, d) for k, d in (  # noqa: E731
        ("src", p), ("tgt", p), ("etype", p), ("gp", p), ("lens", p), ("G", 50), ("nc", 5), ("n", 200), ("q", p), ("bs", 4),
        ("K", 1000), ("ncap", -1), ("edges", p), ("gpo", p), ("npo", p), ("stream", None))]
    assert lib.qagnn_assemble_batch(*args(bs=0)) == -1
    assert lib.qagnn_assemble_batch(*args(G=52)) == -1          # not a multiple of num_choice
    assert lib.qagnn_assemble_batch(*args(K=-1)) == -1
    assert lib.qagnn_assemble_batch(*args(q=None)) == -1
    assert lib.qagnn_assemble_batch(*args(src=None)) == -1
    assert lib.qagnn_assemble_batch(*args(ncap=100, npo=None)) == -1  # ragged without node_ptr
    assert lib.qagnn_assemble_batch(*args(ncap=100, lens=None)) == -1
    assert lib.qagnn_assemble_batch(*args(ncap=-2)) == -1


def _build_log():
    log = os.path.join(os.path.dirname(_lib.LIB_PATH), "build.log")
    if not os.path.exists(log):
        from qagnn_b200 import build
        build.build()
    return open(log).read()


def test_assembly_kernels_do_not_spill():
    props = re.findall(r"Function properties for \S*assemble_\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", _build_log())
    assert len(props) == 2, "expected the scan and the copy kernel"
    assert all(p == ("0", "0", "0") for p in props), props


def test_assembly_kernels_have_no_atomics():
    tool = next((c for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump") if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("no cuobjdump")
    _build_log()
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    bodies = [b for b in re.split(r"\n\s*Function : ", sass)[1:] if "assemble_" in b.split("\n", 1)[0]]
    assert len(bodies) == 2
    for body in bodies:
        ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", body)
        assert ops and not [op for op in ops if op.split(".")[0] in ("ATOM", "ATOMS", "ATOMG", "RED", "REDG")], body[:80]
