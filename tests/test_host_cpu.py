"""CPU-side checks: the C-ABI library loads and exports every symbol the header declares (no
compute calls without a GPU), layout queries, module/state_dict contract, batch packing."""
import ctypes as C
import os
import re

import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import _lib
from qagnn_b200.data import pack_adj

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        from qagnn_b200 import build
        build.build()
    return _lib.load()


def test_header_symbols_are_exported(lib):
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    declared = set(re.findall(r"\b(qagnn_[a-z_0-9]+)\s*\(", header))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/qagnn_b200.h but not exported"
    assert declared == set(_lib.EXPORTS), "ctypes binding and header disagree"
    assert lib.qagnn_abi_version() == 3
    assert lib.qagnn_status_string(-3).decode().startswith("index out of range")


def _c_kind(decl):
    """Coarse ctypes class of one C parameter / return type as written in the header."""
    decl = re.sub(r"/\*.*?\*/", "", decl).strip()
    if "*" in decl:
        return "char*" if re.match(r"(const\s+)?char\s*\*", decl) else "ptr"
    for t in ("int64_t", "int32_t", "size_t", "double", "float"):
        if re.search(rf"\b{t}\b", decl):
            return t
    raise AssertionError(f"unparsed C type: {decl!r}")


def _ctypes_kind(t):
    if t is C.c_char_p:
        return "char*"
    if t is C.c_void_p or (isinstance(t, type) and issubclass(t, C._Pointer)):
        return "ptr"
    return {C.c_int64: "int64_t", C.c_int32: "int32_t", C.c_size_t: "size_t", C.c_double: "double", C.c_float: "float"}[t]


def test_ctypes_signatures_match_the_header_prototypes():
    """Every prototype of include/qagnn_b200.h against the ctypes binding: return type, parameter count, and per parameter
    pointer vs integer width (a drifted binding corrupts the call frame silently)."""
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    header = re.sub(r"//[^\n]*", "", header)
    protos = re.findall(r"^((?:const\s+)?[a-z_0-9]+\s*\*?)\s*(qagnn_[a-z_0-9]+)\s*\(([^;{]*?)\)\s*;", header, flags=re.M | re.S)
    assert len(protos) == len(_lib.EXPORTS), (len(protos), len(_lib.EXPORTS))
    for ret, name, params in protos:
        res, args = _lib.EXPORTS[name]
        assert _c_kind(ret + " ") == _ctypes_kind(res), name
        params = re.sub(r"/\*.*?\*/", "", params, flags=re.S).strip()
        plist = [] if params in ("void", "") else [x.strip() for x in params.split(",")]
        assert len(plist) == len(args), f"{name}: header has {len(plist)} parameters, binding {len(args)}"
        for i, (pdecl, a) in enumerate(zip(plist, args)):
            assert _c_kind(pdecl) == _ctypes_kind(a), f"{name}: parameter {i} ({pdecl})"


def test_ctypes_structs_match_the_header_structs():
    """Field names, order and C type of every struct the ABI passes by pointer."""
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    bind = {"qagnn_shape": _lib.Shape, "qagnn_edge_encoder_params": _lib.EdgeEncoderParams, "qagnn_layer_params": _lib.LayerParams,
            "qagnn_mp_params": _lib.MPParams, "qagnn_prep_layout": _lib.PrepLayout}
    structs = re.findall(r"typedef struct (qagnn_[a-z_]+) \{(.*?)\} \1;", header, flags=re.S)
    assert {n for n, _ in structs} == set(bind)
    for name, body in structs:
        fields = []
        for stmt in body.split(";"):
            stmt = stmt.strip()
            if not stmt:
                continue
            ctype, names = re.match(r"((?:const\s+)?[a-z_0-9]+)\s+(.*)", stmt, flags=re.S).groups()
            for nm in names.split(","):
                nm = nm.strip()
                fields.append((nm.lstrip("*").strip(), "ptr" if nm.startswith("*") else ctype))
        got = [(n, _ctypes_kind(t)) for n, t in bind[name]._fields_]
        assert got == fields, name
    assert C.sizeof(_lib.Shape) == 40 and C.sizeof(_lib.PrepLayout) == 22 * C.sizeof(C.c_size_t)


def test_size_queries_and_argument_checks(lib):
    pl = _lib.PrepLayout()
    assert lib.qagnn_graph_prep_layout(64000, 320000, C.byref(pl)) == 0
    assert pl.total_bytes == lib.qagnn_graph_prep_bytes(64000, 320000) > 12 * 4 * 384000
    offs = [getattr(pl, f) for f, _ in _lib.PrepLayout._fields_[1:]]
    assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)
    assert lib.qagnn_graph_prep_layout(0, 10, C.byref(pl)) == -1
    s = _lib.Shape(64000, 320000, 200, 4, 4, 38, 5, 200)
    assert lib.qagnn_fold_bytes(C.byref(s)) > 5 * (3 * 200 * 400 + 2 * 624 * 200) * 4
    assert lib.qagnn_forward_workspace_bytes(C.byref(s)) >= 64000 * 200 * 4 * 8
    bad = _lib.Shape(64000, 320000, 200, 3, 4, 38, 5, 200)  # D % H != 0
    assert lib.qagnn_fold_bytes(C.byref(bad)) == 0
    # null pointers are rejected before any CUDA call
    assert lib.qagnn_graph_prep(None, None, None, C.byref(s), None, 0, 0, None) == -1
    assert lib.qagnn_mp_forward(C.byref(s), None, None, None, None, None, None, None, None, 0, None) == -1


def test_pool_and_head_argument_refusals(lib):
    """The decoder's pooling and head entry points refuse what their kernels do not take before any CUDA call."""
    nul = [None] * 14
    # more than 8 heads: unsupported; D % n_head != 0: invalid
    assert lib.qagnn_attention_pool(2, 10, 36, 9, *nul[:10]) == -5
    assert lib.qagnn_decoder_tail(2, 10, 36, 9, 8, *nul[:12]) == -5
    assert lib.qagnn_attention_pool(2, 10, 10, 4, *nul[:10]) == -1
    assert lib.qagnn_decoder_tail(2, 10, 10, 4, 8, *nul[:12]) == -1
    # the head copies rows as float4: D % 4 != 0 is invalid
    assert lib.qagnn_decoder_head(2, 10, 6, None, 50, *nul[:7]) == -1
    # one node more than 200 KB of shared memory holds (10 nh D + nh n + nh + 16 floats): refused, so the module pools
    # with its einsum path.  The pointers are never dereferenced on the host.
    for nh, D in ((2, 200), (2, 1024), (8, 512)):
        n = (200 * 1024 // 4 - 10 * nh * D - nh - 16) // nh + 1
        p = [C.c_void_p(64)] * 12
        assert lib.qagnn_attention_pool(1, n, D, nh, *p[:10]) == -5
        assert lib.qagnn_decoder_tail(1, n, D, nh, 8, *p) == -5


def test_state_dict_contract_and_cpu_refusal():
    mod = qagnn_b200.QAGNN_Message_Passing(None, 5, 4, 38, 200, 200, 200).eval()
    sd = O.random_state_dict(5, 200)
    assert sorted(mod.state_dict().keys()) == sorted(sd.keys())
    assert sum(p.numel() for p in mod.parameters()) == 2148200  # SURVEY.md §8 a1
    mod.load_state_dict(sd, strict=True)
    assert mod.gnn_layers[3].edge_encoder is mod.edge_encoder  # one shared module, k aliases
    inp = O.synth_graph_batch(2, 10, 20, 200, 38, 0)
    with pytest.raises(RuntimeError, match="CUDA"):
        mod(inp["H"], (inp["edge_index"], inp["edge_type"]), inp["node_type"], inp["node_score"])


def test_decoder_state_dict_keys_match_reference_golden():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "decoder_fc1.pt"), weights_only=False)
    c = fx["case"]
    dec = qagnn_b200.QAGNN(None, c["k"], 4, 38, c["sent_dim"], c["n_concept"], c["D"], c["concept_in_dim"], c["n_head"],
                           c["D"], c["n_fc_layer"], 0.2, 0.2, 0.2)
    assert sorted(dec.state_dict().keys()) == sorted(fx["state_dict"].keys())
    dec.load_state_dict(fx["state_dict"], strict=True)


def test_pack_adj_equals_batch_graph():
    g = torch.Generator().manual_seed(0)
    bs, nc, n = 3, 5, 50
    ei = [[torch.randint(0, n, (2, int(torch.randint(0, 40, (1,), generator=g))), generator=g) for _ in range(nc)] for _ in range(bs)]
    et = [[torch.randint(0, 38, (e.size(1),), generator=g) for e in row] for row in ei]
    packed = pack_adj(ei, et, n, pin=False)
    ref_ei, ref_et = O.batch_graph(sum(ei, []), sum(et, []), n)
    assert torch.equal(packed.edge_index, ref_ei) and torch.equal(packed.edge_type, ref_et)
    assert packed.graph_ptr[-1] == ref_ei.size(1)
    lm = qagnn_b200.LM_QAGNN.batch_graph(None, sum(ei, []), sum(et, []), n)
    assert torch.equal(lm[0], ref_ei) and torch.equal(lm[1], ref_et)


def test_packed_adj_behaves_as_an_edge_pair_and_keeps_graph_ptr():
    """PackedAdj stands in for the (edge_index, edge_type) pair everywhere (unpacking, indexing) and carries what the
    one-launch graph prep needs (graph_ptr on the device of the edges, the largest sub-graph's edge count)."""
    ei = [[torch.tensor([[0, 1], [1, 2]]), torch.zeros(2, 0, dtype=torch.long)], [torch.tensor([[3], [0]]), torch.tensor([[1, 1, 2], [0, 2, 2]])]]
    et = [[torch.tensor([5, 6]), torch.zeros(0, dtype=torch.long)], [torch.tensor([7]), torch.tensor([1, 2, 3])]]
    p = pack_adj(ei, et, 4, pin=False)
    a, b = p
    assert a is p.edge_index and b is p.edge_type and p[0] is a and p[1] is b and len(p) == 2
    assert p.graph_ptr.tolist() == [0, 2, 2, 3, 6]
    assert p.edge_index.tolist() == [[0, 1, 11, 13, 13, 14], [1, 2, 8, 12, 14, 14]]
    q = p.to("cpu")
    assert q.max_edges == 3 and torch.equal(q.graph_ptr_dev, p.graph_ptr) and torch.equal(q.edge_index, p.edge_index)


def test_header_is_plain_c99_and_the_library_links_from_a_c_program(lib, tmp_path):
    """The drop-in boundary is a C ABI: a strict-C99 translation unit includes the header, links the in-tree library
    (no torch, no CUDA runtime on the link line) and calls the entry points that need no GPU."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "caller.c"
    src.write_text(r'''
#include <stdio.h>
#include "qagnn_b200.h"
int main(void) {
  qagnn_shape s = {64000, 320000, 200, 4, 4, 38, 5, 200};
  qagnn_prep_layout pl;
  if (qagnn_graph_prep_layout(s.N, s.E, &pl) != QAGNN_OK) return 2;
  printf("%d %lu %lu %lu\n", (int)qagnn_abi_version(), (unsigned long)qagnn_graph_prep_bytes(s.N, s.E),
         (unsigned long)pl.total_bytes, (unsigned long)qagnn_fold_bytes(&s));
  return qagnn_mp_forward(&s, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0) == QAGNN_ERR_INVALID_ARGUMENT ? 0 : 1;
}
''')
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = tmp_path / "caller"
    cc = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                         str(src), "-o", str(exe), "-L", libdir, "-lqagnn_b200", f"-Wl,-rpath,{libdir}"],
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    ver, prep_bytes, total, fold = (int(x) for x in run.stdout.split())
    s = _lib.Shape(64000, 320000, 200, 4, 4, 38, 5, 200)
    assert ver == 3 and prep_bytes == total == lib.qagnn_graph_prep_bytes(64000, 320000) and fold == lib.qagnn_fold_bytes(C.byref(s))


def test_loader_fails_loudly_without_library_and_compiler(monkeypatch, tmp_path):
    """No CPU fallback: with the library missing and no nvcc, load() raises (it builds only when a compiler is present)."""
    from qagnn_b200 import build

    def no_nvcc():
        raise RuntimeError("nvcc not found")
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "lib" / "libqagnn_b200.so"))
    monkeypatch.setattr(build, "is_current", lambda: False)
    monkeypatch.setattr(build, "_nvcc", no_nvcc)
    with pytest.raises(RuntimeError, match="missing and there is no nvcc.*no CPU fallback"):
        _lib.load()
    mod = qagnn_b200.QAGNN_Message_Passing(None, 1, 4, 38, 16, 16, 16).eval()
    with pytest.raises(RuntimeError):   # CPU tensors never reach a fallback either
        mod(torch.zeros(1, 2, 16), (torch.zeros(2, 0, dtype=torch.long), torch.zeros(0, dtype=torch.long)),
            torch.zeros(1, 2, dtype=torch.long), torch.zeros(1, 2, 1))
