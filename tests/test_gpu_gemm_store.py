"""The split-bf16 GEMMs' TMA-store epilogue against the direct-store epilogue it replaces, bit for bit.

By default the consumers of `gemm_tc_kernel` and `mlp_tc_kernel` write each column chunk of their tile into shared memory
and one thread stores it with TMA, clipped to M rows and N columns; QAGNN_TC_STORE=direct stores straight from the
accumulator registers.  Only the place and the instruction of the store differ, so every case requires equal bits.  Both
switches are read at every call, so both epilogues run in one process.  Every case runs with CTA pairs and single CTAs.
"""
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import ops
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _both(monkeypatch, fn):
    """fn() with the TMA-store epilogue and with QAGNN_TC_STORE=direct -> (tma, direct)"""
    out = {}
    for mode in ("tma", "direct"):
        monkeypatch.setenv("QAGNN_TC_STORE", mode)
        out[mode] = fn()
    torch.cuda.synchronize()
    return out["tma"], out["direct"]


def _assert_bitwise(a, b, what):
    a, b = (a if isinstance(a, (list, tuple)) else [a]), (b if isinstance(b, (list, tuple)) else [b])
    for i, (x, y) in enumerate(zip(a, b)):
        if not torch.equal(x, y):
            d = (x.double() - y.double()).abs().nan_to_num(float("inf"))
            raise AssertionError(f"{what}[{i}]: TMA-store and direct-store results differ in {int((d > 0).sum())} "
                                 f"elements, max |diff| {d.max().item():.3e}")


def _linear(monkeypatch, ctas, M, N, K1, K2, act, seed=0):
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    g = torch.Generator(device="cpu").manual_seed(seed)
    a1 = torch.randn(M, K1, generator=g).to(DEV)
    a2 = torch.randn(M, K2, generator=g).to(DEV) if K2 else None
    w = (torch.randn(N, K1 + K2, generator=g) / (K1 + K2) ** 0.5).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    tma, direct = _both(monkeypatch, lambda: ops.linear_bf16x3(a1, w, b, a2, act))
    _assert_bitwise(tma, direct, f"linear M={M} N={N} K={K1}+{K2} {act}")


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("M", [1, 127, 129, 64000 + 37])
def test_ragged_rows(M, ctas, monkeypatch):
    _linear(monkeypatch, ctas, M, 200, 200, 0, "none")


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("N", [8, 60, 64, 100, 120, 200, 208, 248, 256, 624])  # tile widths 64 / 128 / 208 / 256
def test_tile_widths(N, ctas, monkeypatch):
    _linear(monkeypatch, ctas, 1000, N, 104, 0, ("none", "relu", "gelu")[N % 3])


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("act", ["none", "relu", "gelu"])
def test_two_segments_every_activation(act, ctas, monkeypatch):
    _linear(monkeypatch, ctas, 1029, 200, 200, 200, act, seed=1)


# ---- head-major projection, bf16 plane outputs inside a wider row and the fused MLP: through the message-passing forward
def _mp_run(mod, d):
    out, layers = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    return [out.clone(), layers.clone()]


@pytest.mark.parametrize("fused", ["1", "0"])
@pytest.mark.parametrize("ctas", ["1", "0"])
def test_bench_workload(ctas, fused, monkeypatch):
    """The cfg2 step's message passing (320 graphs x 200 nodes, D = 200, H = 4, k = 5): head-major projection at DP = 52,
    score_emb planes in columns 200..299 of the [N, 304] x planes, the fused node MLP (or mlp.0 / mlp.3), Vh/Vx."""
    import bench
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    monkeypatch.setenv("QAGNN_MLP_FUSED", fused)
    C = bench.CFG
    inp = bench.synth_step_inputs(0)
    sd = O.random_state_dict(C["k"], C["D"], C["T"], C["R"], "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, C["k"], C["T"], C["R"], C["D"], C["D"], C["D"]).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = {k: inp[k].to(DEV) for k in ("H", "edge_index", "edge_type", "node_type", "node_score")}
    tma, direct = _both(monkeypatch, lambda: _mp_run(mod, d))
    _assert_bitwise(tma, direct, "cfg2 [out, x_layers]")


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_goldens(name, ctas, monkeypatch):
    """Every message-passing golden: the head counts and head widths (H, DP) the tiled path takes, and the odd shapes."""
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    d = {k: v.to(DEV) for k, v in inp.items()}
    mod = qagnn_b200.QAGNN_Message_Passing(None, c["k"], fx["n_ntype"], fx["n_etype"], c["D"], c["D"], c["D"]).eval()
    mod.load_state_dict(sd, strict=True)
    mod = mod.to(DEV)
    tma, direct = _both(monkeypatch, lambda: _mp_run(mod, d))
    _assert_bitwise(tma, direct, f"{name} [out, x_layers]")
