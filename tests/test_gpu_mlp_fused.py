"""The fused node MLP (`mlp_tc_kernel`, one launch, hidden layer in registers) against the two-launch path it replaces.

    out = act2( W2 . ReLU(W1' . aggr + b1') + b2 )

Both paths run the same k16 steps in the same order with the same three split-bf16 passes, and the fused kernel splits the
hidden layer into bf16 hi / lo exactly as mlp.0's plane epilogue does, so every case requires the two results to be bitwise
equal.  QAGNN_MLP_FUSED=0 selects the two launches; the switch is read at every call, so both run in one process.  Launch
counts show which path ran: the fused path saves one launch per layer.
"""
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
T, R = 4, 38


def _launches():
    from qagnn_b200 import _lib
    torch.cuda.synchronize()
    return _lib.load().qagnn_launch_count()


def _both(monkeypatch, fn):
    """fn() under QAGNN_MLP_FUSED=1 and =0 -> (fused result, two-launch result, launches saved by the fused path)"""
    out, cnt = {}, {}
    monkeypatch.setenv("QAGNN_MLP_FUSED", "1")
    fn()  # the first call folds the weights: its launches are not the layer's
    for fused in ("1", "0"):
        monkeypatch.setenv("QAGNN_MLP_FUSED", fused)
        n0 = _launches()
        out[fused] = fn()
        cnt[fused] = _launches() - n0
    return out["1"], out["0"], cnt["0"] - cnt["1"]


def _assert_bitwise(a, b, what):
    a, b = (a if isinstance(a, (list, tuple)) else [a]), (b if isinstance(b, (list, tuple)) else [b])
    for i, (x, y) in enumerate(zip(a, b)):
        if not torch.equal(x, y):
            d = (x.double() - y.double()).abs()
            raise AssertionError(f"{what}[{i}]: fused and two-launch results differ in {int((d > 0).sum())} elements, "
                                 f"max |diff| {d.max().item():.3e}")


# ---- full forward (qagnn_mp_forward): output and every layer's x --------------------------------------------------------
def _mp_run(mod, d):
    out, layers = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    return [out.clone(), layers.clone()]


@pytest.mark.parametrize("ctas", ["1", "0"])
def test_bench_workload_bitwise(ctas, monkeypatch):
    """The cfg2 step's message passing (320 graphs x 200 nodes, D = 200, k = 5): the fast projection path."""
    import bench
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    C = bench.CFG
    inp = bench.synth_step_inputs(0)
    sd = O.random_state_dict(C["k"], C["D"], C["T"], C["R"], "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, C["k"], C["T"], C["R"], C["D"], C["D"], C["D"]).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = {k: inp[k].to(DEV) for k in ("H", "edge_index", "edge_type", "node_type", "node_score")}
    fused, two, saved = _both(monkeypatch, lambda: _mp_run(mod, d))
    assert saved == C["k"], f"the fused path should save one launch per layer, saved {saved}"
    _assert_bitwise(fused, two, "cfg2 [out, x_layers]")


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("name", Hh.golden_names("mp"))
def test_goldens_bitwise_and_golden(name, ctas, monkeypatch):
    """Every message-passing golden; widths the fused kernel takes (D % 8 == 0, D <= 208) must run it."""
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    fx = Hh.load_golden(name)
    c = fx["case"]
    inp, sd = Hh.regen_mp_inputs(fx)
    d = {k: v.to(DEV) for k, v in inp.items()}
    mod = qagnn_b200.QAGNN_Message_Passing(None, c["k"], fx["n_ntype"], fx["n_etype"], c["D"], c["D"], c["D"]).eval()
    mod.load_state_dict(sd, strict=True)
    mod = mod.to(DEV)
    fused, two, saved = _both(monkeypatch, lambda: _mp_run(mod, d))
    takes = c["D"] % 8 == 0 and c["D"] <= 208
    assert saved == (c["k"] if takes else 0), f"D={c['D']}: launches saved {saved}"
    _assert_bitwise(fused, two, f"{name} [out, x_layers]")
    for l, ref_l in fx["layers"].items():
        Hh.assert_close(fused[1][l], ref_l["x"], f"x[{l}]")
    Hh.assert_close(fused[0], fx["out"], "out")


# ---- bare layer (qagnn_gatconve_forward, final_act NONE) ---------------------------------------------------------------
def _enc(D):
    return torch.nn.Sequential(torch.nn.Linear(R + 1 + 2 * T, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))


def _layer_case(N, D, H, seed):
    n = N if N <= 300 else 200
    assert N % n == 0
    b = O.synth_graph_batch(N // n, n, 3 * n, D, R, seed=seed)
    sd = O.random_state_dict(1, D, T, R, "peaky", seed=seed)
    x, nt = b["H"].reshape(-1, D), b["node_type"].reshape(-1)
    extra = torch.randn(x.shape, generator=torch.Generator().manual_seed(seed)) * 0.5
    return sd, x, extra, nt, b["edge_index"], b["edge_type"]


def _layer(sd, D, H):
    layer = qagnn_b200.GATConvE(None, D, T, R, _enc(D), head_count=H)
    layer.load_state_dict({k[len("gnn_layers.0."):]: v for k, v in sd.items() if k.startswith("gnn_layers.0.")}, strict=True)
    return layer.to(DEV).eval()


def _layer_fwd(layer, x, extra, nt, ei, et):
    args = [t.to(DEV) for t in (x, ei, et, nt, extra)]
    return layer(args[0], args[1], args[2], args[3], args[4]).clone()


LAYER_CASES = [  # (N, D, H): ragged rows around the 128-row tile and the 256-row CTA pair; narrow and mid widths
    (1, 200, 4), (127, 200, 4), (128, 200, 4), (129, 200, 4), (1000, 200, 4),
    (257, 8, 2), (257, 96, 4), (600, 96, 4), (129, 8, 2),
]


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("N,D,H", LAYER_CASES)
def test_bare_layer_bitwise_and_oracle(N, D, H, ctas, monkeypatch):
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    seed = 13 * N + D
    sd, x, extra, nt, ei, et = _layer_case(N, D, H, seed)
    layer = _layer(sd, D, H)
    fused, two, saved = _both(monkeypatch, lambda: _layer_fwd(layer, x, extra, nt, ei, et))
    assert saved == 1, f"the fused path should save one launch, saved {saved}"
    _assert_bitwise(fused, two, f"N={N} D={D}")
    ref, _, _, _ = O.gatconve_forward(sd, "gnn_layers.0", x, ei, et, nt, extra, T, R, head_count=H, dtype=F64)
    Hh.assert_close(fused, ref, f"N={N} D={D} fused vs oracle")


def test_one_perturbed_w2_column_is_detected(monkeypatch):
    """The checks above see a single W2 column: the fused kernel on weights whose mlp.3 column c is perturbed differs from
    the two-launch path on the original weights, and fails the oracle bar."""
    N, D, H, c = 257, 200, 4, 137
    sd, x, extra, nt, ei, et = _layer_case(N, D, H, 5)
    sd_bad = dict(sd)
    w = sd["gnn_layers.0.mlp.3.weight"].clone()
    w[:, c] += 0.05
    sd_bad["gnn_layers.0.mlp.3.weight"] = w
    monkeypatch.setenv("QAGNN_MLP_FUSED", "1")
    bad = _layer_fwd(_layer(sd_bad, D, H), x, extra, nt, ei, et)
    monkeypatch.setenv("QAGNN_MLP_FUSED", "0")
    good = _layer_fwd(_layer(sd, D, H), x, extra, nt, ei, et)
    assert not torch.equal(bad, good)
    ref, _, _, _ = O.gatconve_forward(sd, "gnn_layers.0", x, ei, et, nt, extra, T, R, head_count=H, dtype=F64)
    Hh.assert_close(good, ref, "two-launch vs oracle")
    with pytest.raises(AssertionError):
        Hh.assert_close(bad, ref, "perturbed fused vs oracle")
