"""The fast-form projection on `proj_resident_kernel` (W slice resident in shared memory, A-only ring, ping-pong consumer
warpgroups) against `gemm_tc_kernel`.

Both kernels run every output element through the same k16 steps, in the same order, with the same three split-bf16 passes,
the same exact K tail and the same type-bias addition, so every case requires bitwise equal results.  QAGNN_PROJ_RESIDENT=0
selects gemm_tc_kernel; the switch is read at every call, so both run in one process.  The launch lines QAGNN_DEBUG=1 prints
show which one ran: shapes whose head is wider than 52 padded columns or whose K = D + D/2 exceeds 320 must fall back to
gemm_tc_kernel (the projection is the step's only gemm_tc_kernel launch without an activation).
"""
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R = 4, 38
RESIDENT = "proj_resident_kernel"


def _launches(fn, capfd):
    """(fn()'s result, (proj_resident_kernel launches, gemm_tc launches without an activation) during it), from the launch
    lines the library prints to stderr under QAGNN_DEBUG=1"""
    torch.cuda.synchronize()
    capfd.readouterr()
    out = fn()
    torch.cuda.synchronize()
    lines = capfd.readouterr().err.splitlines()
    return out, (sum(ln.startswith("proj_resident: M=") for ln in lines),
                 sum(ln.startswith("gemm_tc: M=") and " act=0 " in ln for ln in lines))


def _both(monkeypatch, capfd, fn):
    """fn() with the resident kernel allowed and forced off -> (result, launch counts) for each"""
    monkeypatch.setenv("QAGNN_DEBUG", "1")
    monkeypatch.setenv("QAGNN_PROJ_RESIDENT", "1")
    fn()  # the first call folds the weights
    res = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("QAGNN_PROJ_RESIDENT", flag)
        res[flag] = _launches(fn, capfd)
    return res["1"], res["0"]


def _assert_bitwise(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        if not torch.equal(x, y):
            d = (x.double() - y.double()).abs()
            raise AssertionError(f"{what}[{i}]: resident and gemm_tc results differ in {int((d > 0).sum())} elements, "
                                 f"max |diff| {d.max().item():.3e}")


def _module(k, D, H=4, seed=5):
    sd = O.random_state_dict(k, D, T, R, "prod", seed=seed)
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, T, R, D, D, D).eval()
    if H != 4:
        mod.gnn_layers = torch.nn.ModuleList([qagnn_b200.GATConvE(None, D, T, R, mod.edge_encoder, head_count=H) for _ in range(k)])
    mod.load_state_dict(sd)
    return mod.to(DEV)


def _run(mod, d):
    with torch.no_grad():
        out, layers = mod(d["H"], (d["edge_index"], d["edge_type"]), d["node_type"], d["node_score"], return_layers=True)
    return [out.clone(), layers.clone()]


def _batch(B, n, D, seed):
    b = O.synth_graph_batch(B, n, 5 * n, D, R, seed=seed)
    return {k: b[k].to(DEV) for k in ("H", "edge_index", "edge_type", "node_type", "node_score")}


def _accepted(D, H):
    DP = (D // H + 3) // 4 * 4
    return DP <= 52 and D + D // 2 <= 320


def _check(monkeypatch, capfd, fn, k, accepted, what):
    (new, (res_new, gemm_new)), (old, (res_old, gemm_old)) = _both(monkeypatch, capfd, fn)
    _assert_bitwise(new, old, what)
    assert res_old == 0, f"{what}: QAGNN_PROJ_RESIDENT=0 still ran {RESIDENT}"
    assert gemm_old >= k, f"{what}: {gemm_old} projections on gemm_tc_kernel with the switch off, expected {k}"
    if accepted:
        assert (res_new, gemm_old - gemm_new) == (k, k), f"{what}: {res_new} {RESIDENT} launches, {gemm_old - gemm_new} fewer on gemm_tc"
    else:
        assert (res_new, gemm_new) == (0, gemm_old), f"{what}: a refused shape must fall back to gemm_tc_kernel"


@pytest.mark.parametrize("ctas", ["1", "0"])
def test_bench_workload_bitwise(ctas, monkeypatch, capfd):
    """The cfg2 step's message passing (320 graphs x 200 nodes, D = 200, H = 4, k = 5)."""
    import bench
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    C = bench.CFG
    inp = bench.synth_step_inputs(0)
    sd = O.random_state_dict(C["k"], C["D"], C["T"], C["R"], "prod", seed=0)
    mod = qagnn_b200.QAGNN_Message_Passing(None, C["k"], C["T"], C["R"], C["D"], C["D"], C["D"]).eval()
    mod.load_state_dict(sd)
    mod = mod.to(DEV)
    d = {k: inp[k].to(DEV) for k in ("H", "edge_index", "edge_type", "node_type", "node_score")}
    _check(monkeypatch, capfd, lambda: _run(mod, d), C["k"], True, "cfg2")


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("B,n", [(1, 37), (1, 64), (3, 50), (2, 96), (5, 200), (7, 131)])
def test_rows_around_the_unit(B, n, ctas, monkeypatch, capfd):
    """M below one 64-row unit, at it, and not a multiple of 64 or 128: TMA zero-fills the rows past M and clips the stores."""
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    mod = _module(2, 200, seed=B * n)
    d = _batch(B, n, 200, seed=B * n)
    _check(monkeypatch, capfd, lambda: _run(mod, d), 2, True, f"M={B * n}")


@pytest.mark.parametrize("ctas", ["1", "0"])
def test_type_classes_at_and_past_both_ends(ctas, monkeypatch, capfd):
    """The bias row of a node is its type clamped to [0, T-1], as in gemm_tc_kernel."""
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    mod = _module(2, 200, seed=3)
    mod.check_indices = False  # out-of-range types are clamped everywhere (graph prep flags them)
    d = _batch(2, 150, 200, seed=3)
    nt = torch.tensor([-7, -1, 0, T - 1, T, T + 9], device=DEV)
    d["node_type"] = nt[torch.arange(d["node_type"].numel(), device=DEV) % nt.numel()].reshape(d["node_type"].shape)
    _check(monkeypatch, capfd, lambda: _run(mod, d), 2, True, "type classes")


@pytest.mark.parametrize("ctas", ["1", "0"])
def test_ragged_node_capacity(ctas, monkeypatch, capfd):
    """A ragged batch: packed rows at a node capacity past the valid rows (zero-filled tail rows)."""
    from tests.test_gpu_ragged import _dev_adj, _loader_batch, ragged_inputs
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    inp, n = _loader_batch(n_questions=3)
    adj, Hp, ntp, nsp, _ = ragged_inputs(inp["H"], inp["edge_index"], inp["edge_type"], inp["node_type"], inp["node_score"],
                                         inp["adj_lengths"], n, node_capacity=int(inp["adj_lengths"].sum()) + 61)
    mod = _module(3, 200, seed=11)
    a, H, nt, ns = _dev_adj(adj), Hp.to(DEV), ntp.to(DEV), nsp.to(DEV)

    def run():
        with torch.no_grad():
            return [mod(H, a, nt, ns).clone()]
    _check(monkeypatch, capfd, run, 3, True, "ragged")


HEAD_SHAPES = [  # (D, H) of the tiled path's fast form: every head count, every K tail, slice widths 8 .. 104, odd slice counts
    (200, 4), (208, 4), (200, 8), (208, 16), (96, 2), (96, 4), (96, 8), (128, 4), (16, 1), (48, 1),
    # refused: a padded head of 64 columns, wider than the 52 a staging buffer holds
    (64, 1), (128, 2),
]


@pytest.mark.parametrize("ctas", ["1", "0"])
@pytest.mark.parametrize("D,H", HEAD_SHAPES)
def test_every_head_shape(D, H, ctas, monkeypatch, capfd):
    monkeypatch.setenv("QAGNN_TC_2CTA", ctas)
    mod = _module(2, D, H, seed=D + H)
    d = _batch(3, 70, D, seed=D + H)
    _check(monkeypatch, capfd, lambda: _run(mod, d), 2, _accepted(D, H), f"D={D} H={H}")
