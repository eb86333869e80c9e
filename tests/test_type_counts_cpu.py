"""The rows of tests/test_gpu_type_counts.py against the limits they are meant to straddle, without a GPU.

Each formula below restates a plan decision of the kernels that depends on the combo count C = R*T*T + T; every limit must have
a row exactly at it (the largest accepted value) and a row just past it, and every row's hand-written path must be the one the
formulas give.  The shared-memory limits take the opt-in shared memory per block as a parameter.  Also: the int16 edge types of
the flat adjacency refuse values they cannot hold instead of wrapping them.
"""
import numpy as np
import pytest
import torch

from qagnn_b200 import data as Dt
from tests import test_gpu_type_counts as TC

OPTINS = {"h100": 227 * 1024, "a100": 163 * 1024}


def offset_ok(H, D, T, R):
    """mp_headtile.cu make_plan: the last table row's offset in 2-byte units fits the 16-bit word."""
    return (TC.combos(T, R) - 1) * (TC.head_dim_padded(H, D) // 4) * 8 <= 65535


def tile_smem_ok(H, D, T, R, n, optin):
    """mp_headtile.cu make_smem_map: edge table, two node tiles, barriers and counters."""
    DP = TC.head_dim_padded(H, D)
    return TC.combos(T, R) * DP * 4 + 2 * n * DP * 4 + 64 <= optin


def slice_width(H, D):
    """mp_slice.cu make_slice_plan: the slice width of head width d, or None when the sliced kernels do not take it."""
    d = D // H
    SL = 64 if d >= 64 else d
    return SL if 32 % H == 0 and SL in (16, 32, 64) and d % SL == 0 and d // SL <= 2 else None


def slice_smem_ok(H, D, T, R, optin):
    return TC.combos(T, R) * slice_width(H, D) * 4 <= optin


def predicted_path(r, optin):
    if TC.head_dim_padded(r.H, r.D) <= 64 and offset_ok(r.H, r.D, r.T, r.R) and tile_smem_ok(r.H, r.D, r.T, r.R, r.n, optin):
        return "tiled"
    if slice_width(r.H, r.D) and slice_smem_ok(r.H, r.D, r.T, r.R, optin):
        return "slice"
    return "basic"


def _rows(optin):
    return TC.OFFSET_ROWS + TC.OTHER_ROWS + TC.smem_rows(optin)


@pytest.mark.parametrize("optin", OPTINS.values(), ids=OPTINS.keys())
def test_every_row_takes_the_path_the_formulas_give(optin):
    for r in _rows(optin):
        assert predicted_path(r, optin) == r.path, f"{r.id}: the formulas give {predicted_path(r, optin)}"


def _accepts(r, optin):
    """Whether row r's own limit accepts it, and whether it would accept one more (R + 1, or n + 1 for the node tile)."""
    if r.limit == "offset":
        return offset_ok(r.H, r.D, r.T, r.R), offset_ok(r.H, r.D, r.T, r.R + 1)
    if r.limit == "tile_smem":
        return tile_smem_ok(r.H, r.D, r.T, r.R, r.n, optin), tile_smem_ok(r.H, r.D, r.T, r.R, r.n + 1, optin)
    return slice_smem_ok(r.H, r.D, r.T, r.R, optin), slice_smem_ok(r.H, r.D, r.T, r.R + 1, optin)


@pytest.mark.parametrize("optin", OPTINS.values(), ids=OPTINS.keys())
def test_every_limit_has_a_row_at_it_and_one_just_past_it(optin):
    rows = [r for r in _rows(optin) if r.limit is not None]
    assert {r.limit for r in rows} == {"offset", "tile_smem", "slice_smem"}
    ats = [r for r in rows if r.side == "at"]
    for r in ats:
        ok, next_ok = _accepts(r, optin)
        assert ok and not next_ok, f"{r.id}: not the largest value {r.limit} accepts"
        step = (0, 1) if r.limit == "tile_smem" else (1, 0)
        past = [p for p in rows if p.side == "past" and p.limit == r.limit and (p.H, p.D, p.T) == (r.H, r.D, r.T)
                and (p.R, p.n) == (r.R + step[0], r.n + step[1])]
        assert len(past) == 1, f"{r.id}: no row just past it"
        assert not _accepts(past[0], optin)[0] and past[0].path != r.path
    assert len(ats) * 2 == len(rows), "a row past a limit without its row at the limit"
    # the offset word is hit exactly (C - 1 = 65535 / (DP/4 * 8)) at T = 1 for every head width of the table
    for DP in (52, 32, 16, 4):
        assert any(r.limit == "offset" and r.T == 1 and r.DP == DP for r in ats), DP
    # the node-tile rows pass the offset word, so their path change is the shared memory's; the slice rows fail it, so the
    # tiled kernel is out and the change from slice to basic is the table slice's
    for r in rows:
        if r.limit == "tile_smem":
            assert offset_ok(r.H, r.D, r.T, r.R), r.id
        if r.limit == "slice_smem":
            assert not offset_ok(r.H, r.D, r.T, r.R), r.id


def test_the_fast_projection_row_has_64_node_types():
    r, = TC.OTHER_ROWS
    assert r.T == 64 and r.fast and r.D // 2 % 4 == 0 and r.D // 2 >= 8 and r.path == "tiled"


def test_graph_prep_and_combo_sort_cases_straddle_their_limits():
    Cs = [TC.combos(T, R) for T, R in TC.PREP_CASES]
    assert max(Cs) == TC.PREP_COMBO_MAX and TC.combos(*TC.PREP_REFUSED) == TC.PREP_COMBO_MAX + 1
    assert {1, 7, 16} <= {T for T, _ in TC.PREP_CASES}
    (ok, a), (no, b) = TC.COMBO_SORT_CASES
    assert a and not b and TC.combos(*ok) == TC.COMBO_SORT_MAX and TC.combos(*no) == TC.COMBO_SORT_MAX + 1
    assert all(TC.combos(T, R) <= TC.COMBO_SORT_MAX for T, R in TC.TRAIN_CASES)


def test_batch_draws_every_type_and_forces_the_extreme_combos():
    from oracle import qagnn_oracle as O
    for T, R in [(1, 5), (7, 3), (16, 23)]:
        b = TC.batch(T, R, 8, seed=1)
        assert set(b["node_type"].unique().tolist()) == set(range(T))
        assert int(b["edge_type"].max()) == R - 1 and int(b["edge_type"].min()) == 0
        combo = O.graph_prep_oracle(b["edge_index"], b["edge_type"], b["node_type"], T, R)["combo"]
        assert (combo == R * T * T - 1).any() and combo.max() == TC.combos(T, R) - 1


def test_synth_graph_batch_types():
    from oracle import qagnn_oracle as O
    a = O.synth_graph_batch(3, 20, 40, 8, 38, seed=2)
    b = O.synth_graph_batch(3, 20, 40, 8, 38, seed=2, n_ntype=4)
    assert all(torch.equal(a[k], b[k]) for k in a)
    c = O.synth_graph_batch(3, 20, 40, 8, 5, seed=2, n_ntype=6)
    assert (c["node_type"][:, 0] == 5).all() and set(c["node_type"][:, 1:].unique().tolist()) == set(range(5))
    assert (O.synth_graph_batch(2, 9, 10, 8, 5, seed=2, n_ntype=1)["node_type"] == 0).all()
    with pytest.raises(ValueError):
        O.synth_graph_batch(2, 20, 40, 8, 38, seed=2, realistic=True, n_ntype=3)


# ---- int16 edge types of the flat adjacency ---------------------------------------------------------------------------
def _nested(types):
    return [[torch.tensor([[0, 1], [1, 0]])]], [[torch.tensor(types)]]


def test_flat_cache_refuses_edge_types_that_do_not_fit_int16():
    ei, et = _nested([3, 32767])
    assert Dt.FlatAdjCache.from_nested(ei, et, 4).etype.tolist() == [3, 32767]
    for bad in (65541, 65536, 32768, -32769):  # numpy's int16 cast gives 5, 0, -32768 and 32767
        ei, et = _nested([3, bad])
        with pytest.raises(ValueError, match=f"edge type {bad} does not fit"):
            Dt.FlatAdjCache.from_nested(ei, et, 4)


def test_device_split_refuses_edge_types_that_do_not_fit_int16():
    def split(etype, n_etype):
        flat = Dt.FlatAdjCache(np.array([0, 1], np.int32), np.array([1, 0], np.int32), etype, np.array([0, 2]), 1, 4)
        z = torch.zeros(1, 1, 4, dtype=torch.long)
        return Dt.DeviceSplit(flat, z, z, torch.zeros(1, 1, 4, 1), torch.tensor([[4]]), "cpu", 4, n_etype)
    assert split(np.array([0, 32767], np.int32), 32768).etype.tolist() == [0, 32767]
    with pytest.raises(ValueError, match="edge type 65541 does not fit"):
        split(np.array([0, 65541], np.int32), 32768)
    with pytest.raises(ValueError, match="n_etype = 65542"):
        split(np.array([0, 5], np.int32), 65542)
