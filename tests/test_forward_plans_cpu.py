"""The case table of tests/test_gpu_forward_plans.py keeps covering every eval forward plan: without a GPU, check that its
hand-written rows hold every value of every ForwardPlan field in both precisions and both batch layouts, every head count,
every tiled-kernel instantiation, k = 0, 1, 2 on both GEMM kinds, and each bit-for-bit pair."""
import itertools

from tests.test_gpu_forward_plans import CASES, PLAN_FIELDS, SWITCHES

GROUPS = {"fp32": ("fp32",), "bf16": ("bf16", "bf16in")}


def _group(c):
    return "fp32" if c.prec == "fp32" else "bf16"


def _laygroup(c):
    return "ragged" if c.layout == "ragged" else "padded"


def test_rows_are_well_formed():
    ids = [c.id for c in CASES]
    assert len(ids) == len(set(ids)), "two rows with one id"
    for c in CASES:
        p = c.plan
        assert set(p) == set(PLAN_FIELDS) and set(c.env) <= set(SWITCHES), c.id
        assert c.D % c.H == 0 and c.D % 2 == 0, c.id
        # what plan_forward can return at all (abi.cu, ForwardPlan's field comments)
        assert p["passes"] == (3 if c.prec == "fp32" else 1), c.id
        assert not (p["tiled"] and p["slice"]), c.id
        assert p["zero_pads"] == (p["tiled"] and not p["tc"]), c.id
        assert not p["fast"] or (p["tc"] and p["tiled"] and c.layers > 0 and c.D // 2 >= 8), c.id
        assert not p["mlp_fused"] or p["tc"], c.id
        assert not c.resident or (p["fast"] and p["passes"] == 3 and c.entry == "mp"), c.id
        assert (c.ht is not None) == (p["tiled"] and c.layers > 0), c.id
        if c.ht is not None:
            assert c.ht[0] == (1 if c.DP <= 32 else 2), f"{c.id}: CPL"
        if p["zero_pads"]:  # the pad-zeroing kernel launches only when a head has pad columns: keep it observable
            assert c.DP != c.d, c.id
        if c.entry == "mp" and c.k == 0:
            assert c.H == 4, f"{c.id}: without layers the plan is made at GATConvE's default head count"


def test_every_plan_field_value_in_both_precisions_and_layouts():
    for prec, lay in itertools.product(GROUPS, ("padded", "ragged")):
        rows = [c for c in CASES if _group(c) == prec and _laygroup(c) == lay]
        for field in PLAN_FIELDS:
            if field == "passes":
                continue
            pool = [c for c in rows if c.entry == "mp" and c.layers > 0] if field == "fast" else rows
            seen = {c.plan[field] for c in pool}
            assert seen == {True, False}, f"{prec}/{lay}: {field} takes only {seen}"
        assert {c.plan["passes"] for c in rows} == {3 if prec == "fp32" else 1}


def test_every_head_count_in_both_precisions():
    for prec in GROUPS:
        assert {c.H for c in CASES if _group(c) == prec and c.layers > 0} == {1, 2, 4, 8, 16}, prec
    single = [c for c in CASES if _group(c) == "bf16" and c.plan["tc"] and c.layers > 0]
    assert any(c.d % 2 == 1 for c in single), "no odd head width on the single-pass path"
    assert any(c.H * c.DP > 256 and c.plan["tiled"] for c in single), "no H * DP > 256 on the single-pass path"
    assert any(c.entry == "mp" and c.plan["fast"] and c.H != 4 for c in single), "no single-pass fast form at H != 4"
    assert {c.H for c in single if c.plan["slice"] or not c.plan["tiled"]} - {4}, "slice / basic under bf16 only at H = 4"


def test_every_tiled_kernel_instantiation():
    seen = {(c.ht[0], c.ht[1], c.layout == "ragged") for c in CASES if c.ht is not None}
    assert seen == set(itertools.product((1, 2), ("narrow", "wide"), (False, True))), seen


def test_k_0_1_2_on_both_gemm_kinds_and_layouts():
    for tc, lay, k in itertools.product((True, False), ("padded", "ragged"), (0, 1, 2)):
        assert any(c.entry == "mp" and c.plan["tc"] == tc and _laygroup(c) == lay and c.k == k for c in CASES), (tc, lay, k)
    for prec in GROUPS:
        assert any(c.entry == "mp" and c.k == 0 and _group(c) == prec for c in CASES), prec
    assert any(c.entry == "mp" and c.k == 0 and c.prec == "bf16in" for c in CASES)


def test_every_bit_for_bit_pair():
    for prec in GROUPS:
        rows = [c for c in CASES if _group(c) == prec]
        assert any(c.layout == "ragged" for c in rows) and any(c.layout == "edgecap" for c in rows), prec
        twins = {(k, c.env.get(k), v) for c in rows if c.twin for k, v in c.twin.items()}
        assert ("QAGNN_TC_2CTA", "0", "1") in twins, prec
        assert ("QAGNN_MLP_FUSED", "0", "1") in twins, prec
    twins = {(k, c.env.get(k), v) for c in CASES if c.twin for k, v in c.twin.items()}
    for w in ("7", "24", "31"):
        assert ("QAGNN_MP_WARPS", w, None) in twins, w
    assert any(c.twin == {"QAGNN_PROJ_RESIDENT": "0"} and c.resident and c.prec == "fp32" for c in CASES)
    # the ragged module runs that never ran before: the switches below, and widths too wide for tiles
    ragged_mp = [c for c in CASES if c.layout == "ragged"]
    for env in ({"QAGNN_MP_FASTPROJ": "0"}, {"QAGNN_MLP_FUSED": "0"}, {"QAGNN_GEMM": "ffma"}):
        assert any(all(c.env.get(k) == v for k, v in env.items()) and c.entry == "mp" for c in ragged_mp), env
    assert any(c.env.get("QAGNN_GEMM") == "ffma" and c.D % 8 == 0 for c in ragged_mp)
    assert any(c.DP > 64 and not c.env for c in ragged_mp)
