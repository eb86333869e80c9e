"""Every eval forward plan against a high-precision reference, with the plan itself read from the kernels that ran.

`plan_forward` (qagnn_b200/csrc/abi.cu) turns a call's shape, batch layout, precision and switches into one ForwardPlan:
passes, tc, tiled, slice, zero_pads, fast and mlp_fused.  Each row of CASES below names an entry point (one GATConvE layer
or QAGNN_Message_Passing), (H, D, k), a batch layout, a precision and the switches, and writes the plan it must get BY HAND,
as tests/test_gpu_heads.py EVAL_SHAPES does.  For every row the test
  * profiles the call (torch.profiler, CUDA kernel records) and requires the kernel set the expected plan implies, the tiled
    kernel's <CPL, WMAX, RAGGED> template arguments included;
  * compares the result with a reference in fp64: the oracle for fp32 plans (the suite's 1e-4 bar), the contract emulation
    of tests/test_gpu_eval_bf16.py for bf16 plans on the wgmma GEMMs (its bf16 bars), and the oracle on bf16-rounded inputs
    for bf16 plans on the FFMA GEMM (the fp32 bar plus one bf16 unit of the output);
  * requires equal bits where the arithmetic is the same: a ragged batch's valid rows against the padded batch, an edge
    capacity against the exact batch, and each row's `twin` switch setting against its own.
tests/test_forward_plans_cpu.py checks, without a GPU, that the rows keep covering every plan field value, head count,
tiled-kernel instantiation and k the kernels branch on.  The last tests show that each bar rejects a seeded fault.
"""
import re

import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from tests import helpers as Hh

DEV = "cuda:0"
F64 = torch.float64
BF = torch.bfloat16
T, R = 4, 38
U = 2.0 ** -8  # one bf16 unit
SWITCHES = ("QAGNN_MP_PATH", "QAGNN_GEMM", "QAGNN_MP_FASTPROJ", "QAGNN_MLP_FUSED", "QAGNN_PROJ_RESIDENT", "QAGNN_TC_2CTA",
            "QAGNN_MP_WARPS")
PLAN_FIELDS = ("passes", "tc", "tiled", "slice", "zero_pads", "fast", "mlp_fused")
LAYOUTS = ("general", "tiled", "packed", "edgecap", "ragged")  # padded with the general prep / with the per-graph prep,
                                                                 # PackedAdj exact / at an edge capacity, ragged
PRECISIONS = ("fp32", "bf16", "bf16in")  # fp32; bf16 autocast with fp32 input; bf16 autocast with bf16 input
WMAX = {"narrow": 24, "wide": 31}       # kWarpsNarrow / kWarpsWide of mp_headtile.cu


class Case:
    """One row.  `plan`: the ForwardPlan flags that are true ('res' = the projection on proj_resident_kernel, a launcher
    choice below the plan); passes follows the precision.  `ht`: (CPL, 'narrow' | 'wide') of the tiled kernel.  `twin`:
    switches of a second run on the same layout whose outputs must equal this row's bit for bit (None = unset)."""

    def __init__(self, entry, H, D, k, layout, prec, plan, env=None, ht=None, twin=None):
        assert entry in ("layer", "mp") and layout in LAYOUTS and prec in PRECISIONS
        self.entry, self.H, self.D, self.k, self.layout, self.prec = entry, H, D, k, layout, prec
        self.env, self.ht, self.twin = dict(env or {}), ht, twin
        flags = plan.split()
        assert set(flags) <= {"tc", "tiled", "slice", "zp", "fast", "fused", "res"}, plan
        self.plan = {"passes": 3 if prec == "fp32" else 1, "tc": "tc" in flags, "tiled": "tiled" in flags,
                     "slice": "slice" in flags, "zero_pads": "zp" in flags, "fast": "fast" in flags,
                     "mlp_fused": "fused" in flags}
        self.resident = "res" in flags
        self.layers = k if entry == "mp" else 1
        sw = "-".join(f"{n[len('QAGNN_'):].lower()}{v}" for n, v in sorted(self.env.items()))
        self.id = f"{entry}-h{H}-d{D}" + (f"-k{k}" if entry == "mp" else "") + f"-{layout}-{prec}" + (f"-{sw}" if sw else "")

    @property
    def d(self):
        return self.D // self.H

    @property
    def DP(self):
        return (self.d + 3) // 4 * 4


L, M = "layer", "mp"
N24, W31 = "narrow", "wide"
# QAGNN_Message_Passing builds its layers with GATConvE's default head count 4; the mp rows at other head counts build them
# with head_count=H (_mp_module).  At k = 0 there are no layers and the plan is made at H = 4.
CASES = [
    # ---- fp32: split-bf16 wgmma GEMMs (passes 3) and the exact-fp32 FFMA GEMM --------------------------------------------
    Case(M, 4, 200, 2, "tiled", "fp32", "tc tiled fast fused res", ht=(2, N24), twin={"QAGNN_PROJ_RESIDENT": "0"}),
    Case(M, 4, 200, 2, "ragged", "fp32", "tc tiled fast fused res", ht=(2, N24)),
    Case(M, 4, 200, 1, "tiled", "fp32", "tc tiled fused", env={"QAGNN_MP_FASTPROJ": "0"}, ht=(2, N24)),
    Case(M, 4, 200, 1, "ragged", "fp32", "tc tiled fused", env={"QAGNN_MP_FASTPROJ": "0"}, ht=(2, N24)),
    Case(M, 4, 200, 1, "ragged", "fp32", "tc tiled fast res", env={"QAGNN_MLP_FUSED": "0"}, ht=(2, N24),
         twin={"QAGNN_MLP_FUSED": "1"}),
    Case(M, 4, 200, 1, "edgecap", "fp32", "tc tiled fast fused res", env={"QAGNN_TC_2CTA": "0"}, ht=(2, N24),
         twin={"QAGNN_TC_2CTA": "1"}),
    Case(M, 4, 200, 0, "tiled", "fp32", "tc tiled fused"),
    Case(M, 4, 200, 0, "ragged", "fp32", "tc tiled fused"),
    Case(M, 4, 200, 0, "ragged", "fp32", "tiled zp", env={"QAGNN_GEMM": "ffma"}),
    Case(M, 4, 100, 0, "tiled", "fp32", "tiled zp"),                                   # d 25: no wgmma (D % 8 != 0)
    Case(M, 4, 200, 1, "general", "fp32", "", env={"QAGNN_GEMM": "ffma"}),             # d 50: basic
    Case(M, 4, 200, 1, "ragged", "fp32", "tiled zp", env={"QAGNN_GEMM": "ffma"}, ht=(2, N24)),
    Case(M, 4, 100, 2, "ragged", "fp32", "tiled zp", ht=(1, N24)),
    # D/2 = 4 is narrower than a wgmma GEMM (N >= 8), so emb_score cannot run on the tensor cores: the general form.  (The
    # fast form was planned here and its emb_score GEMM refused the call.)
    Case(M, 1, 8, 1, "tiled", "fp32", "tc tiled fused", ht=(1, N24)),
    Case(M, 1, 128, 2, "general", "fp32", "tc slice fused"),                           # d 128: two 64-column slices
    Case(M, 1, 128, 1, "ragged", "fp32", "tc slice fused"),                            # DP 128 > 64: no tiles
    Case(M, 8, 64, 1, "ragged", "fp32", "tc tiled fast fused res", env={"QAGNN_MP_WARPS": "31"}, ht=(1, W31),
         twin={"QAGNN_MP_WARPS": None}),
    Case(M, 8, 64, 1, "tiled", "fp32", "tc tiled fast fused res", env={"QAGNN_MP_WARPS": "31"}, ht=(1, W31),
         twin={"QAGNN_MP_WARPS": None}),
    Case(M, 2, 104, 1, "ragged", "fp32", "tc tiled fast fused res", env={"QAGNN_MP_WARPS": "31"}, ht=(2, W31),
         twin={"QAGNN_MP_WARPS": None}),
    Case(M, 8, 400, 1, "edgecap", "fp32", "tc tiled fast", ht=(2, N24)),               # H*DP 416; K 600 > 320: no res
    Case(M, 16, 208, 1, "tiled", "fp32", "tc tiled fast fused res", ht=(1, N24)),      # d 13
    Case(L, 2, 104, 1, "tiled", "fp32", "tc tiled fast fused", env={"QAGNN_MP_WARPS": "31"}, ht=(2, W31),
         twin={"QAGNN_MP_WARPS": None}),
    Case(L, 2, 10, 1, "tiled", "fp32", "tiled zp", ht=(1, N24)),                       # d 5: only the tiled kernel takes it
    Case(L, 1, 256, 1, "general", "fp32", "tc"),                                       # basic, D > 208: two MLP launches
    Case(L, 8, 128, 1, "general", "fp32", "tc slice fused"),
    Case(L, 8, 128, 1, "ragged", "fp32", "tc slice fused", env={"QAGNN_MP_PATH": "csr"}),
    Case(L, 8, 32, 1, "tiled", "fp32", "tc tiled fast fused", env={"QAGNN_MP_WARPS": "24"}, ht=(1, N24),
         twin={"QAGNN_MP_WARPS": None}),
    Case(L, 2, 200, 1, "ragged", "fp32", "tc fused"),                                  # d 100: basic
    Case(L, 16, 320, 1, "tiled", "fp32", "tc tiled fast", ht=(1, N24)),                # H*DP 320 > 256
    Case(L, 16, 64, 1, "packed", "fp32", "tc tiled fast fused", env={"QAGNN_TC_2CTA": "0"}, ht=(1, N24),
         twin={"QAGNN_TC_2CTA": "1"}),
    # ---- bf16 autocast: single-pass bf16 wgmma GEMMs (passes 1), or the FFMA GEMM on rounded inputs -----------------------
    Case(M, 4, 200, 2, "tiled", "bf16", "tc tiled fast fused", ht=(2, N24)),
    Case(M, 4, 200, 2, "ragged", "bf16in", "tc tiled fast fused", ht=(2, N24)),
    Case(M, 4, 200, 1, "tiled", "bf16", "tc tiled fused", env={"QAGNN_MP_FASTPROJ": "0"}, ht=(2, N24)),
    Case(M, 4, 200, 1, "ragged", "bf16", "tc tiled fast", env={"QAGNN_MLP_FUSED": "0"}, ht=(2, N24),
         twin={"QAGNN_MLP_FUSED": "1"}),
    Case(M, 4, 200, 1, "edgecap", "bf16", "tc tiled fast fused", env={"QAGNN_TC_2CTA": "0"}, ht=(2, N24),
         twin={"QAGNN_TC_2CTA": "1"}),
    Case(M, 4, 200, 0, "tiled", "bf16", "tc tiled fused"),
    Case(M, 4, 200, 0, "ragged", "bf16in", "tc tiled fused"),
    Case(M, 4, 200, 0, "tiled", "bf16", "tiled zp", env={"QAGNN_GEMM": "ffma"}),
    Case(M, 4, 200, 0, "ragged", "bf16in", "tiled zp", env={"QAGNN_GEMM": "ffma"}),
    Case(M, 4, 200, 2, "tiled", "bf16", "tiled zp", env={"QAGNN_GEMM": "ffma"}, ht=(2, N24)),
    Case(M, 4, 100, 1, "ragged", "bf16", "tiled zp", ht=(1, N24)),
    Case(M, 1, 8, 2, "tiled", "bf16", "tc tiled fused", ht=(1, N24)),                 # D/2 = 4: the general form
    Case(M, 2, 104, 1, "tiled", "bf16in", "tc tiled fast fused", env={"QAGNN_MP_WARPS": "7"}, ht=(2, N24),
         twin={"QAGNN_MP_WARPS": None}),
    Case(M, 8, 200, 1, "ragged", "bf16", "tc tiled fast fused", ht=(1, N24)),          # d 25, fast form at H = 8
    Case(M, 8, 400, 1, "ragged", "bf16", "tc tiled fast", ht=(2, N24)),                # H*DP 416
    Case(M, 16, 208, 2, "tiled", "bf16", "tc tiled fast fused", ht=(1, N24)),          # d 13
    Case(L, 2, 24, 1, "tiled", "bf16in", "tc tiled fast fused", ht=(1, N24)),
    Case(L, 2, 64, 1, "ragged", "bf16", "tc slice fused", env={"QAGNN_MP_PATH": "csr"}),
    Case(L, 2, 200, 1, "ragged", "bf16", "tc fused"),                                  # d 100: basic
    Case(L, 2, 10, 1, "ragged", "bf16", "tiled zp", ht=(1, N24)),
    Case(L, 8, 200, 1, "tiled", "bf16", "tc tiled fast fused", ht=(1, N24)),           # d 25: aggr split after the kernel
    Case(L, 8, 128, 1, "general", "bf16", "tc slice fused"),
    Case(L, 1, 256, 1, "general", "bf16in", "tc"),
    Case(L, 16, 400, 1, "tiled", "bf16", "tc tiled fast", ht=(1, N24)),                # d 25, H*DP 448 > 256
    Case(L, 16, 64, 1, "ragged", "bf16", "tc tiled fast fused", env={"QAGNN_MP_WARPS": "31"}, ht=(1, W31),
         twin={"QAGNN_MP_WARPS": None}),
]


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _batch(D, seed, n=40):
    """Six graphs of n padded nodes whose edges stay inside each graph's first adj_lengths nodes: a full graph, graphs of
    one node and of nodes without edges, and ordinary ones.  Edges are sorted by graph, so a ragged batch keeps their order."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor([n, 9, 1, n - 3, 17, 28])
    eis, ets = [], []
    for b, L_ in enumerate(lens.tolist()):
        m = 0 if b in (1, 2) else 3 * L_
        eis.append(torch.stack([torch.randint(0, L_, (m,), generator=g), torch.randint(0, L_, (m,), generator=g)]))
        ets.append(torch.randint(0, R, (m,), generator=g))
    B = lens.numel()
    nt = torch.randint(0, 3, (B, n), generator=g)
    nt[:, 0] = 3
    return {"H": torch.randn(B, n, D, generator=g) * 0.5, "extra": torch.randn(B * n, D, generator=g) * 0.5,
            "edge_index": torch.cat([e + b * n for b, e in enumerate(eis)], 1), "edge_type": torch.cat(ets),
            "node_type": nt, "node_score": torch.randn(B, n, 1, generator=g), "adj_lengths": lens, "local": (eis, ets),
            "n": n}


def _state(c):
    return O.random_state_dict(max(c.layers, 1), c.D, T, R, "peaky", seed=97 * c.H + c.D + 7 * c.k)


def _layer_module(H, D, sd):
    enc = torch.nn.Sequential(torch.nn.Linear(R + 1 + 2 * T, D), torch.nn.BatchNorm1d(D), torch.nn.ReLU(), torch.nn.Linear(D, D))
    layer = qagnn_b200.GATConvE(None, D, T, R, enc, head_count=H)
    layer.load_state_dict({k[len("gnn_layers.0."):]: v for k, v in sd.items() if k.startswith("gnn_layers.0.")}, strict=True)
    return layer.eval().to(DEV)


def _mp_module(H, D, k, sd):
    mod = qagnn_b200.QAGNN_Message_Passing(None, k, T, R, D, D, D)
    mod.gnn_layers = torch.nn.ModuleList([qagnn_b200.GATConvE(None, D, T, R, mod.edge_encoder, head_count=H) for _ in range(k)])
    mod.load_state_dict({kk: v for kk, v in sd.items() if k > 0 or not kk.startswith("gnn_layers.")}, strict=True)
    return mod.eval().to(DEV)


def _ragged(b, node_spare=23, **kw):
    from tests.test_gpu_ragged import ragged_inputs
    return ragged_inputs(b["H"], b["edge_index"], b["edge_type"], b["node_type"], b["node_score"], b["adj_lengths"], b["n"],
                         node_capacity=int(b["adj_lengths"].sum()) + node_spare, **kw)


def _call(c, mod, b, layout):
    """One forward of row c's entry point on `layout` -> {out, alpha, aggr, layers} (the entry point's outputs; alpha /
    aggr for a layer, every layer's x for the message passing) as CPU tensors."""
    from qagnn_b200.modeling_qagnn import GraphPrep
    n, D = b["n"], c.D
    dt = BF if c.prec == "bf16in" else torch.float32
    x, extra, nt, ns = b["H"].reshape(-1, D), b["extra"], b["node_type"].reshape(-1), b["node_score"]
    ei, et = b["edge_index"].to(DEV), b["edge_type"].to(DEV)
    adj, prep = (ei, et), None
    if layout in ("packed", "edgecap"):
        cap = ei.size(1) + 37 if layout == "edgecap" else None
        adj = Dt.pack_adj(*b["local"], n, pin=False, edge_capacity=cap).to(DEV)
    elif layout == "ragged":
        adj, Hp, nt, ns, rows = _ragged(b)
        adj = adj.to(DEV)
        x = Hp
        extra = torch.zeros_like(Hp)
        extra[:rows.numel()] = b["extra"][rows]
    elif layout == "general" or c.entry == "layer":
        prep = GraphPrep(ei, et, nt.to(DEV), T, R, n_per_graph=0 if layout == "general" else n)
    ctx = torch.autocast("cuda", dtype=BF) if c.prec != "fp32" else torch.autocast("cuda", enabled=False)
    with torch.no_grad(), ctx:
        if c.entry == "layer":  # a padded batch through its prep, a PackedAdj by itself
            a = None if prep is not None else adj
            (out, (_, alpha)), aggr = mod(x.to(DEV, dt), a, None, nt.to(DEV), extra.to(DEV, dt), return_attention_weights=True,
                                          prep=prep, return_aggr=True)
            res = {"out": out, "alpha": alpha, "aggr": aggr}
        else:
            H_in = x if layout == "ragged" else b["H"]
            out, layers = mod(H_in.to(DEV, dt), adj, nt.to(DEV), ns.to(DEV), prep=prep, return_layers=True)
            res = {"out": out.reshape(-1, D), "layers": layers}
    torch.cuda.synchronize()
    return {k: v.detach().cpu() for k, v in res.items()}


# ---------------------------------------------------------------------------------------------------------------------
# the plan, from the kernels that ran
# ---------------------------------------------------------------------------------------------------------------------
def _kernels(fn, sessions=3):
    """(fn(), names of the CUDA kernels it launched), from torch.profiler's CUPTI kernel records.  On an H100 a session now and
    then comes back with fewer kernel records than kernel launches (seen: none at all, or all but the GEMM's), while the call's
    results are complete.  A lost record can only hide a kernel, never show one that did not run, and every fn here repeats
    the same launches: so fn is profiled until one session has a kernel record per launch, or `sessions` times, and the names
    are the union over those sessions."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for _ in range(sessions):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        evs = prof.events()
        names |= {e.name for e in evs}
        launches = sum(e.name.startswith(("cudaLaunchKernel", "cuLaunchKernel")) for e in evs)
        records = sum(e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")) for e in evs)
        if records >= launches > 0:
            break
    assert any("qagnn" in s for s in names), f"the profiler recorded no kernel of the library: {sorted(names)[:12]}"
    return res, names


def _has(names, kernel):
    return any(re.search(r"\b" + kernel + r"\b", s) for s in names)


def _assert_plan(c, names):
    """The kernels each plan field implies, and no kernel of a plan that did not run."""
    p, nl = c.plan, c.layers
    seen = lambda k: _has(names, k)  # noqa: E731
    want = {}
    ht = sorted({m.groups() for s in names for m in [re.search(r"mp_headtile_kernel<(\d+), ?(\d+), ?(true|false)>", s)] if m})
    if p["tiled"] and nl:
        cpl, build = c.ht
        assert ht == [(str(cpl), str(WMAX[build]), "true" if c.layout == "ragged" else "false")], f"tiled kernel: {ht}"
    else:
        assert not ht, f"tiled kernel ran: {ht}"
    want["mp_slice_scores_kernel"] = want["mp_slice_aggregate_kernel"] = p["slice"] and nl > 0
    basic = not p["tiled"] and not p["slice"] and nl > 0
    want["mp_scores_kernel"] = want["mp_aggregate_kernel"] = basic
    one = p["passes"] == 1
    want["gemm_tc_kernel"] = p["tc"] and not one
    want["gemm_bf16_kernel"] = p["tc"] and one
    want["mlp_tc_kernel"] = p["mlp_fused"] and not one and nl > 0
    want["mlp_bf16_kernel"] = p["mlp_fused"] and one and nl > 0
    want["proj_resident_kernel"] = c.resident
    want["f32_to_bf16_kernel"] = want["bf16_to_f32_kernel"] = not p["tc"] and one
    if not p["tc"]:
        want["sgemm_tn_kernel"] = True
    fast = p["fast"] and c.entry == "mp"  # a single layer never runs the fast-form projection
    want["sin_basis_planes_kernel"] = want["copy_plane_columns_kernel"] = fast
    if not p["zero_pads"] or c.DP != c.d:  # zero_head_pads launches nothing when no head has pad columns
        want["zero_head_pads_kernel"] = p["zero_pads"]
    bad = {k: v for k, v in want.items() if seen(k) != v}
    assert not bad, f"{c.id}: expected presence {bad} differs; kernels: {sorted(s[:60] for s in names if 'qagnn' in s)}"


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def _bf(t):
    return t.float().to(BF).double()


def _valid(res, sel):
    """The part of a padded-layout result that a ragged batch holds: node rows `rows`, every real edge and the self loops
    of those rows (alpha lists real edges, then one self loop per row)."""
    if sel is None:
        return res
    rows, E = sel
    out = {}
    for k, v in res.items():
        if k == "alpha":
            out[k] = torch.cat([v[:E], v[E + rows]])
        elif k == "layers":
            out[k] = v[:, rows]
        else:
            out[k] = v[rows]
    return out


def _ragged_valid(res, nv, E):
    out = {}
    for k, v in res.items():
        if k == "alpha":
            out[k] = torch.cat([v[:E], v[E:E + nv]])
        elif k == "layers":
            out[k] = v[:, :nv]
        else:
            out[k] = v[:nv]
    return out


def _oracle(c, b, sd, rounded):
    """fp64 oracle outputs in the padded layout; `rounded`: on bf16_rn of the call's inputs (the FFMA bf16 contract)."""
    rnd = _bf if rounded else (lambda t: t.double())
    ei, et, nt = b["edge_index"], b["edge_type"], b["node_type"].reshape(-1)
    if c.entry == "layer":
        out, _, alpha, aggr = O.gatconve_forward(sd, "gnn_layers.0", rnd(b["H"].reshape(-1, c.D)), ei, et, nt, rnd(b["extra"]),
                                                 T, R, head_count=c.H, dtype=F64)
        return {"out": out, "alpha": alpha, "aggr": aggr}
    out, _, layers = O.message_passing_forward(sd, rnd(b["H"]), ei, et, b["node_type"], b["node_score"], c.k, T, R,
                                               head_count=c.H, dtype=F64, return_layers=True)
    lay = torch.stack([l_["x"] for l_ in layers]) if layers else torch.zeros(0, out.numel() // c.D, c.D, dtype=F64)
    return {"out": out.reshape(-1, c.D), "layers": lay}


def _check_fp32(c, got, ref, label):
    for k in got:
        Hh.assert_close(got[k], ref[k], f"{c.id} {label} {k}")


def _check_ffma_bf16(c, got, ref, label):
    """the FFMA GEMM under bf16: the fp32 path on rounded inputs, its output rounded once"""
    for k in got:
        rtol = Hh.RTOL + (U if k == "out" else 0.0)
        Hh.assert_close(got[k].float(), ref[k], f"{c.id} {label} {k}", rtol=rtol)


def _emulation(c, b, sd, teacher):
    """the contract emulation of tests/test_gpu_eval_bf16.py at row c's H and k, following the plan that ran"""
    from tests import test_gpu_eval_bf16 as E16
    if c.entry == "layer":
        emu, mag, rss = E16._emulate_layer(sd, "gnn_layers.0", "gnn_layers.0.edge_encoder", _bf(b["H"].reshape(-1, c.D)),
                                           _bf(b["extra"]), b["edge_index"], b["edge_type"], b["node_type"].reshape(-1), T, R,
                                           c.H, E16.Variant())
        return {"out": (_bf(emu), mag, rss)}, None
    fx = {"case": {"D": c.D, "k": c.k}, "n_ntype": T, "n_etype": R}
    fast = c.plan["fast"]
    emu, mag, rss, layers = E16._emulate_mp(fx, b, sd, fast, teacher_layers=teacher, H=c.H, k=c.k)
    whole = E16._emulate_mp(fx, b, sd, fast, H=c.H, k=c.k)
    return {"out": (_bf(emu), mag, rss), "layers": layers}, whole


def _check_emulation(c, got, emu, whole, sel, label):
    from tests import test_gpu_eval_bf16 as E16
    take = lambda t: _valid({"out": t}, sel)["out"]  # noqa: E731
    D = c.D
    for l_, (X, m, r) in enumerate(emu.get("layers", [])):
        ok, frac, worst = E16._bars_hold(got["layers"][l_].reshape(-1, D), take(X), take(m), take(r))
        assert ok, f"{c.id} {label} layer {l_}: {frac:.3f} over the tight bar, worst {worst:.2f} of the loose bar"
    e, m, r = emu["out"]
    ok, frac, worst = E16._bars_hold(got["out"].reshape(-1, D), take(e), take(m), take(r), ulp_out=True)
    assert ok, f"{c.id} {label} out: {frac:.3f} over the tight bar, worst {worst:.2f} of the loose bar"
    if whole is not None:
        e2, m2, r2, _ = whole
        assert E16._whole_forward_holds(got["out"].reshape(-1, D), take(e2), take(m2), take(r2)), f"{c.id} {label}: whole forward"


# ---------------------------------------------------------------------------------------------------------------------
# the table
# ---------------------------------------------------------------------------------------------------------------------
def _set_switches(monkeypatch, env):
    for name in SWITCHES:
        if env.get(name) is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, env[name])


def _assert_bits(a, b, what):
    for k in a:
        if not torch.equal(a[k], b[k]):
            diff = (a[k].double() - b[k].double()).abs()
            raise AssertionError(f"{what} {k}: {int((diff > 0).sum())} elements differ, max |diff| {diff.max().item():.3e}")


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_forward_plan(c, monkeypatch):
    _set_switches(monkeypatch, c.env)
    b = _batch(c.D, seed=97 * c.H + c.D + 7 * c.k)
    sd = _state(c)
    mod = _layer_module(c.H, c.D, sd) if c.entry == "layer" else _mp_module(c.H, c.D, c.k, sd)
    first = _call(c, mod, b, c.layout)  # folds the weights, whose kernels are not the forward's
    got, names = _kernels(lambda: _call(c, mod, b, c.layout))
    _assert_bits(got, first, f"{c.id}: a second call")
    _assert_plan(c, names)
    out_dt = torch.float32 if c.prec == "fp32" else BF
    assert got["out"].dtype == out_dt and bool(torch.isfinite(got["out"].float()).all())

    # equal bits where the arithmetic is the same
    if c.twin is not None:
        _set_switches(monkeypatch, {**c.env, **c.twin})
        _assert_bits(got, _call(c, mod, b, c.layout), f"{c.id} against {c.twin}")
        _set_switches(monkeypatch, c.env)
    sel, full = None, got
    if c.layout == "edgecap":
        _assert_bits(got, _call(c, mod, b, "packed"), f"{c.id} against the exact packed batch")
    if c.layout == "ragged":
        # the padded batch on the same plan (per-graph prep for the tiled kernel): every valid row's sums run in the same order
        padded = _call(c, mod, b, "tiled" if c.plan["tiled"] else "general")
        rows, E = _ragged(b)[4], b["edge_index"].size(1)
        sel = (rows, E)
        _assert_bits(_ragged_valid(got, rows.numel(), E), _valid(padded, sel), f"{c.id}: ragged rows against the padded rows")
        full = padded

    # the high-precision reference, on the padded layout; a ragged batch's valid rows against it gathered at `rows`
    views = [(full, None, "padded" if sel else "")] + ([(_ragged_valid(got, sel[0].numel(), sel[1]), sel, "ragged")] if sel else [])
    if c.prec == "fp32":
        ref = _oracle(c, b, sd, rounded=False)
        for res, s, label in views:
            _check_fp32(c, res, _valid(ref, s), label)
    elif not c.plan["tc"]:
        ref = _oracle(c, b, sd, rounded=True)
        for res, s, label in views:
            _check_ffma_bf16(c, res, _valid(ref, s), label)
    else:
        emu, whole = _emulation(c, b, sd, full.get("layers"))
        for res, s, label in views:
            _check_emulation(c, res, emu, whole, s, label)


# ---------------------------------------------------------------------------------------------------------------------
# the bars reject seeded faults
# ---------------------------------------------------------------------------------------------------------------------
def _find(entry, H, D, k, layout, prec):
    return next(c for c in CASES if (c.entry, c.H, c.D, c.k, c.layout, c.prec) == (entry, H, D, k, layout, prec) and not c.env)


def _run_case(c, monkeypatch):
    _set_switches(monkeypatch, c.env)
    b = _batch(c.D, seed=97 * c.H + c.D + 7 * c.k)
    sd = _state(c)
    mod = _layer_module(c.H, c.D, sd) if c.entry == "layer" else _mp_module(c.H, c.D, c.k, sd)
    return b, sd, _call(c, mod, b, c.layout)


@pytest.mark.gpu
@pytest.mark.parametrize("fp32,bf16", [((L, 16, 320, 1, "tiled", "fp32"), (L, 16, 400, 1, "tiled", "bf16")),
                                       ((L, 2, 10, 1, "tiled", "fp32"), (L, 2, 24, 1, "tiled", "bf16in"))],
                         ids=["H16", "H2"])
def test_bars_reject_two_swapped_heads(fp32, bf16, monkeypatch):
    from tests import test_gpu_eval_bf16 as E16
    c = _find(*fp32)
    b, sd, got = _run_case(c, monkeypatch)
    ref = _oracle(c, b, sd, rounded=False)
    _check_fp32(c, got, ref, "")
    perm = [1, 0] + list(range(2, c.H))
    with pytest.raises(AssertionError):
        Hh.assert_close(got["alpha"], ref["alpha"][:, perm], "alpha, heads 0 and 1 swapped")
    with pytest.raises(AssertionError):
        Hh.assert_close(got["aggr"], ref["aggr"].view(-1, c.H, c.d)[:, perm].reshape(-1, c.D), "aggr, heads 0 and 1 swapped")
    c = _find(*bf16)
    b, sd, got = _run_case(c, monkeypatch)
    emu, _ = _emulation(c, b, sd, None)
    _check_emulation(c, got, emu, None, None, "")
    e, m, r = E16._emulate_layer(sd, "gnn_layers.0", "gnn_layers.0.edge_encoder", _bf(b["H"].reshape(-1, c.D)), _bf(b["extra"]),
                                 b["edge_index"], b["edge_type"], b["node_type"].reshape(-1), T, R, c.H,
                                 E16.Variant(swap_heads=True))
    assert not E16._bars_hold(got["out"], _bf(e), m, r, ulp_out=True)[0], "a reference with two heads swapped passes"


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_bars_reject_a_perturbed_vx_column_at_k0(prec, monkeypatch):
    """At k = 0 the output is GELU(Vh(H) + Vx(H)): a reference with one column of Vx changed must fail, so the plain
    reference passing shows that the Vx operand was H."""
    c = _find(M, 4, 200, 0, "tiled", prec)
    b, sd, got = _run_case(c, monkeypatch)
    bad = dict(sd)
    bad["Vx.weight"] = sd["Vx.weight"].clone()
    bad["Vx.weight"][:, 5] += 0.25
    if prec == "fp32":
        _check_fp32(c, got, _oracle(c, b, sd, rounded=False), "")
        with pytest.raises(AssertionError):
            _check_fp32(c, got, _oracle(c, b, bad, rounded=False), "perturbed Vx")
    else:
        emu, whole = _emulation(c, b, sd, got["layers"])
        _check_emulation(c, got, emu, whole, None, "")
        emu, whole = _emulation(c, b, bad, got["layers"])
        with pytest.raises(AssertionError):
            _check_emulation(c, got, emu, whole, None, "perturbed Vx")


@pytest.mark.gpu
def test_bf16_bars_reject_the_fp32_forward_at_one_head(monkeypatch):
    c = _find(L, 1, 256, 1, "general", "bf16in")
    b, sd, got = _run_case(c, monkeypatch)
    emu, _ = _emulation(c, b, sd, None)
    _check_emulation(c, got, emu, None, None, "")
    c32 = _find(L, 1, 256, 1, "general", "fp32")
    b32, sd32, got32 = _run_case(c32, monkeypatch)
    assert torch.equal(b32["H"], b["H"]) and all(torch.equal(sd32[k], sd[k]) for k in sd)
    with pytest.raises(AssertionError):
        _check_emulation(c, {"out": got32["out"].to(BF)}, emu, None, None, "fp32 forward")


@pytest.mark.gpu
def test_ragged_bar_rejects_a_reference_one_row_off(monkeypatch):
    c = _find(M, 4, 200, 2, "ragged", "fp32")
    b, sd, got = _run_case(c, monkeypatch)
    rows, E = _ragged(b)[4], b["edge_index"].size(1)
    ref = _oracle(c, b, sd, rounded=False)
    mine = _ragged_valid(got, rows.numel(), E)
    _check_fp32(c, mine, _valid(ref, (rows, E)), "")
    with pytest.raises(AssertionError):
        _check_fp32(c, mine, _valid(ref, (rows + 1, E)), "one row off")
