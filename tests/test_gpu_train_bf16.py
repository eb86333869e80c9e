"""Training under fp16 / bf16 autocast: the message-passing core on 16-bit operands and the edge encoder's BatchNorm moments.

  * the 16-bit core (qagnn_mp_core_*_typed) against the fp32 core run on the same values widened: aggr, alpha and d_qkm bit
    for bit after rounding, d_ke / d_me within one unit in the last place, at every head count and chunk count the kernels
    dispatch on, on the training goldens' graphs and on a 320-graph loader batch at an edge capacity;
  * the edge encoder's running statistics after a micro-step with more than 65504 edge positions (fp16's largest value);
  * the module under bf16 autocast against the same module with the graph part in fp64 torch ops;
  * TrainStep(autocast_dtype=torch.bfloat16) against eager bf16 micro-steps, and an eager bf16 step without host syncs.
Needs a GPU: run with -m gpu."""
import copy
import math

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import make_goldens as MG
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200 import training as TR
from qagnn_b200.modeling_qagnn import SUPPORTED_HEAD_COUNTS, GraphPrep
from qagnn_b200.pipeline import TrainStep
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R = 4, 38
NC = R * T * T + T
DTYPES = [torch.float16, torch.bfloat16]
MANT = {torch.float16: 10, torch.bfloat16: 7}  # explicit mantissa bits: one ulp at 1.0 is 2^-MANT


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


# ---- the core on 16-bit operands against the fp32 core -------------------------------------------------------------------
def _run_core(prep, shape, qkm, ke, me, G):
    leaves = [t.detach().clone().requires_grad_(True) for t in (qkm, ke, me)]
    aggr, alpha = TR._MPCore.apply(*leaves, prep, shape, True)
    return (aggr.detach(), alpha) + tuple(torch.autograd.grad(aggr, leaves, G))


def _check_exact(prep, N, D, H, dt, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkm = torch.randn(N, 3 * D, generator=g, device=DEV)
    qkm[:, :D] /= (D // H) ** 0.5  # Q / sqrt(d) as the layer scales it
    ke, me = torch.randn(NC, D, generator=g, device=DEV), torch.randn(NC, D, generator=g, device=DEV)
    G = torch.randn(N, D, generator=g, device=DEV)
    lo = [t.to(dt) for t in (qkm, ke, me, G)]
    shape = (N, prep.E, D, H, T, R)
    aggr, alpha, d_qkm, d_ke, d_me = _run_core(prep, shape, *lo)
    raggr, ralpha, rd_qkm, rd_ke, rd_me = _run_core(prep, shape, *(t.float() for t in lo))
    assert aggr.dtype == d_qkm.dtype == d_ke.dtype == d_me.dtype == dt and alpha.dtype == torch.float32
    assert bool(torch.isfinite(raggr).all()) and bool(torch.isfinite(rd_qkm).all())
    # atomic-free kernels: the fp32 result rounded to nearest even, bit for bit
    for name, got, ref in (("aggr", aggr, raggr.to(dt)), ("alpha", alpha, ralpha), ("d_qkm", d_qkm, rd_qkm.to(dt))):
        bad = int((_bits(got) != _bits(ref)).sum())
        assert bad == 0, f"{dt} H={H} D={D}: {name} differs from the rounded fp32 core in {bad} of {got.numel()} elements"
    # d_ke / d_me: fp32 atomics in both runs, in no fixed order, so a value that lands near a rounding boundary may round
    # the other way: one ulp of the dtype at the element's magnitude.  The fp32 reference itself moves between runs by the
    # order of its additions (at most n 2^-24 of the row's absolute sum for n edges per combo): 2^-16 of the row's largest
    # entry covers that for the few thousand edges per combo here.
    for name, got, ref in (("d_ke", d_ke, rd_ke), ("d_me", d_me, rd_me)):
        a, b = got.double(), ref.to(dt).double()
        mag = torch.maximum(a.abs(), b.abs()).clamp_min(torch.finfo(dt).tiny)
        tol = torch.exp2(torch.floor(torch.log2(mag)) - MANT[dt]) + 2.0 ** -16 * ref.double().abs().amax(1, keepdim=True)
        over = float(((a - b).abs() - tol).max())
        assert over <= 0, f"{dt} H={H} D={D}: {name} is more than one ulp from the rounded fp32 core (by {over:.3e})"


def _d_for(H):
    return 200 if 200 % H == 0 else 208  # the decoder's width; 16 heads need D % 16 == 0 (d = 13)


# D per head count giving CH = ceil(D / 128) = 1, 2, 4, 8: every (H, CH) instantiation; several have d % 4 != 0, so the
# 4-element chunks straddle two heads
SHAPES = [(1, 36), (1, 200), (1, 500), (1, 1020), (2, 40), (2, 200), (2, 388), (2, 1000), (4, 100), (4, 232), (4, 400),
          (4, 1020), (8, 64), (8, 200), (8, 488), (8, 1000), (16, 64), (16, 208), (16, 400), (16, 1024)]


@pytest.fixture(scope="module")
def random_prep():
    g = torch.Generator().manual_seed(0)
    N, E = 300, 1200
    ei = torch.randint(0, N, (2, E), generator=g)
    return N, GraphPrep(ei.to(DEV), torch.randint(0, R, (E,), generator=g).to(DEV), torch.randint(0, T, (N,), generator=g).to(DEV), T, R)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("H,D", SHAPES)
def test_16bit_core_equals_rounded_fp32_core_every_instantiation(random_prep, H, D, dt):
    assert (D + 127) // 128 in (1, 2, 4, 8)
    N, prep = random_prep
    _check_exact(prep, N, D, H, dt, seed=H * 4096 + D)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", Hh.golden_names("train"))
def test_16bit_core_on_training_golden_graphs(name, dt):
    inp, _ = Hh.regen_mp_inputs(Hh.load_golden(name))
    nt = inp["node_type"].reshape(-1)
    prep = GraphPrep(inp["edge_index"].to(DEV), inp["edge_type"].to(DEV), nt.to(DEV), T, R)
    for H in SUPPORTED_HEAD_COUNTS:
        _check_exact(prep, nt.numel(), _d_for(H), H, dt, seed=H)


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    """A loader-shaped split of 64 questions x 5 choices (n = 200 nodes per sub-graph)."""
    path = str(tmp_path_factory.mktemp("split") / "train.graph.adj.pk")
    Dt.synth_adj_pickle(path, 64 * 5, seed=5)
    _, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, 200, 5)
    return ntypes, scores, lens, flat


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_16bit_core_on_a_320_graph_batch_at_an_edge_capacity(split, dt):
    ntypes, _, _, flat = split
    qs = np.arange(64)
    K = flat.max_batch_edges(64) + 1000
    adj = flat.pack(qs, pin=False, edge_capacity=K).to(DEV)
    nt = ntypes[qs].reshape(-1).to(DEV)
    prep = GraphPrep(adj.edge_index, adj.edge_type, nt, T, R, 200, graph_ptr=adj.graph_ptr_dev, max_edges=adj.max_edges)
    assert prep.packed and prep.E == K > adj.n_edges and adj.n_edges + nt.numel() > 65504
    for H in SUPPORTED_HEAD_COUNTS:
        _check_exact(prep, nt.numel(), _d_for(H), H, dt, seed=100 + H)


# ---- decoders and batches (as tests/test_gpu_train_step.py builds them) ---------------------------------------------------
def _split_batch(split, qs, capacity, seed, sent_dim=48, n_concept=300):
    ntypes, scores, lens, flat = split
    adj = flat.pack(np.asarray(qs), pin=False, edge_capacity=capacity).to(DEV)
    B = len(qs) * 5
    g = torch.Generator().manual_seed(seed)
    cid = torch.randint(1, n_concept + 1, (B, 200), generator=g)
    cid[:, 0] = 0
    batch = {"sent_vecs": torch.randn(B, sent_dim, generator=g), "concept_ids": cid, "node_type_ids": ntypes[qs].reshape(B, 200),
             "node_scores": scores[qs].reshape(B, 200, 1), "adj_lengths": lens[qs].reshape(B)}
    return {k: v.to(DEV) for k, v in batch.items()}, adj


def _split_decoder(dropout=0.0, D=64):
    torch.manual_seed(8)
    dec = qagnn_b200.QAGNN(None, 2, T, R, 48, 300, D, 32, 2, D, 1, dropout, dropout, dropout)
    dec.gnn.load_state_dict(O.random_state_dict(2, D, T, R, "prod", seed=8))
    return dec.to(DEV).train()


def _zero_dropout(dec):
    for m in dec.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    dec.gnn.dropout_rate = 0.0


def _args(batch, sv, ns, adj):
    return sv, batch["concept_ids"], batch["node_type_ids"], ns, batch["adj_lengths"], adj


def _leaves(batch):
    return batch["sent_vecs"].clone().requires_grad_(True), batch["node_scores"].clone().requires_grad_(True)


def _autocast(dt):
    return torch.autocast("cuda", dtype=dt, cache_enabled=False) if dt is not None else torch.enable_grad()


# ---- BatchNorm moments of the edge encoder at scale ------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_edge_encoder_running_statistics_past_fp16_range(split, dt):
    """One micro-step on 320 sub-graphs (E' = E + N > 65504 edge positions).  Under fp16 the edge count overflowed when the
    moments were taken in the autocast dtype, and running_var became NaN."""
    qs = list(range(64))
    batch, adj = _split_batch(split, qs, None, 1)
    assert adj.n_edges + batch["node_type_ids"].numel() > 65504
    dec = _split_decoder()
    _zero_dropout(dec)
    ref_dec, dec = copy.deepcopy(dec), dec
    w = torch.randn(len(qs) * 5, 1, device=DEV)
    for d, amp in ((ref_dec, None), (dec, dt)):
        sv, ns = _leaves(batch)
        with _autocast(amp):
            logits, _ = d(*_args(batch, sv, ns, adj))
            loss = (logits.float() * w).sum()
        loss.backward()
        assert bool(torch.isfinite(loss)) and bool(torch.isfinite(sv.grad).all())
    bn, ref_bn = dec.gnn.edge_encoder[1], ref_dec.gnn.edge_encoder[1]
    assert int(bn.num_batches_tracked) == int(ref_bn.num_batches_tracked) > 0
    # h = lin0(onehot) is computed from weights rounded to the dtype and is itself rounded to it: each entry is the sum of
    # three weights and a bias, so it carries a relative error of a few units u = 2^-(MANT+1).  The moments are then exact
    # fp32 weighted sums of those entries, so mean and variance move by a few u of the tensor's scale (max |h| and max h^2),
    # and the running statistics by that times (1 - keep).  The bar is 16 u of the tensor's largest entry.
    u = 2.0 ** -(MANT[dt] + 1)
    for name, got, ref in (("running_mean", bn.running_mean, ref_bn.running_mean), ("running_var", bn.running_var, ref_bn.running_var)):
        assert bool(torch.isfinite(got).all()), f"{dt}: edge encoder {name} is not finite"
        scale = float(ref.abs().max())
        err = float((got - ref).abs().max())
        assert err <= 16 * u * scale, f"{dt}: edge encoder {name} is {err / scale / u:.2f} u of its scale from the fp32 step's"


# ---- module parity under bf16 autocast ------------------------------------------------------------------------------------
def _mp_core_ref64(qkm, ke, me, src, tgt, combo, H):
    """The graph part of one GATConvE layer in differentiable fp64 torch ops (tests/test_gpu_heads.py: mp_core_ref), on the
    device of its inputs."""
    N, D = qkm.size(0), qkm.size(1) // 3
    d = D // H
    dev, f = qkm.device, qkm.dtype
    Q, Kx, Mx = (qkm[:, i * D:(i + 1) * D].reshape(N, H, d) for i in range(3))
    s = (Q[src] * (Kx[tgt] + ke.reshape(-1, H, d)[combo])).sum(-1)
    smax = torch.full((N, H), float("-inf"), dtype=f, device=dev).scatter_reduce(0, src[:, None].expand(-1, H), s.detach(), "amax")
    e = torch.exp(s - smax[src])
    alpha = e / (torch.zeros(N, H, dtype=f, device=dev).index_add(0, src, e)[src] + 1e-16)
    outdeg = torch.bincount(src, minlength=N).to(f)
    msg = (alpha * outdeg[src][:, None])[:, :, None] * (Mx[src] + me.reshape(-1, H, d)[combo])
    return torch.zeros(N, H, d, dtype=f, device=dev).index_add(0, tgt, msg).reshape(N, D), alpha


class _Fp64Core:
    """Stands in for training._MPCore: the same operands in, aggr in their dtype out, computed in fp64 and rounded once.
    What an exact core would give: the module around it runs exactly as with the CUDA core."""

    @staticmethod
    def apply(qkm, ke, me, prep, shape_args, want_alpha):
        N, E, D, H = shape_args[:4]
        Ep = E + N
        src, tgt, combo = (prep.array(k)[:Ep].long() for k in ("src", "tgt", "combo"))
        with torch.autocast("cuda", enabled=False):
            aggr, alpha = _mp_core_ref64(qkm.double(), ke.double(), me.double(), src, tgt, combo, H)
        return aggr.to(qkm.dtype), (alpha.float() if want_alpha else None)


def _module(fx, sd):
    c = fx["case"]
    mod = qagnn_b200.QAGNN_Message_Passing(None, c["k"], fx["n_ntype"], fx["n_etype"], c["D"], c["D"], c["D"], dropout=0.0)
    mod.load_state_dict(sd, strict=True)
    return mod.to(DEV).train()


def _step(fx, inp, sd, amp):
    mod = _module(fx, sd)
    H = inp["H"].to(DEV).requires_grad_(True)
    score = inp["node_score"].to(DEV).requires_grad_(True)
    with _autocast(amp):
        out = mod(H, (inp["edge_index"].to(DEV), inp["edge_type"].to(DEV)), inp["node_type"].to(DEV), score)
        loss = (out.float() * MG.train_loss_weights(fx["case"]).to(DEV)).sum()
    loss.backward()
    grads = {"H": H.grad, "node_score": score.grad}
    grads.update({k: p.grad for k, p in mod.named_parameters()})
    return out.detach().float(), float(loss.detach()), grads


@pytest.mark.parametrize("name", Hh.golden_names("train"))
def test_module_under_bf16_autocast_matches_an_fp64_graph_part(name, monkeypatch):
    """Every training golden under bf16 autocast, with the CUDA core and with the graph part in fp64 torch ops (what an exact
    core gives, rounded once).  Both run the same bf16 dense layers, so their difference is this path's precision alone; the
    bar is the difference bf16 autocast already makes to the same model (the fp64-core bf16 run against the fp32 run), plus one
    bf16 ulp (2^-8) of the tensor's scale: the graph part may not cost more precision than autocast does.  Measured on the
    training goldens on an H100, the path's difference is 0 to 0.4 of autocast's for the output and most gradients, and up to
    0.85 for the bias in front of the edge encoder's BatchNorm, whose gradient is mathematically zero (rounding noise in
    every run; judged on 1e-2 of the model's largest gradient, as tests/test_gpu_training.py does)."""
    fx = Hh.load_golden(name)
    inp, sd = Hh.regen_mp_inputs(fx)
    out, loss, grads = _step(fx, inp, sd, torch.bfloat16)
    f32_out, f32_loss, f32_grads = _step(fx, inp, sd, None)
    monkeypatch.setattr(TR, "_MPCore", _Fp64Core)
    ref_out, ref_loss, ref_grads = _step(fx, inp, sd, torch.bfloat16)
    monkeypatch.undo()
    ulp = 2.0 ** -8
    assert bool(torch.isfinite(out).all()) and math.isfinite(loss)
    oscale = float(ref_out.abs().max())
    err, auto = float((out - ref_out).abs().max()), float((ref_out - f32_out).abs().max())
    assert err <= auto + ulp * oscale, f"module output: {err:.3e} vs autocast's {auto:.3e}"
    assert abs(loss - ref_loss) <= abs(ref_loss - f32_loss) + ulp * abs(ref_loss), f"loss {loss} vs {ref_loss} (fp32 {f32_loss})"
    assert grads.keys() == ref_grads.keys() == f32_grads.keys()
    gmax = max(float(g.abs().max()) for g in ref_grads.values() if g is not None)
    for k, g in grads.items():
        assert g is not None and bool(torch.isfinite(g).all()), f"dL/d{k} is missing or not finite"
        scale = max(float(ref_grads[k].abs().max()), 1e-2 * gmax)
        err = float((g.float() - ref_grads[k].float()).abs().max())
        auto = float((ref_grads[k].float() - f32_grads[k].float()).abs().max())
        assert err <= auto + ulp * scale, f"dL/d{k}: max|err| {err:.3e}, autocast's {auto:.3e}, scale {scale:.3e}"


# ---- TrainStep under bf16 autocast -----------------------------------------------------------------------------------------
def _bn_buffers(dec):
    return {k: v.detach().clone() for k, v in dec.named_buffers() if "running" in k or "num_batches" in k}


def test_train_step_bf16_matches_eager_bf16_training(split):
    """The comparisons of tests/test_gpu_train_step.py (logits, pool_attn, loss, BatchNorm buffers, dL/dsent_vecs,
    dL/dnode_scores and every parameter gradient after one and after three micro-steps).  Replay and eager run the same
    kernels on the same bf16 values: the forward is deterministic, so logits and buffers agree to fp32 rounding.  In the
    backward, d_ke / d_me are fp32 atomic sums rounded to bf16 once: a sum near a rounding boundary may round to the other
    neighbour in one run, which moves the gradients it feeds by one bf16 ulp of that entry; gradients are therefore compared
    to 2^-7 of their scale (two bf16 ulps) plus the fp32 test's 1e-4."""
    K, M = split[3].max_batch_edges(2), split[3].max_graph_edges()
    dec = _split_decoder()
    _zero_dropout(dec)
    eager_dec, step_dec = copy.deepcopy(dec), copy.deepcopy(dec)
    batch, cap = _split_batch(split, [3, 9], K, 21)
    exact = _split_batch(split, [3, 9], None, 21)[1]
    step = TrainStep(step_dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=M,
                     autocast_dtype=torch.bfloat16)
    assert step.mode.startswith("two CUDA graphs")
    B = batch["concept_ids"].size(0)
    w = torch.randn(B, 1, device=DEV)
    es, en = _leaves(batch)
    ss, sn = _leaves(batch)

    def grad_close(got, ref, what, floor=0.0):
        scale = max(float(ref.abs().max()), floor, 1e-6)
        Hh.assert_close(got.float(), ref.float(), what, atol=(2.0 ** -7 + 1e-4) * scale, rtol=1e-4)

    def compare():
        grad_close(ss.grad, es.grad, "dL/dsent_vecs")
        grad_close(sn.grad, en.grad, "dL/dnode_scores")
        ref = {k: p.grad for k, p in eager_dec.named_parameters() if p.grad is not None}
        got = {k: p.grad for k, p in step_dec.named_parameters() if p.grad is not None}
        assert got.keys() == ref.keys() and len(ref) > 10
        gmax = max(float(g.abs().max()) for g in ref.values())
        for k in ref:
            grad_close(got[k], ref[k], f"dL/d{k}", floor=1e-2 * gmax)

    for it in range(3):
        with _autocast(torch.bfloat16):
            logits_e, attn_e = eager_dec(*_args(batch, es, en, exact))
        logits_s, attn_s = step(*_args(batch, ss, sn, cap))
        Hh.assert_close(logits_s.float(), logits_e.float(), f"step {it}: logits")
        Hh.assert_close(attn_s.float(), attn_e.float(), f"step {it}: pool_attn")
        loss_e, loss_s = (logits_e.float() * w).sum(), (logits_s.float() * w).sum()
        assert abs(float(loss_s.detach()) - float(loss_e.detach())) <= 1e-4 * (1 + abs(float(loss_e.detach())))
        loss_e.backward()
        loss_s.backward()
        got_b, ref_b = _bn_buffers(step_dec), _bn_buffers(eager_dec)
        for k in ref_b:
            if "num_batches" in k:
                assert int(got_b[k]) == int(ref_b[k]), f"step {it}: {k}"
            else:
                Hh.assert_close(got_b[k], ref_b[k], f"step {it}: {k}", atol=1e-5, rtol=1e-4)
        if it == 0:
            compare()
    compare()


def test_eager_bf16_training_step_does_not_synchronise(split):
    dec = _split_decoder(dropout=0.2)
    batch, adj = _split_batch(split, [4, 8], split[3].max_batch_edges(2) + 300, 2)
    dec.gnn.check_batch(adj, batch["node_type_ids"])  # index validation: once, eagerly
    dec.gnn.check_indices = False
    w = torch.randn(batch["concept_ids"].size(0), 1, device=DEV)

    def step():
        sv, ns = _leaves(batch)
        with _autocast(torch.bfloat16):
            logits, _ = dec(*_args(batch, sv, ns, adj))
            loss = (logits.float() * w).sum()
        loss.backward()
        return sv

    step()  # first step: builds the constant one-hot table
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sv = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert sv.grad is not None and bool(torch.isfinite(sv.grad).all())
    assert all(p.grad is None or bool(torch.isfinite(p.grad).all()) for p in dec.parameters())


def test_bf16_train_step_optimiser_step_without_grad_scaler(split):
    """The loop body of qagnn.py:252-278 under bf16: no GradScaler, loss.backward() and an optimiser step; the eval path
    then sees the new weights and running statistics."""
    dec = _split_decoder(dropout=0.1)
    batch, cap = _split_batch(split, [5, 6], split[3].max_batch_edges(2), 5)
    exact = _split_batch(split, [5, 6], None, 5)[1]
    with torch.no_grad():
        before = dec.eval()(*_args(batch, batch["sent_vecs"], batch["node_scores"], exact))[0].clone()
    dec.train()
    step = TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=split[3].max_graph_edges(),
                     autocast_dtype=torch.bfloat16)
    opt = torch.optim.SGD([p for p in dec.parameters() if p.requires_grad], lr=0.05)
    sv, ns = _leaves(batch)
    logits, _ = step(*_args(batch, sv, ns, cap))
    loss = torch.nn.functional.cross_entropy(logits.float().view(2, 5), torch.tensor([1, 3], device=DEV))
    loss.backward()
    opt.step()
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(sv.grad).all())
    assert all(p.grad is None or bool(torch.isfinite(p.grad).all()) for p in dec.parameters())
    with torch.no_grad():
        after = dec.eval()(*_args(batch, batch["sent_vecs"], batch["node_scores"], exact))[0]
    assert bool(torch.isfinite(after).all()) and not torch.allclose(before, after, atol=1e-5)
