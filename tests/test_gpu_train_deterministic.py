"""Bit-reproducible training under torch.use_deterministic_algorithms(True).

  * the message-passing core's deterministic backward (qagnn_mp_core_backward_det) at every (head count, chunk count,
    dtype) it dispatches on: two runs give the same bits, d_qkm is the default backward's bit for bit, d_ke / d_me are
    within the training bar of an fp64 evaluation, and a 16-bit call is the fp32 call on the widened operands, rounded;
  * combo layouts that exercise the cross-run combine: one combo over hundreds of runs, combos ending and starting on a run
    boundary, a whole combo between two crossing ones, E' not a multiple of the run length, combos without edges, the
    no-edge and single-node graphs, a cfg2-size batch;
  * a batch packed at an edge capacity trains to the exact batch's gradients bit for bit;
  * the QAGNN decoder: two eager micro-steps give the same logits, loss, gradients and BatchNorm buffers bit for bit in fp32,
    fp16 autocast with GradScaler and bf16 autocast, with and without dropout; the training goldens stay within their bars;
  * TrainStep built under the flag replays to the same gradients bit for bit, and refuses a call after the flag changed;
  * an eager deterministic micro-step without host synchronisation.
Needs a GPU: run with -m gpu."""
import contextlib
import copy

import numpy as np
import pytest
import torch

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200 import training as TR
from qagnn_b200.modeling_qagnn import GraphPrep
from qagnn_b200.pipeline import TrainStep
from tests import helpers as Hh
from tests import test_gpu_training as TG

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R = 4, 38
NC = R * T * T + T
RUN = 64  # positions per run of the edge-table kernel
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["fp32", "fp16", "bf16"]


@contextlib.contextmanager
def _flag(on):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.fixture
def deterministic(monkeypatch):
    """torch.use_deterministic_algorithms(True) for one test; cuBLAS needs a fixed workspace for it, read at call time."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    with _flag(True):
        yield


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    bad = int((_bits(a) != _bits(b)).sum())
    assert bad == 0, f"{what}: {bad} of {a.numel()} elements differ"


def _grad_close(got, ref, what, floor=0.0):
    scale = max(float(ref.abs().max()), floor, 1e-6)  # the training bar of test_gpu_training.py
    Hh.assert_close(got, ref, what, atol=1e-4 * scale, rtol=1e-4)


# ---- the core ------------------------------------------------------------------------------------------------------------
def _core_grads(prep, N, D, H, qkm, ke, me, G, det):
    leaves = [t.detach().clone().requires_grad_(True) for t in (qkm, ke, me)]
    with _flag(det):
        aggr, _ = TR._MPCore.apply(*leaves, prep, (N, prep.E, D, H, T, R), False)
        return torch.autograd.grad(aggr, leaves, G)


def _operands(N, D, H, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkm = torch.randn(N, 3 * D, generator=g, device=DEV)
    qkm[:, :D] /= (D // H) ** 0.5  # Q / sqrt(d) as the layer scales it
    ke, me = torch.randn(NC, D, generator=g, device=DEV), torch.randn(NC, D, generator=g, device=DEV)
    return qkm, ke, me, torch.randn(N, D, generator=g, device=DEV)


def _fp64_tables(ei, et, nt, N, D, H, qkm, ke, me, G):
    """d_ke, d_me of the core's forward evaluated per edge in fp64 (self loops appended, combo as graph prep numbers it)."""
    ei, et, nt = ei.to(DEV), et.to(DEV), nt.to(DEV)
    loop = torch.arange(N, device=DEV)
    s, t = torch.cat([ei[0], loop]), torch.cat([ei[1], loop])
    cb = torch.cat([(et * T + nt[ei[0]]) * T + nt[ei[1]], R * T * T + nt])
    q64, k64, m64 = (x.detach().double().requires_grad_(True) for x in (qkm, ke, me))
    d = D // H
    q, kx, mx = q64[:, :D], q64[:, D:2 * D], q64[:, 2 * D:]
    logit = (q[s] * (kx[t] + k64[cb])).view(-1, H, d).sum(-1)
    top = torch.full((N, H), -torch.inf, dtype=torch.float64, device=DEV).scatter_reduce(
        0, s[:, None].expand(-1, H), logit.detach(), "amax")
    ex = torch.exp(logit - top[s])
    den = torch.zeros(N, H, dtype=torch.float64, device=DEV).index_add(0, s, ex)
    deg = torch.bincount(s, minlength=N).double()
    a = ex / den[s] * deg[s][:, None]
    msg = (mx[s] + m64[cb]).view(-1, H, d) * a[:, :, None]
    aggr = torch.zeros(N, H, d, dtype=torch.float64, device=DEV).index_add(0, t, msg).view(N, D)
    return torch.autograd.grad(aggr, [k64, m64], G.double())


def _check_core(prep, ei, et, nt, D, H, dt, seed, fp64=True):
    """Everything the deterministic backward promises on one prep; returns the combo counts."""
    N = nt.numel()
    qkm, ke, me, G = _operands(N, D, H, seed)
    lo = [x.to(dt) for x in (qkm, ke, me, G)]
    first = _core_grads(prep, N, D, H, *lo, det=True)
    second = _core_grads(prep, N, D, H, *lo, det=True)
    for name, a, b in zip(("d_qkm", "d_ke", "d_me"), first, second):
        assert a.dtype == dt
        _same_bits(a, b, f"{dt} H={H} D={D}: {name}, two deterministic runs")
    default = _core_grads(prep, N, D, H, *lo, det=False)
    _same_bits(first[0], default[0], f"{dt} H={H} D={D}: d_qkm against the default backward")
    count = prep.combo_count()
    empty = count == 0
    for name, g in zip(("d_ke", "d_me"), first[1:]):
        assert bool((g[empty] == 0).all()) and not bool(torch.signbit(g[empty]).any()), f"{name}: rows without edges"
    if dt == torch.float32:
        if fp64:
            ref_ke, ref_me = _fp64_tables(ei, et, nt, N, D, H, qkm, ke, me, G)
            _grad_close(first[1], ref_ke, f"H={H} D={D}: d_ke against fp64")
            _grad_close(first[2], ref_me, f"H={H} D={D}: d_me against fp64")
    else:
        wide = _core_grads(prep, N, D, H, *(x.float() for x in lo), det=True)
        for name, a, b in zip(("d_qkm", "d_ke", "d_me"), first, wide):
            _same_bits(a, b.to(dt), f"{dt} H={H} D={D}: {name} against the fp32 deterministic call, rounded")
    return count


# D per head count giving CH = ceil(D / 128) = 1, 2, 4, 8 (as test_gpu_train_bf16.py)
SHAPES = [(1, 36), (1, 200), (1, 500), (1, 1020), (2, 40), (2, 200), (2, 388), (2, 1000), (4, 100), (4, 232), (4, 400),
          (4, 1020), (8, 64), (8, 200), (8, 488), (8, 1000), (16, 64), (16, 208), (16, 400), (16, 1024)]


@pytest.fixture(scope="module")
def random_graph():
    g = torch.Generator().manual_seed(0)
    N, E = 300, 1200
    ei, et, nt = torch.randint(0, N, (2, E), generator=g), torch.randint(0, R, (E,), generator=g), torch.randint(0, T, (N,), generator=g)
    return ei, et, nt, GraphPrep(ei.to(DEV), et.to(DEV), nt.to(DEV), T, R)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("H,D", SHAPES)
def test_deterministic_core_every_instantiation(random_graph, H, D, dt):
    assert (D + 127) // 128 in (1, 2, 4, 8)
    ei, et, nt, prep = random_graph
    _check_core(prep, ei, et, nt, D, H, dt, seed=H * 4096 + D)


def _layout(case):
    """(edge_index, edge_type, node_type) of a combo layout; node types are all 0, so combo = 16 * edge type."""
    g = torch.Generator().manual_seed(7)
    if case == "one_combo_hundreds_of_runs":  # 20000 positions of combo 0, 3000 self loops in one more combo
        N, sizes = 3000, {0: 20000}
    elif case == "run_boundaries":
        # combo 0: [0, 128) ends on a boundary; combo 16: [128, 228) starts on it and crosses into run 3; combo 32:
        # [228, 248) lies inside run 3; combo 48: [248, 400) crosses out of it; combo 80 and the self loops: E' = 487
        N, sizes = 50, {0: 128, 1: 100, 2: 20, 3: 152, 5: 37}
    elif case == "no_edges":
        inp, _ = Hh.regen_mp_inputs(Hh.load_golden("no_edges"))
        return inp["edge_index"], inp["edge_type"], inp["node_type"].reshape(-1)
    elif case == "single_node":
        return torch.zeros(2, 0, dtype=torch.long), torch.zeros(0, dtype=torch.long), torch.tensor([2])
    elif case == "single_node_self_edge":
        return torch.zeros(2, 1, dtype=torch.long), torch.tensor([7]), torch.tensor([2])
    elif case == "cfg2":  # 320 graphs x 200 nodes x 1000 edges: E' = 384 k
        inp = O.synth_graph_batch(320, 200, 1000, 2, R, seed=3)
        return inp["edge_index"], inp["edge_type"], inp["node_type"].reshape(-1)
    et = torch.cat([torch.full((n,), r, dtype=torch.long) for r, n in sizes.items()])
    return torch.randint(0, N, (2, et.numel()), generator=g), et, torch.zeros(N, dtype=torch.long)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", ["one_combo_hundreds_of_runs", "run_boundaries", "no_edges", "single_node",
                                  "single_node_self_edge", "cfg2"])
def test_deterministic_core_combo_layouts(case, dt):
    ei, et, nt = _layout(case)
    prep = GraphPrep(ei.to(DEV), et.to(DEV), nt.to(DEV), T, R)
    for H, D in ((4, 64), (2, 200)):
        count = _check_core(prep, ei, et, nt, D, H, dt, seed=H + D)
        c = count.cpu()
        off = torch.cumsum(c, 0) - c
        Ep = int(c.sum())
        assert Ep == ei.size(1) + nt.numel()
        if case == "one_combo_hundreds_of_runs":
            assert int(c[0]) // RUN >= 300
        elif case == "run_boundaries":
            assert Ep % RUN != 0
            assert int(off[16]) == 2 * RUN and int(off[16] + c[16]) > 3 * RUN
            assert 3 * RUN < int(off[32]) and int(off[32] + c[32]) < 4 * RUN and int(off[48] + c[48]) > 4 * RUN


def _split(tmp_path_factory, n_questions, seed):
    path = str(tmp_path_factory.mktemp("split") / "train.graph.adj.pk")
    Dt.synth_adj_pickle(path, n_questions * 5, seed=seed)
    _, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, 200, 5)
    return ntypes, scores, lens, flat


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    return _split(tmp_path_factory, 24, 31)


# ---- edge capacity -------------------------------------------------------------------------------------------------------
def test_training_at_capacity_is_bitwise_the_exact_batch(split, deterministic):
    ntypes, scores, lens, flat = split
    D, qs = 200, np.array([2, 4, 6, 8])
    mod0 = qagnn_b200.QAGNN_Message_Passing(None, 3, T, R, D, D, D, dropout=0.0)
    mod0.load_state_dict(O.random_state_dict(3, D, T, R, "prod", seed=9))
    mod0 = mod0.to(DEV)
    B = len(qs) * 5
    g = torch.Generator().manual_seed(1)
    H0, w = torch.randn(B, 200, D, generator=g).to(DEV), torch.randn(B, 200, D, generator=g).to(DEV)
    nt, ns = ntypes[qs].reshape(B, 200).to(DEV), scores[qs].reshape(B, 200, 1).to(DEV)

    def run(capacity):
        adj = flat.pack(qs, pin=False, edge_capacity=capacity).to(DEV)
        mod = copy.deepcopy(mod0).train()
        H = H0.clone().requires_grad_(True)
        out = mod(H, adj, nt, ns)
        (out * w).sum().backward()
        grads = {n: p.grad for n, p in mod.named_parameters() if p.grad is not None}
        grads["H"] = H.grad
        return out.detach(), grads, adj.n_edges

    out_e, g_e, E = run(None)
    out_c, g_c, _ = run(E + 301)
    _same_bits(out_c, out_e, "out")
    assert g_e.keys() == g_c.keys() and len(g_e) > 10
    for name in g_e:
        _same_bits(g_c[name], g_e[name], f"dL/d{name}")


# ---- the decoder ---------------------------------------------------------------------------------------------------------
def _batch(split, qs, capacity, seed):
    ntypes, scores, lens, flat = split
    adj = flat.pack(np.asarray(qs), pin=False, edge_capacity=capacity).to(DEV)
    B = len(qs) * 5
    g = torch.Generator().manual_seed(seed)
    cid = torch.randint(1, 301, (B, 200), generator=g)
    cid[:, 0] = 0
    batch = {"sent_vecs": torch.randn(B, 48, generator=g), "concept_ids": cid, "node_type_ids": ntypes[qs].reshape(B, 200),
             "node_scores": scores[qs].reshape(B, 200, 1), "adj_lengths": lens[qs].reshape(B)}
    return {k: v.to(DEV) for k, v in batch.items()}, adj


def _decoder(dropout):
    torch.manual_seed(8)
    dec = qagnn_b200.QAGNN(None, 2, T, R, 48, 300, 64, 32, 2, 64, 1, dropout, dropout, dropout)
    dec.gnn.load_state_dict(O.random_state_dict(2, 64, T, R, "prod", seed=8))
    return dec.to(DEV).train()


def _args(batch, sv, ns, adj):
    return sv, batch["concept_ids"], batch["node_type_ids"], ns, batch["adj_lengths"], adj


def _leaves(batch):
    return batch["sent_vecs"].clone().requires_grad_(True), batch["node_scores"].clone().requires_grad_(True)


def _state(dec, sv, ns):
    out = {f"grad {k}": p.grad for k, p in dec.named_parameters() if p.grad is not None}
    out.update({f"buffer {k}": v for k, v in dec.named_buffers()})
    out["dL/dsent_vecs"], out["dL/dnode_scores"] = sv.grad, ns.grad
    return {k: v.detach().clone() for k, v in out.items()}


def _micro_step(dec0, batch, adj, autocast, rng):
    dec = copy.deepcopy(dec0)
    torch.cuda.set_rng_state(rng, DEV)
    sv, ns = _leaves(batch)
    labels = torch.arange(batch["concept_ids"].size(0) // 5, device=DEV) % 5
    ctx = torch.autocast("cuda", dtype=autocast) if autocast else contextlib.nullcontext()
    with ctx:
        logits, _ = dec(*_args(batch, sv, ns, adj))
    loss = torch.nn.functional.cross_entropy(logits.float().view(-1, 5), labels)
    if autocast == torch.float16:
        torch.amp.GradScaler("cuda").scale(loss).backward()
    else:
        loss.backward()
    out = _state(dec, sv, ns)
    out["logits"], out["loss"] = logits.detach().clone(), loss.detach().clone()
    return out


@pytest.mark.parametrize("dropout", [0.0, 0.3])
@pytest.mark.parametrize("autocast", [None, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
def test_two_decoder_micro_steps_are_bitwise_equal(split, deterministic, autocast, dropout):
    dec = _decoder(dropout)
    batch, adj = _batch(split, [1, 5, 9, 13], split[3].max_batch_edges(4) + 100, 2)
    rng = torch.cuda.get_rng_state(DEV)
    a = _micro_step(dec, batch, adj, autocast, rng)
    b = _micro_step(dec, batch, adj, autocast, rng)
    assert a.keys() == b.keys() and sum(k.startswith("grad ") for k in a) > 10
    assert a["dL/dnode_scores"] is not None
    for k in a:
        _same_bits(a[k], b[k], k)


@pytest.mark.parametrize("name", Hh.golden_names("train"))
def test_training_goldens_under_the_flag(name, deterministic):
    TG.test_training_forward_and_gradients_match_reference(name)


def test_decoder_golden_under_the_flag(deterministic):
    TG.test_whole_decoder_training_step_matches_reference()


# ---- TrainStep -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dropout", [0.0, 0.2])
def test_train_step_replays_bitwise_and_refuses_a_changed_flag(split, deterministic, dropout):
    dec = _decoder(dropout)
    K, M = split[3].max_batch_edges(2), split[3].max_graph_edges()
    batch, cap = _batch(split, [3, 11], K, 4)
    eager_dec = copy.deepcopy(dec)
    step_dec = copy.deepcopy(dec)
    step = TrainStep(step_dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=M)
    assert step.deterministic and step.mode.startswith("two CUDA graphs")
    params = [p for p in step_dec.parameters() if p.requires_grad]
    w = torch.randn(10, 1, device=DEV)
    rng = torch.cuda.get_rng_state(DEV)
    runs = []
    for _ in range(2):
        for p in params:
            p.grad = None
        torch.cuda.set_rng_state(rng, DEV)
        sv, ns = _leaves(batch)
        logits, _ = step(*_args(batch, sv, ns, cap))
        (logits * w).sum().backward()
        runs.append(_state(step_dec, sv, ns))
    for k in runs[0]:
        if k.startswith("buffer "):
            continue  # the second replay advances the running statistics again
        _same_bits(runs[0][k], runs[1][k], f"two replays: {k}")
    if dropout > 0:  # a replay's masks come from the graph's own RNG offsets: eager is compared without dropout
        return
    torch.cuda.set_rng_state(rng, DEV)
    sv, ns = _leaves(batch)
    (eager_dec(*_args(batch, sv, ns, cap))[0] * w).sum().backward()
    ref = _state(eager_dec, sv, ns)
    gmax = max(float(v.abs().max()) for k, v in ref.items() if k.startswith("grad "))
    bitwise = []
    for k in ref:
        if k.startswith("buffer "):
            continue
        _grad_close(runs[0][k], ref[k], f"replay vs eager: {k}", floor=1e-2 * gmax if k.startswith("grad ") else 0.0)
        bitwise.append(torch.equal(runs[0][k], ref[k]))
    print(f"\nTrainStep replay vs eager under the flag: {sum(bitwise)} of {len(bitwise)} gradients bitwise equal")
    with _flag(False):
        with pytest.raises(RuntimeError, match="use_deterministic_algorithms"):
            step(*_args(batch, batch["sent_vecs"], batch["node_scores"], cap))


def test_train_step_built_without_the_flag_refuses_it(split):
    dec = _decoder(0.0)
    K, M = split[3].max_batch_edges(2), split[3].max_graph_edges()
    batch, cap = _batch(split, [0, 7], K, 6)
    with _flag(False):
        step = TrainStep(dec, *_args(batch, batch["sent_vecs"], batch["node_scores"], cap), max_edges=M)
    assert not step.deterministic
    with _flag(True):
        with pytest.raises(RuntimeError, match="Build a new TrainStep"):
            step(*_args(batch, batch["sent_vecs"], batch["node_scores"], cap))


# ---- no host synchronisation ---------------------------------------------------------------------------------------------
def test_eager_deterministic_step_does_not_synchronise(split, deterministic):
    dec = _decoder(0.2)
    batch, adj = _batch(split, [2, 6], split[3].max_batch_edges(2) + 50, 3)
    dec.gnn.check_batch(adj, batch["node_type_ids"])  # index validation: once, eagerly
    dec.gnn.check_indices = False
    w = torch.randn(10, 1, device=DEV)

    def step():
        sv, ns = _leaves(batch)
        (dec(*_args(batch, sv, ns, adj))[0] * w).sum().backward()
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
