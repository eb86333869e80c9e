"""Training from a split held on the GPU: pipeline.SplitTrainStep against eager training on DeviceSplit.batch, i.e.
`decoder(sent_vecs, *split.batch(qids, K))`, F.cross_entropy under the same autocast and `(loss * w).backward()` with
autograd's accumulation.  Under torch.use_deterministic_algorithms(True) with dropout 0 the comparison is bit for bit over two
optimiser batches (losses, logits, dL/dsent_vecs, every .grad after every micro-step, BatchNorm buffers, parameters after
Adam); in the default mode it is within the training bars.  Also: a frozen encoder, .grad that is not None, one capture
for every micro-batch, dropout masks, the state the capture leaves, the refusals, and SplitEvalStep after training.
Needs a GPU: run with -m gpu."""
import contextlib
import copy
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import data as Dt
from qagnn_b200.pipeline import SplitEvalStep, SplitTrainStep
from tests import helpers as Hh

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T, R, N, NC = 4, 38, 200, 5
N_CONCEPT, SENT_DIM, D = 300, 48, 64
DTYPES = [None, torch.bfloat16, torch.float16]
DT_IDS = ["fp32", "bf16", "fp16"]


class Split:
    def __init__(self, n_questions, seed, labels=True):
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "s.graph.adj.pk")
            Dt.synth_adj_pickle(path, n_questions * NC, seed=seed)
            cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N, NC)
        self.flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr),
                                    NC, N)
        cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)  # inside the decoder's table; the context node keeps id 0
        self.labels = torch.from_numpy(np.random.default_rng(seed).integers(0, NC, n_questions))
        self.host = (cids, ntypes, scores, lens)
        self.dev = Dt.DeviceSplit(self.flat, *self.host, DEV, T, R, labels=self.labels if labels else None)
        self.Q = n_questions

    def edges(self, q):
        gids = (np.asarray(q)[:, None] * NC + np.arange(NC)).reshape(-1)
        return np.diff(self.flat.graph_ptr)[gids]


@pytest.fixture(scope="module")
def s48():
    return Split(48, seed=51)


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
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # cuBLAS reads it at call time
    with _flag(True):
        yield


def _decoder(dropout=0.0, seed=8):
    torch.manual_seed(seed)
    dec = qagnn_b200.QAGNN(None, 2, T, R, SENT_DIM, N_CONCEPT, D, 32, 2, D, 1, dropout, dropout, dropout)
    dec.gnn.load_state_dict(O.random_state_dict(2, D, T, R, "prod", seed=seed))
    for m in dec.modules():  # the pooler's attention dropout included, which the constructor does not set
        if isinstance(m, torch.nn.Dropout):
            m.p = dropout
    return dec.to(DEV).train()


def _autocast(dt):
    return torch.autocast("cuda", dtype=dt, cache_enabled=False) if dt is not None else torch.autocast("cuda", enabled=False)


def _eager(dec, s, q, sv, K, dt):
    """The reference micro-step forward: (loss, logits, pool_attn)."""
    with _autocast(dt):
        logits, attn = dec(sv, *s.dev.batch(q, K))
        loss = F.cross_entropy(logits.view(-1, NC), s.dev.labels[torch.from_numpy(np.asarray(q)).to(DEV)])
    return loss, logits, attn


def _bn(dec):
    return {k: v.detach().clone() for k, v in dec.named_buffers() if "running" in k or "num_batches" in k}


def _sv(bs, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(bs * NC, SENT_DIM, device=DEV, generator=g)


def _plan(s, mbs, seed, n_opt=2, n_micro=3):
    """n_opt optimiser batches of n_micro micro-batches of mbs shuffled question ids."""
    order = np.random.default_rng(seed).permutation(s.Q)[:n_opt * n_micro * mbs]
    return [[order[(o * n_micro + m) * mbs:(o * n_micro + m + 1) * mbs] for m in range(n_micro)] for o in range(n_opt)]


def _train(dec, s, plan, dt, K, M, use_step, frozen=False, reset=None):
    """Runs the optimiser batches of `plan` (qagnn.py:249-278 with Adam and clip_grad_norm_) through SplitTrainStep or
    eagerly; returns every micro-step's and optimiser step's results.  `reset(o, params)` replaces optimizer.zero_grad()."""
    params = [p for p in dec.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-3)
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    mbs = len(plan[0][0])
    step = SplitTrainStep(dec, s.dev, mbs, edge_capacity=K, max_edges=M, autocast_dtype=dt) if use_step else None
    rec = []
    for o, micro in enumerate(plan):
        if reset is None:
            opt.zero_grad()
        else:
            reset(o, params)
        total = sum(len(q) for q in micro)
        for m, q in enumerate(micro):
            sv = _sv(mbs, 100 * o + m).requires_grad_(not frozen)
            if use_step:
                loss, logits = step(q, sv), step.logits
            else:
                loss, logits, _ = _eager(dec, s, q, sv, K, dt)
            r = {"loss": loss.detach().clone(), "logits": logits.detach().clone()}
            w = loss * len(q) / total
            (scaler.scale(w) if scaler is not None else w).backward()
            if not frozen:
                r["dL/dsent_vecs"] = sv.grad.clone()
            r.update({f"grad {k}": p.grad.clone() for k, p in dec.named_parameters() if p.grad is not None})
            rec.append(r)
        if scaler is not None:
            scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        r = {f"param {k}": p.detach().clone() for k, p in dec.named_parameters()}
        r.update({f"buffer {k}": v for k, v in _bn(dec).items()})
        rec.append(r)
    return rec, step


def _same(got, ref, bitwise):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys(), (i, sorted(set(g) ^ set(r)))
        assert sum(k.startswith("grad ") for k in r) > 10 or any(k.startswith("param ") for k in r)
        gmax = max([float(v.abs().max()) for k, v in r.items() if k.startswith("grad ")] or [0.0])
        for k in r:
            what = f"record {i}: {k}"
            if bitwise or "num_batches" in k:
                assert g[k].dtype == r[k].dtype and torch.equal(g[k], r[k]), what
            elif k.startswith("param "):
                # Adam's first steps move a parameter by about lr whatever its gradient's size: a gradient near zero that
                # the two routes' summation orders round to opposite signs moves it by up to 2 lr apart
                Hh.assert_close(g[k], r[k], what, atol=1e-4 * float(r[k].abs().max()) + 2e-3, rtol=1e-4)
            else:
                floor = 1e-2 * gmax if k.startswith("grad ") else 0.0
                scale = max(float(r[k].abs().max()), floor, 1e-6)  # the training bar of test_gpu_training.py
                Hh.assert_close(g[k].float(), r[k].float(), what, atol=1e-4 * scale, rtol=1e-4)


def _both(s, mbs, dt, seed, n_opt=2, **kw):
    dec = _decoder()
    plan = _plan(s, mbs, seed, n_opt)
    K, M = s.flat.max_batch_edges(mbs), s.flat.max_graph_edges()
    ref, _ = _train(copy.deepcopy(dec), s, plan, dt, K, M, False, **kw)
    got, step = _train(copy.deepcopy(dec), s, plan, dt, K, M, True, **kw)
    assert step.captures == 1 and step.mode.startswith("two CUDA graphs")
    return got, ref


@pytest.mark.parametrize("mbs", [2, 8])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_two_optimiser_batches_equal_eager_bit_for_bit(s48, deterministic, dt, mbs):
    got, ref = _both(s48, mbs, dt, seed=mbs)
    _same(got, ref, bitwise=True)


@pytest.mark.parametrize("mbs", [2, 8])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_an_optimiser_batch_equals_eager_in_the_default_mode(s48, dt, mbs):
    # one optimiser batch: Adam moves a parameter whose gradient the two summation orders round differently by up to 2 lr,
    # and the next batch's forward carries that past the training bars
    got, ref = _both(s48, mbs, dt, seed=10 + mbs, n_opt=1)
    _same(got, ref, bitwise=False)


@pytest.mark.parametrize("dt", [None, torch.float16], ids=["fp32", "fp16"])
def test_a_frozen_encoder_still_accumulates_the_decoders_gradients(s48, deterministic, dt):
    got, ref = _both(s48, 2, dt, seed=3, frozen=True)
    assert all("dL/dsent_vecs" not in r for r in got)
    _same(got, ref, bitwise=True)


def test_grad_that_is_not_none_is_continued(s48, deterministic):
    def reset(o, params):
        if o == 0:  # user-assigned gradients
            g = torch.Generator(device=DEV).manual_seed(5)
            for i, p in enumerate(params):
                p.grad = torch.randn(p.shape, device=DEV, generator=g) if i % 2 else None
        else:  # zero_grad(set_to_none=False)
            for p in params:
                if p.grad is not None:
                    p.grad.zero_()

    got, ref = _both(s48, 2, None, seed=4, reset=reset)
    _same(got, ref, bitwise=True)


def test_hooks_on_decoder_parameters_do_not_fire_and_grad_is_the_steps_buffer(s48):
    dec = _decoder()
    K, M = s48.flat.max_batch_edges(2), s48.flat.max_graph_edges()
    step = SplitTrainStep(dec, s48.dev, 2, edge_capacity=K, max_edges=M)
    step([0, 1], _sv(2, 0)).backward()  # captures: the warm-up runs autograd.grad, which calls tensor hooks
    fired = []
    p0 = dec.svec2nvec.weight
    p0.register_hook(lambda g: fired.append(g))
    step([4, 5], _sv(2, 2)).backward()
    buf = p0.grad
    step([2, 3], _sv(2, 1)).backward()
    assert p0.grad is buf and not fired


def test_micro_batches_of_different_edge_counts_replay_one_capture(s48, deterministic):
    mbs = 3
    tops = np.argsort([-int(s48.edges([q]).sum()) for q in range(s48.Q)])
    biggest = int(np.argmax([s48.edges([q]).max() for q in range(s48.Q)]))
    qsets = [tops[:mbs], [0, 1, 2], [biggest, 5, 9], [7, 30, 41], tops[-mbs:]]
    K, M = int(s48.edges(tops[:mbs]).sum()), s48.flat.max_graph_edges()
    assert len({int(s48.edges(q).sum()) for q in qsets}) == len(qsets) and int(s48.edges([biggest]).max()) == M
    dec = _decoder()
    eager_dec, step_dec = copy.deepcopy(dec), copy.deepcopy(dec)
    step = SplitTrainStep(step_dec, s48.dev, mbs, edge_capacity=K, max_edges=M)
    for i, q in enumerate(qsets):
        sv_e, sv_s = _sv(mbs, i).requires_grad_(True), _sv(mbs, i).requires_grad_(True)
        loss_e, logits_e, attn_e = _eager(eager_dec, s48, q, sv_e, K, None)
        loss_s = step(q, sv_s)
        assert torch.equal(loss_s, loss_e) and torch.equal(step.logits, logits_e) and torch.equal(step.pool_attn, attn_e), i
        loss_e.backward()
        loss_s.backward()
        assert torch.equal(sv_s.grad, sv_e.grad), i
    assert step.captures == 1
    for (k, p), pe in zip(step_dec.named_parameters(), eager_dec.parameters()):
        assert (p.grad is None) == (pe.grad is None) and (p.grad is None or torch.equal(p.grad, pe.grad)), k
    for k, v in _bn(eager_dec).items():
        assert torch.equal(_bn(step_dec)[k], v), k


def test_dropout_draws_a_new_mask_on_every_replay_and_the_same_from_the_same_rng_state(s48, deterministic):
    dec = _decoder(dropout=0.2)
    K, M = s48.flat.max_batch_edges(2), s48.flat.max_graph_edges()
    step = SplitTrainStep(dec, s48.dev, 2, edge_capacity=K, max_edges=M)
    q, sv = [4, 9], _sv(2, 7).requires_grad_(True)
    step(q, sv)  # captures
    rng = torch.cuda.get_rng_state(DEV)
    runs = []
    for again in (True, True, False):
        if again:
            torch.cuda.set_rng_state(rng, DEV)
        sv.grad = None
        loss = step(q, sv)
        runs.append((loss.detach().clone(), step.logits.clone(), step.pool_attn.clone()))
        loss.backward()
        runs[-1] += (sv.grad.clone(),)
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    assert not torch.equal(runs[1][1], runs[2][1]) and not torch.equal(runs[1][2], runs[2][2]), "a replay reused the masks"


def test_construction_and_capture_leave_the_model_state_as_it_was(s48):
    dec = _decoder(dropout=0.3)
    params = [p for p in dec.parameters() if p.requires_grad]
    for i, p in enumerate(params):
        if i % 3 == 0:
            p.grad = torch.full_like(p, 0.25 * i)
    grads = {k: None if v.grad is None else v.grad.clone() for k, v in dec.named_parameters()}
    buffers = _bn(dec)
    one = copy.deepcopy(dec)
    _eager(one, s48, [1, 7], _sv(2, 0), s48.flat.max_batch_edges(2), None)  # what one forward does to the buffers
    torch.cuda.manual_seed(123)
    rng = torch.cuda.get_rng_state()
    K, M = s48.flat.max_batch_edges(2), s48.flat.max_graph_edges()
    step = SplitTrainStep(dec, s48.dev, 2, edge_capacity=K, max_edges=M)
    assert torch.equal(torch.cuda.get_rng_state(), rng) and step.captures == 0
    step([1, 7], _sv(2, 0))  # capture (warm-up included) + one replay, no backward
    for k, v in dec.named_parameters():
        assert (v.grad is None) == (grads[k] is None) and (v.grad is None or torch.equal(v.grad, grads[k])), k
    after_one, ref = _bn(dec), _bn(one)
    for k, v in buffers.items():  # the replay's forward only, not the warm-up's
        if "num_batches" in k:
            assert int(after_one[k]) == int(ref[k]) > int(v), k
    rng_after = torch.cuda.get_rng_state()
    torch.cuda.set_rng_state(rng)
    step([1, 7], _sv(2, 0))
    assert torch.equal(torch.cuda.get_rng_state(), rng_after), "the capture advanced the RNG beyond one replay"


def test_refusals(s48):
    K, M = s48.flat.max_batch_edges(2), s48.flat.max_graph_edges()
    dec = _decoder()
    with pytest.raises(ValueError, match="train"):
        SplitTrainStep(copy.deepcopy(dec).eval(), s48.dev, 2, edge_capacity=K, max_edges=M)
    with pytest.raises(ValueError, match="labels"):
        SplitTrainStep(dec, Split(6, seed=52, labels=False).dev, 2, edge_capacity=K, max_edges=M)
    with pytest.raises(ValueError, match="autocast_dtype"):
        SplitTrainStep(dec, s48.dev, 2, edge_capacity=K, max_edges=M, autocast_dtype=torch.float64)
    with pytest.raises(ValueError, match="max_edges"):
        SplitTrainStep(dec, s48.dev, 2, edge_capacity=K, max_edges=M - 1)
    step = SplitTrainStep(dec, s48.dev, 2, edge_capacity=K, max_edges=M)
    with pytest.raises(ValueError, match="sent_vecs"):
        step([0, 1], _sv(3, 0))
    assert step.captures == 0
    dec.eval()
    with pytest.raises(RuntimeError, match="train"):
        step([0, 1], _sv(2, 0))
    dec.train()
    step([0, 1], _sv(2, 0)).backward()
    torch.cuda.synchronize()
    kept = (step._qids.clone(), step.logits.clone())

    def unchanged():
        torch.cuda.synchronize()
        assert torch.equal(step._qids, kept[0]) and torch.equal(step.logits, kept[1])

    for bad in ([0, 48], [-1, 0], [0, 10 ** 9]):
        with pytest.raises(IndexError):
            step(bad, _sv(2, 0))
        unchanged()
    for bad in ([0], [0, 1, 2]):
        with pytest.raises(ValueError, match="questions"):
            step(bad, _sv(2, 0))
        unchanged()
    small = SplitTrainStep(dec, s48.dev, 2, edge_capacity=int(s48.edges([0, 1]).sum()), max_edges=M)
    small([0, 1], _sv(2, 0)).backward()
    more = next(q for q in range(s48.Q) if s48.edges([0, q]).sum() > s48.edges([0, 1]).sum())
    with pytest.raises(ValueError, match="edge capacity"):
        small([0, more], _sv(2, 0))
    for bad_sv in (_sv(2, 0).half(), _sv(2, 0)[:, :-1]):
        with pytest.raises(ValueError, match="sent_vecs"):
            step([0, 1], bad_sv)
        unchanged()
    stale = step([2, 3], _sv(2, 1))
    step([4, 5], _sv(2, 2)).backward()
    with pytest.raises(RuntimeError, match="earlier call"):
        stale.backward()
    with _flag(not torch.are_deterministic_algorithms_enabled()):
        with pytest.raises(RuntimeError, match="use_deterministic_algorithms"):
            step([0, 1], _sv(2, 0))
    dec.svec2nvec.bias.requires_grad_(False)
    with pytest.raises(RuntimeError, match="require grad"):
        step([0, 1], _sv(2, 0))
    dec.svec2nvec.bias.requires_grad_(True)
    dec.cpu()
    with pytest.raises(RuntimeError, match="moved"):
        step([0, 1], _sv(2, 0))


def test_evaluation_after_training_recaptures_and_equals_eager_eval(s48):
    dev_split = Split(12, seed=53)
    dec = _decoder()
    mbs, bs = 2, 3
    K, M = s48.flat.max_batch_edges(mbs), s48.flat.max_graph_edges()
    Ke, Me = dev_split.flat.max_batch_edges(bs), dev_split.flat.max_graph_edges()
    ev = SplitEvalStep(dec.eval(), dev_split.dev, bs, edge_capacity=Ke, max_edges=Me)
    sv = _sv(bs, 9)
    ev([0, 1, 2], sv)
    assert ev.captures == 1
    dec.train()
    _train(dec, s48, _plan(s48, mbs, seed=6), None, K, M, True)
    dec.eval()
    for i, q in enumerate(([3, 4, 5], [9, 0, 11])):
        logits, attn = ev(q, sv)
        with torch.no_grad():
            ref = dec(sv, *dev_split.dev.batch(q, Ke))
        assert ev.captures == 2, i
        assert torch.equal(logits, ref[0]) and torch.equal(attn, ref[1]), i
