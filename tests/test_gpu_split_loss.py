"""The margin-rank loss in pipeline.SplitTrainStep and the scoring in pipeline.SplitEvalStep, against eager runs on
DeviceSplit.batch with the reference's own formulation (tests/answer_oracle.py: boolean-mask margin-rank loss, per-batch
argmax counts).  Training under torch.use_deterministic_algorithms(True) with dropout 0 is compared bit for bit over two
optimiser batches (losses, logits, dL/dsent_vecs, every .grad after every micro-step, BatchNorm buffers, parameters after
Adam); in the default mode within the training bars.  After capture neither step reads the device.  Needs a GPU: run with
-m gpu."""
import copy
import os
import tempfile

import numpy as np
import pytest
import torch

from qagnn_b200 import data as Dt
from qagnn_b200.pipeline import SplitEvalStep, SplitTrainStep
from tests import answer_oracle as A
from tests.test_gpu_split_train import DT_IDS, DTYPES, N, N_CONCEPT, R, SENT_DIM, T, _autocast, _bn, _decoder, _flag, _same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class Split:
    def __init__(self, n_questions, nc, seed, labels=True):
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "s.graph.adj.pk")
            Dt.synth_adj_pickle(path, n_questions * nc, seed=seed)
            cids, ntypes, scores, lens, flat = Dt.load_flat_adj_cache(path, N, nc)
        self.flat = Dt.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype), np.array(flat.graph_ptr),
                                    nc, N)
        cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)  # inside the decoder's table; the context node keeps id 0
        self.lens = lens
        self.labels = torch.from_numpy(np.random.default_rng(seed).integers(0, nc, n_questions))
        self.dev = Dt.DeviceSplit(self.flat, cids, ntypes, scores, lens, DEV, T, R,
                                  labels=self.labels if labels else None)
        self.Q, self.nc = n_questions, nc

    def sv(self, bs, seed, scale=1.0):
        g = torch.Generator(device=DEV).manual_seed(seed)
        return torch.randn(bs * self.nc, SENT_DIM, device=DEV, generator=g) * scale


@pytest.fixture(scope="module")
def s5():
    return Split(48, 5, seed=61)


@pytest.fixture(scope="module")
def s4():
    return Split(48, 4, seed=62)


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # cuBLAS reads it at call time
    with _flag(True):
        yield


def _labels(s, q):
    return s.dev.labels[torch.from_numpy(np.asarray(q)).to(DEV)]


def _eager(dec, s, q, sv, K, dt, loss):
    """The reference micro-step forward with the reference's loss: (loss, logits)."""
    with _autocast(dt):
        logits, _ = dec(sv, *s.dev.batch(q, K))
        return A.compute_loss(logits.view(-1, s.nc), _labels(s, q), loss), logits


def _plan(s, mbs, seed, n_opt, n_micro=3):
    order = np.random.default_rng(seed).permutation(s.Q)[:n_opt * n_micro * mbs]
    return [[order[(o * n_micro + m) * mbs:(o * n_micro + m + 1) * mbs] for m in range(n_micro)] for o in range(n_opt)]


def _train(dec, s, plan, dt, K, M, loss, use_step, step_loss=None):
    """The optimiser batches of `plan` (qagnn.py:249-278 with Adam and clip_grad_norm_) through SplitTrainStep built with
    `step_loss` (default: no loss keyword) or eagerly with the reference's `loss`; every micro-step's and optimiser step's
    results."""
    params = [p for p in dec.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-3)
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    mbs = len(plan[0][0])
    kw = {} if step_loss is None else {"loss": step_loss}
    step = SplitTrainStep(dec, s.dev, mbs, edge_capacity=K, max_edges=M, autocast_dtype=dt, **kw) if use_step else None
    rec = []
    for o, micro in enumerate(plan):
        opt.zero_grad()
        total = sum(len(q) for q in micro)
        for m, q in enumerate(micro):
            sv = s.sv(mbs, 100 * o + m).requires_grad_(True)
            if use_step:
                out, logits = step(q, sv), step.logits
            else:
                out, logits = _eager(dec, s, q, sv, K, dt, loss)
            r = {"loss": out.detach().clone(), "logits": logits.detach().clone()}
            w = out * len(q) / total
            (scaler.scale(w) if scaler is not None else w).backward()
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


def _both(s, mbs, dt, seed, n_opt, loss):
    dec = _decoder()
    plan = _plan(s, mbs, seed, n_opt)
    K, M = s.flat.max_batch_edges(mbs), s.flat.max_graph_edges()
    ref, _ = _train(copy.deepcopy(dec), s, plan, dt, K, M, loss, False)
    got, step = _train(copy.deepcopy(dec), s, plan, dt, K, M, loss, True, step_loss=loss)
    assert step.captures == 1 and step.mode.startswith("two CUDA graphs") and step.loss == loss
    return got, ref


@pytest.mark.parametrize("nc", [5, 4])
@pytest.mark.parametrize("mbs", [1, 2, 8])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_margin_rank_two_optimiser_batches_equal_eager_bit_for_bit(s5, s4, deterministic, dt, mbs, nc):
    got, ref = _both(s5 if nc == 5 else s4, mbs, dt, seed=mbs + nc, n_opt=2, loss="margin_rank")
    _same(got, ref, bitwise=True)


def _fp16_ulp(x):
    """The spacing of fp16 numbers at |x| (normal range)."""
    return torch.ldexp(torch.ones_like(x), torch.frexp(x.abs().clamp_min(2 ** -14))[1] - 11)


@pytest.mark.parametrize("mbs", [2, 8])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_margin_rank_an_optimiser_batch_equals_eager_in_the_default_mode(s5, dt, mbs):
    got, ref = _both(s5, mbs, dt, seed=20 + mbs, n_opt=1, loss="margin_rank")
    if dt == torch.float16:
        # Under fp16 autocast each micro-step's gradient of a weight is rounded to fp16 once, at the GradScaler's scale. Two
        # summation orders of the edge-table gradient (float atomics) can leave an element one fp16 ulp apart, which is above
        # the 1e-4 bar for elements near the gradient's maximum. Take that ulp off before the training bars.
        for g, r in zip(got, ref):
            for k in r:
                if k.startswith(("grad ", "dL/")):
                    near = (g[k].float() - r[k].float()).abs() <= _fp16_ulp(r[k].float())
                    g[k] = torch.where(near, r[k], g[k])
    _same(got, ref, bitwise=False)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_explicit_cross_entropy_equals_the_default_step_bit_for_bit(s5, deterministic, dt):
    dec = _decoder()
    plan = _plan(s5, 2, seed=30, n_opt=2)
    K, M = s5.flat.max_batch_edges(2), s5.flat.max_graph_edges()
    default, _ = _train(copy.deepcopy(dec), s5, plan, dt, K, M, None, True)
    explicit, step = _train(copy.deepcopy(dec), s5, plan, dt, K, M, None, True, step_loss="cross_entropy")
    assert step.loss == "cross_entropy"
    _same(explicit, default, bitwise=True)


def test_a_bad_loss_is_refused_at_construction(s5):
    K, M = s5.flat.max_batch_edges(2), s5.flat.max_graph_edges()
    with pytest.raises(ValueError, match="loss must be one of"):
        SplitTrainStep(_decoder(), s5.dev, 2, edge_capacity=K, max_edges=M, loss="margin")
    one = Split(4, 1, seed=63)
    with pytest.raises(ValueError, match="at least 2 choices"):
        SplitTrainStep(_decoder(), one.dev, 2, edge_capacity=one.flat.max_batch_edges(2),
                       max_edges=one.flat.max_graph_edges(), loss="margin_rank")


def test_after_capture_neither_step_reads_the_device(s5):
    K, M = s5.flat.max_batch_edges(2), s5.flat.max_graph_edges()
    dec = _decoder()
    train = SplitTrainStep(dec, s5.dev, 2, edge_capacity=K, max_edges=M, loss="margin_rank")
    sv = s5.sv(2, 0).requires_grad_(True)
    train([0, 1], sv).backward()  # captures
    ev_dec = copy.deepcopy(dec).eval()
    ev = SplitEvalStep(ev_dec, s5.dev, 2, edge_capacity=K, max_edges=M)
    ev([0, 1], s5.sv(2, 1))  # captures
    sv_ev, labels = s5.sv(2, 2), _labels(s5, [2, 3])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        train([2, 3], sv).backward()
        ev([4, 5], sv_ev)
        with pytest.raises(RuntimeError):  # the reference's boolean masks do read the device
            A.compute_loss(train.logits.view(-1, 5), labels, "margin_rank")
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert ev.accuracy() >= 0 and int(ev.n_scored) == 4 and train.captures == 1 and ev.captures == 1


def _eager_eval(dec, s, q, sv, K, N_cap, dt):
    with torch.no_grad(), _autocast(dt):
        logits, attn = dec(sv, *s.dev.batch(q, K, N_cap))
    return logits.clone(), attn.clone()


@pytest.mark.parametrize("ragged", [False, True], ids=["padded", "ragged"])
@pytest.mark.parametrize("dt", [None, torch.bfloat16], ids=["fp32", "bf16"])
def test_scoring_a_split_equals_the_reference_count(s5, dt, ragged):
    bs = 4
    scored = s5.Q - 5  # 10 full batches and a partial one of 3; the last 5 questions are not scored
    order = np.random.default_rng(7).permutation(scored - 3)
    batches = [order[i * bs:(i + 1) * bs] for i in range(len(order) // bs)]
    partial = np.arange(scored - 3, scored)
    K, M = s5.flat.max_batch_edges(bs), s5.flat.max_graph_edges()
    N_cap = Dt.split_node_capacity(s5.lens[torch.from_numpy(order)], bs) if ragged else None
    dec = _decoder().eval()
    step = SplitEvalStep(dec, s5.dev, bs, edge_capacity=K, max_edges=M, node_capacity=N_cap, autocast_dtype=dt)
    assert int(step.n_correct) == int(step.n_scored) == 0 and bool((step.predictions == -1).all())
    want = torch.full((s5.Q,), -1, dtype=torch.long)
    n_correct = n_seen = 0
    for i, q in enumerate(batches):
        if i == len(batches) // 2:  # new weights for the second half: the step captures again
            with torch.no_grad():
                for p in dec.fc.parameters():
                    p.mul_(1.5)
        sv = s5.sv(bs, i, scale=3.0)
        logits, attn = step(q, sv)
        ref = _eager_eval(dec, s5, q, sv, K, N_cap, dt)
        assert torch.equal(logits, ref[0]) and torch.equal(attn, ref[1]), i
        c, n = A.evaluate_counts(ref[0].view(bs, 5), _labels(s5, q))
        n_correct, n_seen = n_correct + c, n_seen + n
        want[torch.from_numpy(q)] = ref[0].view(bs, 5).argmax(1).cpu()
    assert step.captures == 2
    sv = s5.sv(len(partial), 99, scale=3.0)
    with torch.no_grad(), _autocast(dt):
        logits, _ = dec(sv, *s5.dev.batch(partial, K))
    step.score(partial, logits)
    c, n = A.evaluate_counts(logits.view(-1, 5), _labels(s5, partial))
    n_correct, n_seen = n_correct + c, n_seen + n
    want[torch.from_numpy(partial)] = logits.view(-1, 5).argmax(1).cpu()
    assert (int(step.n_correct), int(step.n_scored)) == (n_correct, n_seen) == (n_correct, scored)
    assert step.accuracy() == n_correct / scored
    assert step.predictions.dtype == torch.long and torch.equal(step.predictions.cpu(), want)
    assert bool((step.predictions[scored:] == -1).all())

    step.reset_scores()
    assert int(step.n_correct) == int(step.n_scored) == 0 and bool((step.predictions == -1).all())
    q = batches[0]
    logits, _ = step(q, s5.sv(bs, 0, scale=3.0))
    pred = logits.view(bs, 5).argmax(1)
    assert int(step.n_scored) == bs and int(step.n_correct) == int((pred == _labels(s5, q)).sum())
    assert int((step.predictions >= 0).sum()) == bs and torch.equal(step.predictions[torch.from_numpy(q).to(DEV)], pred)


def test_a_repeated_question_counts_every_time_and_keeps_its_last_prediction(s5):
    bs, q = 5, [3, 7, 3, 9, 3]
    K, M = s5.flat.max_batch_edges(bs), s5.flat.max_graph_edges()
    dec = _decoder().eval()
    # sent_vecs whose three slots of question 3 do not all agree, so that which slot's prediction is kept shows
    for seed in range(50):
        sv = s5.sv(bs, 1000 + seed, scale=5.0)
        ref = _eager_eval(dec, s5, q, sv, K, None, None)[0].view(bs, 5).argmax(1)
        if int(ref[4]) != int(ref[0]) and int(ref[4]) != int(ref[2]):
            break
    else:
        pytest.fail("no sent_vecs found whose slots of question 3 disagree")
    step = SplitEvalStep(dec, s5.dev, bs, edge_capacity=K, max_edges=M)
    runs = []
    for _ in range(2):
        step.reset_scores()
        step(q, sv)
        runs.append(step.predictions.clone())
        assert int(step.n_scored) == bs
        assert int(step.n_correct) == int((ref == _labels(s5, q)).sum())
    assert torch.equal(runs[0], runs[1])
    assert int(runs[0][3]) == int(ref[4]) and int(runs[0][7]) == int(ref[1]) and int(runs[0][9]) == int(ref[3])
    assert int((runs[0] >= 0).sum()) == 3
    step.reset_scores()
    step.score(q, _eager_eval(dec, s5, q, sv, K, None, None)[0])  # the same order rule eagerly
    assert torch.equal(step.predictions, runs[0])


def test_a_split_without_labels_is_not_scored(s5):
    plain = Split(12, 5, seed=61, labels=False)
    bs = 3
    K, M = plain.flat.max_batch_edges(bs), plain.flat.max_graph_edges()
    dec = _decoder().eval()
    step = SplitEvalStep(dec, plain.dev, bs, edge_capacity=K, max_edges=M)
    logits, attn = step([0, 4, 8], plain.sv(bs, 0))
    ref = _eager_eval(dec, plain, [0, 4, 8], plain.sv(bs, 0), K, None, None)
    assert torch.equal(logits, ref[0]) and torch.equal(attn, ref[1]) and step.captures == 1
    assert step.n_correct is None and step.n_scored is None and step.predictions is None
    for call in (step.accuracy, step.reset_scores, lambda: step.score([0], logits[:5])):
        with pytest.raises(ValueError, match="no labels"):
            call()
