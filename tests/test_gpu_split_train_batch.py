"""Concurrent micro-steps of an optimiser batch on one GPU: pipeline.SplitTrainBatch against the plain SplitTrainStep loop.
Under torch.use_deterministic_algorithms(True) with dropout 0, two optimiser batches of 6 full micro-batches (the second
ending in a partial one, run eagerly) at branches 1, 2, 4 and 8, micro-batches of 1 and 2 questions, fp32, bf16 and fp16
with a GradScaler and both losses: every micro-batch's loss, logits and dL/dsent_vecs and every decoder `.grad` after
every chunk equal the loop's bit for bit, and so do the parameters after optim.RAdam, with zero_grad() before the first
batch and zero_grad(set_to_none=False) before the second.  The BatchNorm running statistics are within the fold's bar and
num_batches_tracked is exact.  Branches given the same micro-batch write the same slot rows, each the plain step's gradient
of that micro-batch; a chunk after capture reads nothing on the host; with dropout each branch draws its own masks; and
the refusals.  Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

import qagnn_b200.training
from qagnn_b200 import optim
from qagnn_b200.pipeline import SplitTrainBatch, SplitTrainStep, train_chunks
from tests.test_data_parallel_cpu import BN_BAR
from tests.test_gpu_split_train import DT_IDS, DTYPES, NC, SENT_DIM, _autocast, _decoder, deterministic, s48  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_MICRO = 6  # full micro-batches per optimiser batch: uneven chunks at branches 4 (4 + 2) and 8 (one chunk of 6)


def _sv(q, requires_grad=True):
    """The stand-in encoder output of a micro-batch: a function of its question ids alone, a leaf."""
    g = torch.Generator(device=DEV).manual_seed(int(np.asarray(q)[0]) * 1000 + len(q))
    return torch.randn(len(q) * NC, SENT_DIM, device=DEV, generator=g).requires_grad_(requires_grad)


def _batches(s, mbs, seed):
    order = np.random.default_rng(seed).permutation(s.Q)
    n = N_MICRO * mbs
    second = order[n:2 * n + (1 if mbs > 1 else 0)]  # ends in a partial micro-batch of one question when mbs > 1
    return [order[:n], second]


def _grads(dec):
    return {f"grad {k}": p.grad.clone() for k, p in dec.named_parameters() if p.grad is not None}


def _bn(dec):
    return {k: v.detach().clone() for k, v in dec.named_buffers() if "running" in k or "num_batches" in k}


def _kw(s, mbs, dt, loss_name):
    return dict(edge_capacity=s.flat.max_batch_edges(mbs), max_edges=s.flat.max_graph_edges(), autocast_dtype=dt,
                loss=loss_name)


def _backward(x, scaler):
    (scaler.scale(x) if scaler is not None else x).backward()


def _train(dec, s, batches, mbs, dt, loss_name, branches, plain):
    """The recipe's loop over `batches` in chunks of at most `branches` micro-batches, through SplitTrainBatch or (plain)
    a SplitTrainStep per micro-batch.  Returns one record per chunk and one per optimiser batch, and the SplitTrainBatch."""
    kw = _kw(s, mbs, dt, loss_name)
    tb = None if plain else SplitTrainBatch(dec, s.dev, mbs, branches=branches, **kw)
    step = SplitTrainStep(dec, s.dev, mbs, **kw) if plain else None
    opt = optim.RAdam([p for p in dec.parameters() if p.requires_grad], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    rec = []
    for b, batch in enumerate(batches):
        opt.zero_grad(set_to_none=b == 0)
        for chunk in train_chunks(batch, mbs, branches):
            svs = [_sv(q) for q in chunk]
            w = torch.tensor([len(q) / len(batch) for q in chunk], device=DEV)
            if plain:
                losses, logits = [], []
                for j, (q, sv) in enumerate(zip(chunk, svs)):
                    loss = step(q, sv)
                    losses.append(loss.detach().clone())
                    logits.append(step.logits.clone())
                    _backward(loss * w[j], scaler)
                losses = torch.stack(losses)
            else:
                losses = tb(chunk, svs)
                logits = [x.clone() for x in tb.logits]
                _backward((losses * w).sum(), scaler)
            r = {"losses": losses.detach().clone(), "logits": torch.stack(logits)}
            r.update({f"dL/dsent_vecs {j}": sv.grad.clone() for j, sv in enumerate(svs)})
            r.update(_grads(dec))
            rec.append(r)
        rest = batch[len(batch) // mbs * mbs:]
        if len(rest):  # the final partial micro-batch, eagerly in both loops
            with _autocast(dt):
                logits, _ = dec(_sv(rest), *s.dev.batch(rest, kw["edge_capacity"]))
                loss = qagnn_b200.training.answer_loss(logits, s.dev.labels[torch.from_numpy(rest).to(DEV)], NC, loss_name)
            _backward(loss * (len(rest) / len(batch)), scaler)
        r = _grads(dec)
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        r.update({f"param {k}": p.detach().clone() for k, p in dec.named_parameters()})
        r.update({f"buffer {k}": v for k, v in _bn(dec).items()})
        rec.append(r)
    return rec, tb


def _compare(got, ref):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys(), (i, sorted(set(g) ^ set(r)))
        assert sum(k.startswith("grad ") for k in r) > 10
        for k in r:
            what = f"record {i}: {k}"
            if k.startswith("buffer ") and "num_batches" not in k:
                assert float((g[k] - r[k]).abs().max()) <= BN_BAR * float(r[k].abs().max()), what
            else:
                assert g[k].dtype == r[k].dtype and torch.equal(g[k], r[k]), what


def _check_equal(s, mbs, dt, loss_name, branches, seed):
    base = _decoder()
    batches = _batches(s, mbs, seed)
    ref, _ = _train(copy.deepcopy(base), s, batches, mbs, dt, loss_name, branches, plain=True)
    got, tb = _train(copy.deepcopy(base), s, batches, mbs, dt, loss_name, branches, plain=False)
    assert tb.mode.startswith(f"{branches} branches")
    _compare(got, ref)


@pytest.mark.parametrize("branches", [1, 2, 4, 8])
@pytest.mark.parametrize("mbs", [1, 2])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_two_optimiser_batches_equal_the_plain_loop_bit_for_bit(s48, deterministic, dt, mbs, branches):
    _check_equal(s48, mbs, dt, "cross_entropy", branches, seed=10 * mbs + branches)


@pytest.mark.parametrize("branches", [1, 4])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_the_margin_rank_loss_equals_the_plain_loop_bit_for_bit(s48, deterministic, dt, branches):
    _check_equal(s48, 2, dt, "margin_rank", branches, seed=77 + branches)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_branches_given_one_micro_batch_write_the_plain_steps_gradient(s48, deterministic, dt):
    """Branches 0, 2 and 3 take the same micro-batch and sent_vecs: their slot rows are the same bits, and every row is the
    plain step's gradient of its micro-batch.  A chunk after capture reads nothing on the host."""
    base = _decoder()
    mbs = 2
    q0, q1 = np.arange(0, mbs), np.arange(10, 10 + mbs)
    chunk = [q0, q1, q0, q0]
    kw = _kw(s48, mbs, dt, "cross_entropy")
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    w = torch.full((4,), 0.25, device=DEV)

    dec = copy.deepcopy(base)
    tb = SplitTrainBatch(dec, s48.dev, mbs, branches=4, **kw)
    for call in range(2):  # the first call captures; the second runs under the sync check
        svs = [_sv(q, requires_grad=False) for q in chunk]
        for p in dec.parameters():
            p.grad = None
        if call:
            torch.cuda.set_sync_debug_mode("error")
        try:
            losses = tb(chunk, svs)
            _backward((losses * w).sum(), scaler)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    rows = [[t.clone() for t in tb._row_views(j, tb._used)] for j in range(4)]
    names = [n for n, p in dec.named_parameters() if p.requires_grad]
    names = [names[i] for i in tb._used]

    pdec = copy.deepcopy(base)
    step = SplitTrainStep(pdec, s48.dev, mbs, **kw)
    pscaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    plain = {}
    for q in (q0, q1):
        for p in pdec.parameters():
            p.grad = None
        _backward(step(q, _sv(q, requires_grad=False)) * w[0], pscaler)
        grads = dict(pdec.named_parameters())
        plain[int(q[0])] = [grads[n].grad.clone() for n in names]
    for j in (2, 3):
        for a, b in zip(rows[j], rows[0]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"branch {j}"
    for j, q in enumerate(chunk):
        for n, a, b in zip(names, rows[j], plain[int(q[0])]):
            assert torch.equal(a, b), f"branch {j}: {n}"


def test_dropout_draws_other_masks_per_branch_and_batchnorm_advances_by_the_count(s48):
    base = _decoder(dropout=0.2)
    mbs, q = 2, np.arange(4, 6)
    kw = _kw(s48, mbs, None, "cross_entropy")
    dec = copy.deepcopy(base)
    tb = SplitTrainBatch(dec, s48.dev, mbs, branches=2, **kw)
    sv = _sv(q)
    before = _bn(dec)
    losses = tb([q, q], [sv, sv])
    losses.sum().backward()
    after = _bn(dec)
    rows = [torch.cat([t.reshape(-1) for t in tb._row_views(j, tb._used)]) for j in range(2)]
    assert torch.isfinite(losses).all() and all(torch.isfinite(r).all() for r in rows)
    assert torch.isfinite(sv.grad).all()
    assert not torch.equal(losses[0], losses[1]) and not torch.equal(rows[0], rows[1])
    # the plain step's count for two micro-steps
    pdec = copy.deepcopy(base)
    step = SplitTrainStep(pdec, s48.dev, mbs, **kw)
    for _ in range(2):
        step(q, _sv(q)).backward()
    plain = _bn(pdec)
    for k in before:
        if "num_batches" in k:
            assert int(after[k]) == int(plain[k]) and int(after[k]) > int(before[k]), k
        else:
            assert torch.isfinite(after[k]).all() and not torch.equal(after[k], before[k]), k


def test_refusals(s48):
    mbs = 2
    kw = _kw(s48, mbs, None, "cross_entropy")
    dec = _decoder()
    tb = SplitTrainBatch(dec, s48.dev, mbs, branches=2, **kw)
    q0, q1 = np.arange(0, 2), np.arange(2, 4)
    losses = tb([q0, q1], [_sv(q0), _sv(q1)])
    stale = tb([q0], [_sv(q0)])
    with pytest.raises(RuntimeError, match="earlier call"):
        losses.sum().backward()
    stale.sum().backward()
    with pytest.raises(ValueError, match="sent_vecs is"):
        tb([q0], [_sv(q0).double()])
    with pytest.raises(ValueError, match="sent_vecs is"):
        tb([q0], [torch.zeros(3, SENT_DIM, device=DEV)])
    with pytest.raises(ValueError, match="a micro-batch of 1 questions"):
        tb([q0, q1[:1]], [_sv(q0), _sv(q1[:1])])
    with pytest.raises(ValueError, match="a chunk of 3"):
        tb([q0, q1, q0], [_sv(q0), _sv(q1), _sv(q0)])
    dec.eval()
    with pytest.raises(RuntimeError, match="train"):
        tb([q0], [_sv(q0)])
    dec.train()
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not was)
    try:
        with pytest.raises(RuntimeError, match="deterministic"):
            tb([q0], [_sv(q0)])
    finally:
        torch.use_deterministic_algorithms(was)
    p = dec.fc.layers[0].weight
    p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="require grad"):
        tb([q0], [_sv(q0)])
    p.requires_grad_(True)
    tb([q0], [_sv(q0)]).sum().backward()  # still usable
    p.data = p.data.clone()
    with pytest.raises(RuntimeError, match="moved"):
        tb([q0], [_sv(q0)])
