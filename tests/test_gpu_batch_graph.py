"""A whole optimiser batch as one CUDA graph replay: pipeline.SplitTrainBatchGraph against the eager composition it replaces,
SplitTrainBatch chunks + scaler.scale((losses * w).sum()).backward() + optim.CapturedTail + key.advance_(), on a copy of
the decoder.  Under torch.use_deterministic_algorithms(True) with a DropoutKey at the recipes' dropout, over three consecutive
batches of one epoch order: every parameter, `.grad` and optimiser state, the scaler's scale and growth tracker, the BatchNorm
buffers and each micro-batch's loss and logits agree bit for bit, and the log accumulator equals the Python sum of the loop's
`(loss * mbs / bs).item()`.  Also: an fp16 overflow the scaler skips, a trainable stand-in encoder, a bad question id, a
counter past the epoch, re-capture after a freeze and an unfreeze, and the refusals.  Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

from qagnn_b200 import optim
from qagnn_b200.pipeline import SplitTrainBatch, SplitTrainBatchGraph
from qagnn_b200.training import DropoutKey
from tests.test_gpu_split_train import NC, SENT_DIM, _decoder, deterministic, s48  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DROPOUT = 0.2  # the csqa / obqa recipes' dropout
N_BATCHES = 3
KEY_SEED = 1234


def _kw(s, mbs, dt, loss):
    return dict(edge_capacity=s.dev.max_batch_edges(mbs), max_edges=s.flat.max_graph_edges(), autocast_dtype=dt, loss=loss)


def _sent_vecs(b, bs):
    """The stand-in encoder output of batch b: [bs * nc, S]."""
    g = torch.Generator(device=DEV).manual_seed(100 + b)
    return torch.randn(bs * NC, SENT_DIM, device=DEV, generator=g)


def _optimizer(name, params):
    if name == "radam":
        return optim.RAdam(params, lr=1e-3, weight_decay=0.01)
    return optim.SGD(params, lr=1e-2, momentum=0.9)


class Run:
    """One side of a comparison: a decoder copy, its SplitTrainBatch, optimiser, scaler, scheduler and tail, and (optional)
    a stand-in encoder whose parameters the optimiser also holds."""

    def __init__(self, base, s, mbs, branches, dt, loss, opt_name, clip, init_scale=2.0 ** 16, encoder=None,
                 dropout=DROPOUT):
        self.dec = copy.deepcopy(base)
        self.enc = None if encoder is None else copy.deepcopy(encoder)
        self.key = DropoutKey(KEY_SEED, DEV) if dropout > 0 else None
        self.tb = SplitTrainBatch(self.dec, s.dev, mbs, branches=branches, dropout_key=self.key, **_kw(s, mbs, dt, loss))
        self.named = [(f"dec.{k}", p) for k, p in self.dec.named_parameters()]
        if self.enc is not None:
            self.named += [(f"enc.{k}", p) for k, p in self.enc.named_parameters()]
        self.opt = _optimizer(opt_name, [p for _, p in self.named])
        self.scaler = torch.amp.GradScaler("cuda", init_scale=init_scale) if dt == torch.float16 else None
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda t: 1.0 / (1 + t))
        self.tail = optim.CapturedTail(self.opt, self.scaler, self.sched, clip, [p for _, p in self.named])
        self.total = 0.0

    def record(self, losses, logits, total):
        r = {"losses": losses.clone(), "logits": logits.clone(), "total": total}
        for k, p in self.named:
            r[f"param {k}"] = p.detach().clone()
            if p.grad is not None:
                r[f"grad {k}"] = p.grad.clone()
            for sk, v in self.opt.state.get(p, {}).items():
                if torch.is_tensor(v):
                    r[f"state {k} {sk}"] = v.clone()
        for k, v in self.dec.named_buffers():
            if "running" in k or "num_batches" in k:
                r[f"buffer {k}"] = v.clone()
        if self.scaler is not None:
            r["scale"] = self.scaler._scale.clone()
            r["growth"] = self.scaler._growth_tracker.clone()
        return r


def _backward(run, x):
    (run.scaler.scale(x) if run.scaler is not None else x).backward()


def _eager_batch(run, batch, sv, bs, mbs, enc_in=None):
    """The eager composition of one optimiser batch; with enc_in the encoder runs per micro-batch and its backward follows
    each chunk's, in micro-batch order."""
    run.dec.zero_grad(set_to_none=True)  # the decoder's part of the recipe's zero_grad; the caller owns the encoder's
    if enc_in is not None:
        run.enc.zero_grad(set_to_none=True)
    rows = mbs * NC
    losses, logits = [], []
    j0 = 0
    for chunk in run.tb.chunks(batch):
        if enc_in is None:
            full = [sv[(j0 + j) * rows:(j0 + j + 1) * rows] for j in range(len(chunk))]
            svs = full
        else:
            full = [run.enc(enc_in[(j0 + j) * rows:(j0 + j + 1) * rows]) for j in range(len(chunk))]
            svs = [v.detach().requires_grad_(True) for v in full]
        out = run.tb(chunk, svs)
        logits += [x.clone() for x in run.tb.logits]
        w = torch.full((len(chunk),), mbs / bs, dtype=torch.float32, device=DEV)
        _backward(run, (out * w).sum())
        if enc_in is not None:
            for v, leaf in zip(full, svs):
                v.backward(leaf.grad)
        for x in out:
            run.total += (x * mbs / bs).item()  # qagnn.py:261 and `total_loss += loss.item()`
        losses.append(out.detach().clone())
        j0 += len(chunk)
    run.tail()
    if run.key is not None:
        run.key.advance_()
    return run.record(torch.cat(losses), torch.stack(logits), run.total)


def _graph_batch(run, gb, sv, mbs, enc_in=None, check_sync=False):
    if enc_in is None:
        gb.sent_vecs.copy_(sv)
        if check_sync:
            torch.cuda.set_sync_debug_mode("error")
        try:
            gb.step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    else:
        rows = mbs * NC
        run.enc.zero_grad(set_to_none=True)
        full = [run.enc(enc_in[j * rows:(j + 1) * rows]) for j in range(gb.n_micro)]
        for j, v in enumerate(full):
            gb.sent_vecs[j * rows:(j + 1) * rows].copy_(v.detach())
        gb.step()
        for j, v in enumerate(full):
            v.backward(gb.d_sent_vecs[j])
        run.tail()
    return run.record(gb.losses, gb.logits, float(gb.total_loss.item()))


def _compare(got, ref):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys(), (i, sorted(set(g) ^ set(r)))
        assert sum(k.startswith("grad dec.") for k in r) > 10
        for k in r:
            if k == "total":
                assert g[k] == r[k], f"batch {i}: total_loss {g[k]!r} != {r[k]!r}"
            else:
                assert g[k].dtype == r[k].dtype and torch.equal(_bits(g[k]), _bits(r[k])), f"batch {i}: {k}"


def _bits(t):
    """The tensor's bit patterns: a skipped fp16 step leaves NaN in .grad, which torch.equal never calls equal."""
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.int8}[t.element_size()]) if t.is_floating_point() else t


def _order(s, seed):
    return np.random.default_rng(seed).permutation(s.Q)


def _check(s, *, branches, mbs, bs, dt, loss, opt_name, clip, init_scale=2.0 ** 16, seed=0, eager_first=False):
    """N_BATCHES graph batches against the eager composition; with eager_first both sides first train one batch eagerly
    through the same SplitTrainBatch and tail, which the graph then takes over."""
    base = _decoder(dropout=DROPOUT)
    order = _order(s, seed)
    args = (s, mbs, branches, dt, loss, opt_name, clip, init_scale)
    ref_run, run = Run(base, *args), Run(base, *args)
    first = int(eager_first)

    def batch(b):
        return order[b * bs:(b + 1) * bs]

    ref = [_eager_batch(ref_run, batch(b), _sent_vecs(b, bs), bs, mbs) for b in range(first + N_BATCHES)]
    got = [_eager_batch(run, batch(b), _sent_vecs(b, bs), bs, mbs) for b in range(first)]
    gb = SplitTrainBatchGraph(run.tb, bs, scaler=run.scaler, tail=run.tail)
    gb.set_epoch(order[first * bs:])
    gb.total_loss.fill_(run.total)
    got += [_graph_batch(run, gb, _sent_vecs(b, bs), mbs, check_sync=b > first) for b in range(first, first + N_BATCHES)]
    _compare(got, ref)
    assert gb.captures == 1 and run.tail.captures == first
    assert gb.node_count() > 0 and gb.node_count(recursive=True) > gb.node_count()
    assert int(gb.counter) == N_BATCHES and int(run.key.draw) == first + N_BATCHES
    return ref, got


CASES = [  # branches, mbs, bs, autocast, loss, optimiser, clip
    (1, 2, 4, None, "cross_entropy", "radam", 1.0),
    (2, 2, 8, torch.float16, "cross_entropy", "radam", 1.0),
    (4, 1, 6, torch.bfloat16, "margin_rank", "sgd", 0.0),
    (2, 2, 2, torch.float16, "margin_rank", "sgd", 1.0),   # one micro-batch per batch
    (2, 1, 6, None, "margin_rank", "sgd", 1.0),
    (4, 2, 12, torch.bfloat16, "cross_entropy", "radam", 0.0),
]


@pytest.mark.parametrize("branches,mbs,bs,dt,loss,opt_name,clip", CASES,
                         ids=[f"S{c[0]}-mbs{c[1]}-bs{c[2]}-{c[3]}-{c[4]}-{c[5]}-clip{c[6]}" for c in CASES])
def test_three_batches_equal_the_eager_composition_bit_for_bit(s48, deterministic, branches, mbs, bs, dt, loss, opt_name,
                                                               clip):
    _check(s48, branches=branches, mbs=mbs, bs=bs, dt=dt, loss=loss, opt_name=opt_name, clip=clip, seed=branches * 10 + mbs)


def test_the_graph_takes_over_from_eager_batches_of_its_split_train_batch(s48, deterministic):
    _check(s48, branches=4, mbs=1, bs=6, dt=torch.float16, loss="cross_entropy", opt_name="radam", clip=1.0, seed=8,
           eager_first=True)


def test_an_fp16_overflow_skips_the_step_as_the_scaler_does(s48, deterministic):
    ref, got = _check(s48, branches=2, mbs=2, bs=8, dt=torch.float16, loss="cross_entropy", opt_name="radam", clip=1.0,
                      init_scale=2.0 ** 100, seed=5)
    first = _decoder(dropout=DROPOUT)
    for k, p in first.named_parameters():
        assert torch.equal(got[-1][f"param dec.{k}"], p.detach()), k  # every step was skipped
    assert float(got[-1]["scale"]) == 2.0 ** (100 - N_BATCHES)


def test_a_trainable_encoder_takes_d_sent_vecs_in_micro_batch_order(s48, deterministic):
    base = _decoder(dropout=DROPOUT)
    torch.manual_seed(3)
    encoder = torch.nn.Linear(SENT_DIM, SENT_DIM).to(DEV)
    branches, mbs, bs = 2, 2, 8
    order = _order(s48, 9)
    args = (s48, mbs, branches, torch.float16, "cross_entropy", "radam", 1.0)
    ref_run, run = Run(base, *args, encoder=encoder), Run(base, *args, encoder=encoder)

    def enc_in(b):
        return torch.randn(bs * NC, SENT_DIM, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7 + b))

    ref = [_eager_batch(ref_run, order[b * bs:(b + 1) * bs], None, bs, mbs, enc_in(b)) for b in range(N_BATCHES)]
    gb = SplitTrainBatchGraph(run.tb, bs, scaler=run.scaler, tail=None)
    gb.set_epoch(order)
    got = [_graph_batch(run, gb, None, mbs, enc_in(b)) for b in range(N_BATCHES)]
    assert all(any(k.startswith("grad enc.") for k in r) for r in ref)
    _compare(got, ref)
    assert gb.d_sent_vecs.shape == (bs // mbs, mbs * NC, SENT_DIM)


def _graph_run(s, bs=4, mbs=2, branches=2, **kw):
    run = Run(_decoder(dropout=DROPOUT), s, mbs, branches, None, "cross_entropy", "radam", 1.0, **kw)
    return run, SplitTrainBatchGraph(run.tb, bs, scaler=run.scaler, tail=run.tail)


def test_a_bad_question_id_raises_index_error_at_the_next_call(s48):
    run, gb = _graph_run(s48)
    order = _order(s48, 1)
    order[5] = s48.Q + 3  # in batch 1
    gb.set_epoch(order)
    gb.step()
    gb.step()
    torch.cuda.synchronize()
    with pytest.raises(IndexError, match="question id outside"):
        gb.step()
    gb.step()  # the word was cleared: the epoch goes on
    assert int(gb.counter) == 3


def test_a_counter_past_the_epoch_raises_value_error(s48):
    run, gb = _graph_run(s48)
    order = _order(s48, 2)[:10]  # two full batches of 4 and a partial one
    gb.set_epoch(order)
    assert gb.n_batches == 2
    gb.step()
    gb.counter.fill_(2)  # the device counter past the epoch behind the host's back
    gb.step()
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="past its epoch"):
        gb.step()
    gb.set_epoch(order)
    gb.step()
    gb.step()
    with pytest.raises(ValueError, match="full batches are done"):
        gb.step()


def test_a_freeze_and_an_unfreeze_capture_again(s48, deterministic):
    base = _decoder(dropout=DROPOUT)
    torch.manual_seed(4)
    encoder = torch.nn.Linear(SENT_DIM, SENT_DIM).to(DEV).requires_grad_(False)
    branches, mbs, bs = 2, 2, 8
    order = _order(s48, 3)
    args = (s48, mbs, branches, torch.float16, "cross_entropy", "radam", 1.0)
    runs = [Run(base, *args, encoder=encoder), Run(base, *args, encoder=encoder)]
    gb = SplitTrainBatchGraph(runs[1].tb, bs, scaler=runs[1].scaler, tail=runs[1].tail)
    gb.set_epoch(order)
    x = torch.randn(3, SENT_DIM, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    recs = [[], []]
    for b in range(N_BATCHES):
        for i, run in enumerate(runs):
            enc = run.enc
            if b == 1:  # unfreeze: the encoder's parameters get a gradient the tail then steps too
                enc.requires_grad_(True)
                enc(x).square().sum().backward()
            if b == 2:  # freeze again
                enc.requires_grad_(False)
                enc.zero_grad(set_to_none=True)
            sv, batch = _sent_vecs(b, bs), order[b * bs:(b + 1) * bs]
            recs[i].append(_eager_batch(run, batch, sv, bs, mbs) if i == 0 else _graph_batch(run, gb, sv, mbs))
        assert gb.captures == b + 1
    assert any(k.startswith("grad enc.") for k in recs[0][1]) and not any(k.startswith("grad enc.") for k in recs[0][2])
    _compare(recs[1], recs[0])
    p = runs[1].dec.fc.layers[0].weight
    p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="require grad"):
        gb.step()


def test_refusals(s48):
    run, gb = _graph_run(s48)
    with pytest.raises(RuntimeError, match="set_epoch"):
        gb.step()
    with pytest.raises(ValueError, match="multiple"):
        SplitTrainBatchGraph(run.tb, 5)
    with pytest.raises(ValueError, match="scaler"):
        SplitTrainBatchGraph(run.tb, 4, scaler=torch.amp.GradScaler("cuda"), tail=run.tail)
    small = SplitTrainBatch(run.dec, s48.dev, 2, branches=2, edge_capacity=s48.dev.max_batch_edges(2) - 1,
                            max_edges=s48.flat.max_graph_edges(), dropout_key=run.key)
    with pytest.raises(ValueError, match="edge capacity"):
        SplitTrainBatchGraph(small, 4)
    unkeyed = SplitTrainBatch(run.dec, s48.dev, 2, branches=2, **_kw(s48, 2, None, "cross_entropy"))
    with pytest.raises(ValueError, match="DropoutKey"):
        SplitTrainBatchGraph(unkeyed, 4)
    gb.set_epoch(_order(s48, 4))
    gb.step()
    run.dec.eval()
    with pytest.raises(RuntimeError, match="train"):
        gb.step()
    run.dec.train()
    p = run.dec.fc.layers[0].weight
    p.data = p.data.clone()
    with pytest.raises(RuntimeError, match="moved"):
        gb.step()
