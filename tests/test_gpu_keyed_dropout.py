"""Keyed dropout on the GPU (qagnn_keyed_dropout_forward_typed / _backward_typed, training.keyed_dropout).

The kernel equals the numpy mirror bit for bit (values and mask bits) for fp32, fp16 and bf16 at p in {0, 0.1, 0.2, 0.5, 1},
A in {1, 4}, rows with L % 4 != 0 and == 0, several questions and choices, draws 0, 1 and 2^32 - 1, aligned and unaligned;
its backward is dy * mask * scale.  A question's masks do not depend on its row, the batch size or the stream; a new draw or
seed changes them.  The headline: under torch.use_deterministic_algorithms(True) with every dropout site of the decoder at
the recipe's rate (0.2, the pooler's 0.1), two optimiser batches through SplitTrainBatch at branches 1, 2, 4 and 8 equal
the keyed SplitTrainStep loop bit for bit, and so does DataParallelSplitTrain at one rank (and at two, with two GPUs); the
eager decoder under keyed_dropout equals the step's replay.  A replayed keyed chunk and advance_() read nothing on the
host, and the refusals.  Needs a GPU: run with -m gpu."""
import copy
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import qagnn_b200
from oracle import qagnn_oracle as O
from qagnn_b200 import distributed as D
from qagnn_b200 import optim, training
from qagnn_b200.pipeline import SplitTrainBatch, SplitTrainStep, train_chunks
from tests import keyed_dropout_oracle as K
from tests.test_gpu_data_parallel import _free_port, _split
from tests.test_gpu_split_train import D as D_
from tests.test_gpu_split_train import (DT_IDS, DTYPES, N_CONCEPT, NC, R, SENT_DIM, T, _autocast, deterministic,  # noqa: F401
                                        s48)
from tests.test_gpu_split_train_batch import _backward, _batches, _bn, _compare, _grads, _kw, _sv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TORCH_DT = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
SEED = 0x9E37_79B9_7F4A_7C15


# ---- the kernel against the mirror -----------------------------------------------------------------------------------------

def _keyed(x, key, qids, p, site, graph_dim):
    """The keyed op at one site on x."""
    with training.keyed_dropout(key, qids, NC):
        y = training.dropout(x, p, True, site, graph_dim=graph_dim)
    return y


def _mask_words(y):
    return y.grad_fn.saved_tensors[0].cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("p", [0.0, 0.1, 0.2, 0.5, 1.0])
@pytest.mark.parametrize("A", [1, 4])
@pytest.mark.parametrize("L", [37, 40])
@pytest.mark.parametrize("dt", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("aligned", [True, False])
def test_kernel_equals_the_mirror_bit_for_bit(dt, p, A, L, aligned):
    dtype = TORCH_DT[dt]
    qids_h = np.array([3, 2 ** 33 + 11, 0], dtype=np.int64)  # a question id past 32 bits keeps its low word
    G = len(qids_h) * NC
    qids = torch.from_numpy(qids_h).to(DEV)
    key = training.DropoutKey(SEED, DEV)
    shape = (G, L) if A == 1 else (A, G, L)
    n = A * G * L
    g = torch.Generator(device=DEV).manual_seed(A * 1000 + L)
    off = 0 if aligned else 1
    buf = torch.randn(n + off, device=DEV, generator=g).to(dtype)
    x = buf[off:].view(shape).detach().requires_grad_(True)
    dy_buf = torch.randn(n + off, device=DEV, generator=g).to(dtype)
    dy = dy_buf[off:].view(shape)
    site = 33 if A > 1 else 5
    for draw in (0, 1, 2 ** 32 - 1):
        key.draw.fill_(draw)
        y = _keyed(x, key, qids, p, site, graph_dim=1 if A > 1 else 0)
        keep = K.keep_mask(A, G, L, p, SEED, draw, qids_h, NC, site)
        want = K.apply(x.detach().float().cpu().numpy().reshape(A, G, L), keep, p, dtype).view(shape)
        assert y.dtype == dtype and y.shape == x.shape
        bits = torch.int32 if dtype == torch.float32 else torch.int16
        assert torch.equal(y.detach().cpu().view(bits), want.view(bits)), f"draw {draw}"
        assert np.array_equal(_mask_words(y), K.pack_bits(keep)), f"draw {draw}"
        if p == 0.0:
            assert torch.equal(y.detach().view(bits), x.detach().view(bits))
        (dx,) = torch.autograd.grad(y, x, dy)
        want_dx = K.apply(dy.float().cpu().numpy().reshape(A, G, L), keep, p, dtype).view(shape)
        assert torch.equal(dx.cpu().view(bits), want_dx.view(bits)), f"draw {draw}"


def test_a_questions_masks_depend_on_nothing_but_the_question():
    """Question 9's masks at one site: the same in any row of any batch size, on any stream; not under another draw or
    seed."""
    L, site = 1203, 0
    key = training.DropoutKey(7, DEV)
    ones = torch.ones(6 * NC, L, device=DEV)

    def masks_of_9(order, stream=None, k=key):
        q = torch.tensor(order, device=DEV)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream or torch.cuda.current_stream()):
            y = _keyed(ones[:len(order) * NC], k, q, 0.5, site, 0)
        torch.cuda.synchronize()
        r = order.index(9)
        return y[r * NC:(r + 1) * NC] != 0

    ref = masks_of_9([9])
    assert 0.3 < float(ref.float().mean()) < 0.7
    assert torch.equal(masks_of_9([4, 9]), ref) and torch.equal(masks_of_9([1, 2, 3, 9, 5, 6]), ref)
    assert torch.equal(masks_of_9([9, 4], stream=torch.cuda.Stream()), ref)
    key.advance_()
    assert not torch.equal(masks_of_9([9]), ref)
    assert not torch.equal(masks_of_9([9], k=training.DropoutKey(8, DEV)), ref)


# ---- the training loops --------------------------------------------------------------------------------------------------

def _recipe_decoder(dev=DEV, seed=8):
    """test_gpu_split_train._decoder at the recipe's rates: 0.2 at the embedding, GNN and fc sites, 0.1 in the pooler."""
    torch.manual_seed(seed)
    dec = qagnn_b200.QAGNN(None, 2, T, R, SENT_DIM, N_CONCEPT, D_, 32, 2, D_, 1, 0.2, 0.2, 0.2)
    dec.gnn.load_state_dict(O.random_state_dict(2, D_, T, R, "prod", seed=seed))
    dec.pooler.attn_dropout.p = dec.pooler.dropout.p = 0.1
    return dec.to(dev).train()


def _eager_loss(dec, split, q, sv, K_, dt, loss_name, key):
    """The partial micro-batch of the loop: split.batch + decoder + answer loss under keyed_dropout."""
    qd = torch.from_numpy(np.asarray(q, dtype=np.int64)).to(split.device)
    with training.keyed_dropout(key, qd, NC), _autocast(dt):
        logits, attn = dec(sv, *split.batch(q, K_))
        return training.answer_loss(logits, split.labels[qd], NC, loss_name), logits, attn


def _train_keyed(dec, s, batches, mbs, dt, loss_name, branches, plain):
    """test_gpu_split_train_batch._train with a DropoutKey, advanced after every optimiser step."""
    kw = _kw(s, mbs, dt, loss_name)
    key = training.DropoutKey(SEED, DEV)
    tb = None if plain else SplitTrainBatch(dec, s.dev, mbs, branches=branches, dropout_key=key, **kw)
    step = SplitTrainStep(dec, s.dev, mbs, dropout_key=key, **kw) if plain else None
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
        if len(rest):
            loss = _eager_loss(dec, s.dev, rest, _sv(rest), kw["edge_capacity"], dt, loss_name, key)[0]
            _backward(loss * (len(rest) / len(batch)), scaler)
        r = _grads(dec)
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        key.advance_()
        r.update({f"param {k}": p.detach().clone() for k, p in dec.named_parameters()})
        r.update({f"buffer {k}": v for k, v in _bn(dec).items()})
        rec.append(r)
    return rec, tb


def _check_keyed(s, mbs, dt, loss_name, branches, seed):
    base = _recipe_decoder()
    batches = _batches(s, mbs, seed)
    ref, _ = _train_keyed(copy.deepcopy(base), s, batches, mbs, dt, loss_name, branches, plain=True)
    got, tb = _train_keyed(copy.deepcopy(base), s, batches, mbs, dt, loss_name, branches, plain=False)
    assert tb.mode.startswith(f"{branches} branches")
    _compare(got, ref)


@pytest.mark.parametrize("branches", [1, 2, 4, 8])
@pytest.mark.parametrize("mbs", [1, 2])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_keyed_split_train_batch_equals_the_keyed_loop_bit_for_bit(s48, deterministic, dt, mbs, branches):
    _check_keyed(s48, mbs, dt, "cross_entropy", branches, seed=10 * mbs + branches)


@pytest.mark.parametrize("branches", [1, 4])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_keyed_margin_rank_loss_equals_the_keyed_loop_bit_for_bit(s48, deterministic, dt, branches):
    _check_keyed(s48, 2, dt, "margin_rank", branches, seed=77 + branches)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_eager_decoder_under_the_key_equals_the_steps_replay(s48, deterministic, dt):
    mbs = 2
    kw = _kw(s48, mbs, dt, "cross_entropy")
    base = _recipe_decoder()
    eager_dec, step_dec = copy.deepcopy(base), copy.deepcopy(base)
    key = training.DropoutKey(SEED, DEV)
    step = SplitTrainStep(step_dec, s48.dev, mbs, dropout_key=key, **kw)
    for i, q in enumerate([np.array([0, 1]), np.array([17, 3]), np.array([40, 41])]):
        sv_e, sv_s = _sv(q), _sv(q)
        loss_e, logits_e, attn_e = _eager_loss(eager_dec, s48.dev, q, sv_e, kw["edge_capacity"], dt, "cross_entropy", key)
        loss_s = step(q, sv_s)
        assert torch.equal(loss_s, loss_e) and torch.equal(step.logits, logits_e) and torch.equal(step.pool_attn, attn_e), i
        loss_e.backward()
        loss_s.backward()
        assert torch.equal(sv_s.grad, sv_e.grad), i
        key.advance_()
    for (k, p), pe in zip(step_dec.named_parameters(), eager_dec.parameters()):
        assert (p.grad is None) == (pe.grad is None) and (p.grad is None or torch.equal(p.grad, pe.grad)), k
    # without the key the same decoder draws torch's masks: another loss
    with _autocast(dt):
        logits, _ = copy.deepcopy(base)(_sv(np.array([0, 1])), *s48.dev.batch(np.array([0, 1]), kw["edge_capacity"]))
    key.draw.zero_()
    assert not torch.equal(logits, _eager_loss(copy.deepcopy(base), s48.dev, np.array([0, 1]), _sv(np.array([0, 1])),
                                               kw["edge_capacity"], dt, "cross_entropy", key)[1])


def _run_dp(dec, split, edges, batches, mbs, dt, dp):
    """The loop over `batches`, plain (dp False) or through DataParallelSplitTrain, with one DropoutKey of SEED; `edges` is
    (edge capacity, max edges)."""
    dev = split.device
    K_, M = edges
    step = SplitTrainStep(dec, split, mbs, edge_capacity=K_, max_edges=M, autocast_dtype=dt,
                          dropout_key=training.DropoutKey(SEED, dev))
    key = step.dropout_key
    opt = optim.RAdam([p for p in dec.parameters() if p.requires_grad], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    dpt = D.DataParallelSplitTrain(step, split, batch_size=max(len(b) for b in batches), micro_batch_size=mbs,
                                   ) if dp else None
    rec = []
    for batch in batches:
        opt.zero_grad()
        micro = dpt.micro_batches(batch) if dp else [batch[a:a + mbs] for a in range(0, len(batch), mbs)]
        for q in micro:
            g = torch.Generator(device=dev).manual_seed(int(q[0]) * 1000 + len(q))
            sv = torch.randn(len(q) * NC, SENT_DIM, device=dev, generator=g)
            if dp:
                with dpt.micro_step():
                    _backward(dpt.loss(q, sv) * len(q) / len(batch), scaler)
            else:
                loss = step(q, sv) if len(q) == mbs else _eager_loss(dec, split, q, sv, K_, dt, "cross_entropy", key)[0]
                _backward(loss * len(q) / len(batch), scaler)
        if dp:
            dpt.reduce_(len(batch))
        r = {f"grad {k}": p.grad.clone() for k, p in dec.named_parameters() if p.grad is not None}
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        key.advance_()
        r.update({f"param {k}": p.detach().clone() for k, p in dec.named_parameters()})
        rec.append(r)
    return rec


def _dp_batches(Q, mbs, n_ranks):
    order = np.random.default_rng(5).permutation(Q)
    bs = 3 * mbs * n_ranks
    return [order[:bs], order[bs:2 * bs - mbs + 1]]  # the second ends in a micro-batch of one question


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_keyed_data_parallel_at_one_rank_equals_the_keyed_loop(s48, deterministic, dt):
    mbs = 2
    edges = (s48.flat.max_batch_edges(mbs), s48.flat.max_graph_edges())
    batches = _dp_batches(s48.Q, mbs, 1)
    base = _recipe_decoder()
    ref = _run_dp(copy.deepcopy(base), s48.dev, edges, batches, mbs, dt, dp=False)
    got = _run_dp(copy.deepcopy(base), s48.dev, edges, batches, mbs, dt, dp=True)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys() and sum(k.startswith("grad ") for k in r) > 10, i
        for k in r:
            assert torch.equal(g[k], r[k]), f"batch {i}: {k}"


def _rank_main(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), CUBLAS_WORKSPACE_CONFIG=":4096:8")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
    try:
        torch.use_deterministic_algorithms(True)
        s = _split(dev, n_questions=64)
        mbs = 2
        edges = (s.flat.max_batch_edges(mbs), s.flat.max_graph_edges())
        batches = _dp_batches(64, mbs, world)
        base = _recipe_decoder(dev)
        got = _run_dp(copy.deepcopy(base), s.dev, edges, batches, mbs, torch.float16, dp=True)
        torch.save([{k: v.cpu() for k, v in r.items()} for r in got], os.path.join(out_dir, f"rank{rank}.pt"))
        if rank == 0:
            ref = _run_dp(copy.deepcopy(base), s.dev, edges, batches, mbs, torch.float16, dp=False)
            torch.save([{k: v.cpu() for k, v in r.items()} for r in ref], os.path.join(out_dir, "one_gpu.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_keyed_ranks_equal_one_keyed_gpu():
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"{world} ranks need {world} GPUs, {torch.cuda.device_count()} visible")
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(_rank_main, args=(world, _free_port(), tmp), nprocs=world, join=True)
        ranks = [torch.load(os.path.join(tmp, f"rank{r}.pt")) for r in range(world)]
        ref = torch.load(os.path.join(tmp, "one_gpu.pt"))
    for i, r in enumerate(ref):
        for got in ranks:
            assert got[i].keys() == r.keys(), i
            for k in r:
                assert torch.equal(got[i][k], r[k]), f"batch {i}: {k}"


# ---- host reads and refusals ------------------------------------------------------------------------------------------------

def test_a_replayed_keyed_chunk_and_advance_read_nothing_on_the_host(s48):
    mbs = 2
    kw = _kw(s48, mbs, torch.float16, "cross_entropy")
    dec = _recipe_decoder()
    key = training.DropoutKey(SEED, DEV)
    tb = SplitTrainBatch(dec, s48.dev, mbs, branches=2, dropout_key=key, **kw)
    scaler = torch.amp.GradScaler("cuda")
    chunk = [np.arange(0, 2), np.arange(2, 4)]
    seen = []
    for call in range(3):  # the first call captures; the next two replay under the sync check
        svs = [_sv(q, requires_grad=False) for q in chunk]
        if call:
            torch.cuda.set_sync_debug_mode("error")
        try:
            losses = tb(chunk, svs)
            scaler.scale(losses.sum()).backward()
            key.advance_()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        seen.append(losses.detach().clone())
    assert int(key.draw) == 3
    assert not torch.equal(seen[1], seen[2]), "a new draw must draw new masks in the replayed graphs"


def test_refusals(s48):
    key = training.DropoutKey(SEED, DEV)
    qids = torch.arange(2, device=DEV)
    x = torch.randn(2 * NC, 8, device=DEV)
    with pytest.raises(ValueError, match="is on"):
        _keyed(x.cpu(), key, qids, 0.2, 0, 0)
    with pytest.raises(ValueError, match="graphs"):
        _keyed(x, key, qids[:1], 0.2, 0, 0)
    for p in (-0.1, 1.1):
        with pytest.raises(ValueError, match="must be in"):
            _keyed(x, key, qids, p, 0, 0)
    with pytest.raises(ValueError, match="site"):
        _keyed(x, key, qids, 0.2, 256, 0)
    with pytest.raises(ValueError, match="question_ids"):
        with training.keyed_dropout(key, qids.cpu(), NC):
            pass
    with pytest.raises(ValueError, match="question_ids"):
        with training.keyed_dropout(key, qids.int(), NC):
            pass
    # eval mode and no context: torch's dropout, untouched
    with training.keyed_dropout(key, qids, NC):
        assert torch.equal(training.dropout(x, 0.2, False, 0), x)
    kw = _kw(s48, 2, None, "cross_entropy")
    with pytest.raises(ValueError, match="dropout key"):
        SplitTrainStep(_recipe_decoder(), s48.dev, 2, dropout_key=type("K", (), {"device": torch.device("cpu")})(), **kw)
