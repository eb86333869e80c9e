"""Data-parallel training of a split (qagnn_b200.distributed.DataParallelSplitTrain) on the GPU.  ordered_grad_sum_ equals a
Python loop of torch._foreach_add_ bit for bit over the recipe decoder's 86 gradients, sizes 0, 1, 3 and 8193, odd-offset
views, 700 tensors (two launches), 1, 2, 33 and 64 slots, `.grad` None or zeroed, and slots holding -0.0, inf and NaN; so
does GradSlots onto a `.grad` that is None, transposed or held by the caller.  With one rank, under
torch.use_deterministic_algorithms(True) with dropout 0, two optimiser batches (the second ending in a partial
micro-batch) equal the plain SplitTrainStep loop bit for bit: every `.grad`, the BatchNorm buffers and the parameters
after optim.RAdam, in fp32, fp16 with a GradScaler and bf16, and reduce_ reads nothing on the host.  With 2, 4 and 8 ranks
(NCCL, one process per GPU; skipped when fewer than 2 GPUs are visible) the decoder's `.grad` and the parameters after RAdam
equal the one-GPU run bit for bit, a batch with fewer micro-batches than ranks included; the BatchNorm statistics are within
the fold's bar, the stand-in encoder's `.grad` within fp32 summation error and the same bits on every rank, and every rank's
parameters are the same bits.  Needs a GPU: run with -m gpu."""
import copy
import os
import socket
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import qagnn_b200
import qagnn_b200.training
from oracle import qagnn_oracle as O
from qagnn_b200 import distributed as D
from qagnn_b200 import optim
from qagnn_b200.pipeline import SplitTrainStep
from tests import helpers as Hh
from tests.test_gpu_split_train import (DT_IDS, DTYPES, N, N_CONCEPT, NC, R, SENT_DIM, T, Split, _decoder,  # noqa: F401
                                         deterministic, s48)
from tests.test_gpu_split_train import D as D_
from tests.test_data_parallel_cpu import BN_BAR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---- ordered_grad_sum_ ---------------------------------------------------------------------------------------------------

def _loop(before, slot_grads, n_valid):
    """One GPU's accumulation: .grad = slot 0 (or .grad + slot 0), then torch._foreach_add_ of every later slot."""
    acc = [s.clone() if b is None else b.clone() for b, s in zip(before, slot_grads[0])]
    if any(b is not None for b in before):
        idx = [i for i, b in enumerate(before) if b is not None]
        torch._foreach_add_([acc[i] for i in idx], [slot_grads[0][i] for i in idx])
    for j in range(1, n_valid):
        torch._foreach_add_(acc, slot_grads[j])
    return acc


def _slots(slot_grads, n_rows, offset=0):
    cols, ld = D.slot_columns([g.numel() for g in slot_grads[0]])
    buf = torch.full((n_rows * ld + offset,), float("nan"), device=DEV)  # rows past n_valid must not be read
    slots = buf[offset:].view(n_rows, ld)
    for j, row in enumerate(slot_grads):
        for c, g in zip(cols, row):
            slots[j, c:c + g.numel()] = g.reshape(-1)
    return slots


def _check(sizes, n_valid, before_kind, seed, special=False, offset=0, grad_offset=0, extra_rows=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rows = [[torch.randn(n, device=DEV, generator=g) * 10.0 ** torch.randint(-3, 4, (1,), generator=g, device=DEV).item()
             for n in sizes] for _ in range(n_valid)]
    if special:
        for j, row in enumerate(rows):
            for t in row:
                if t.numel() >= 4:
                    t[0], t[1], t[2] = -0.0, float("inf") if j % 3 == 0 else -0.0, float("nan") if j == 1 else 0.0
    before = [None] * len(sizes)
    if before_kind == "zeroed":
        before = [torch.zeros(n, device=DEV) for n in sizes]
    elif before_kind == "values":
        before = [torch.randn(n, device=DEV, generator=g) for n in sizes]
    ref = _loop(before, rows, n_valid)
    outs = []
    for b, n in zip(before, sizes):
        store = torch.full((n + grad_offset,), 7.0, device=DEV)[grad_offset:]
        if b is not None:
            store.copy_(b)
        outs.append(store)
    D.ordered_grad_sum_(outs, _slots(rows, n_valid + extra_rows, offset), n_valid, [b is not None for b in before])
    for o, r in zip(outs, ref):
        assert torch.equal(o.view(torch.int32), r.view(torch.int32))


@pytest.mark.parametrize("n_valid", [1, 2, 33, 64])
@pytest.mark.parametrize("before", ["none", "zeroed", "values"])
def test_sizes_0_1_3_8193_equal_the_foreach_loop(n_valid, before):
    _check([0, 1, 3, 8193, 5, 16384], n_valid, before, seed=n_valid)


@pytest.mark.parametrize("before", ["none", "zeroed"])
def test_negative_zero_inf_and_nan_keep_the_loops_bits(before):
    _check([4, 7, 8193], 5, before, seed=2, special=True)


@pytest.mark.parametrize("offset,grad_offset", [(1, 0), (0, 1), (3, 5)])
def test_odd_offset_views_take_the_scalar_path(offset, grad_offset):
    _check([1, 3, 8193, 20000], 33, "values", seed=3, offset=offset, grad_offset=grad_offset)


def test_700_tensors_take_two_launches():
    lib = qagnn_b200._lib.load()
    before = lib.qagnn_launch_count()
    _check([(i * 37) % 300 + 1 for i in range(700)], 3, "none", seed=4, extra_rows=0)
    assert lib.qagnn_launch_count() - before == 2


def test_the_recipe_decoders_86_gradients():
    dec = qagnn_b200.QAGNN(None, 5, 4, 38, 1024, 100, 200, 1024, 2, 200, 0, 0.2, 0.2, 0.2,
                           pretrained_concept_emb=torch.zeros(100, 1024), freeze_ent_emb=True)
    sizes = [p.numel() for p in dec.parameters() if p.requires_grad]
    assert len(sizes) == 86 and sum(sizes) == 2845025
    for n_valid in (2, 32):
        _check(sizes, n_valid, "none", seed=n_valid)


def test_refusals():
    x = torch.zeros(4, device=DEV)
    with pytest.raises(ValueError, match="n_valid"):
        D.ordered_grad_sum_([x], torch.zeros(2, 4, device=DEV), 3, False)
    with pytest.raises(ValueError, match="slot rows"):
        D.ordered_grad_sum_([x, x], torch.zeros(2, 4, device=DEV), 1, False)
    with pytest.raises(ValueError, match="contiguous fp32"):
        D.ordered_grad_sum_([x.half()], torch.zeros(2, 4, device=DEV), 1, False)
    with pytest.raises(ValueError, match="init_from_grad"):
        D.ordered_grad_sum_([x], torch.zeros(2, 4, device=DEV), 1, [True, False])


def test_grad_slots_sum_onto_none_a_transposed_grad_and_a_held_one():
    """GradSlots: rows written by copy_row_ (None as zeros) and summed by sum_ equal the foreach loop bit for bit, and `.grad`
    becomes a view of the helper's own buffer for a start of None or a non-contiguous one, the start itself otherwise."""
    g = torch.Generator(device=DEV).manual_seed(6)
    params = [torch.nn.Parameter(torch.empty(s, device=DEV)) for s in ((3, 5), (4, 6), (7,))]
    rows = [[torch.randn(p.shape, device=DEV, generator=g) for p in params] for _ in range(3)]
    rows[1][0] = None
    ld = D.slot_columns([p.numel() for p in params])[1]
    gs = D.GradSlots(params, torch.full((4, ld), float("nan"), device=DEV), torch.empty(ld, device=DEV))
    for j, row in enumerate(rows):
        gs.copy_row_(j, row)
    held = torch.randn(7, device=DEV, generator=g)
    starts = [None, torch.randn(6, 4, device=DEV, generator=g).t(), held]
    ref = _loop([None if s is None else s.clone() for s in starts],
                [[torch.zeros(p.shape, device=DEV) if t is None else t for p, t in zip(params, row)] for row in rows], 3)
    gs.sum_(starts, 3)
    for p, r in zip(params, ref):
        assert torch.equal(p.grad.view(torch.int32), r.view(torch.int32))
    assert params[0].grad.data_ptr() == gs.own[0].data_ptr() and params[1].grad.data_ptr() == gs.own[1].data_ptr()
    assert params[1].grad.is_contiguous() and params[2].grad is held


# ---- the training loop ---------------------------------------------------------------------------------------------------

def _autocast(dt):
    return torch.autocast("cuda", dtype=dt, cache_enabled=False) if dt is not None else torch.autocast("cuda", enabled=False)


def _encoder(dev, seed=5):
    torch.manual_seed(seed)
    return torch.nn.Linear(SENT_DIM, SENT_DIM).to(dev)


def _inputs(qids, dev):
    """The stand-in encoder's input for a micro-batch: a function of its question ids alone."""
    g = torch.Generator(device=dev).manual_seed(int(np.asarray(qids)[0]) * 1000 + len(qids))
    return torch.randn(len(qids) * NC, SENT_DIM, device=dev, generator=g)


def _loop_state(dec, enc):
    r = {f"grad {k}": p.grad.clone() for k, p in dec.named_parameters() if p.grad is not None}
    r.update({f"enc grad {k}": p.grad.clone() for k, p in enc.named_parameters() if p.grad is not None})
    r.update({f"buffer {k}": v.detach().clone() for k, v in dec.named_buffers() if "running" in k or "num_batches" in k})
    return r


def _params_state(dec, enc):
    return {f"param {k}": p.detach().clone() for k, p in list(dec.named_parameters()) + [("enc." + k, p) for k, p in
                                                                                      enc.named_parameters()]}


def _run(dec, enc, split, batches, mbs, dt, dp_kw=None, sync_check=False, enc_lr=1e-3, unfreeze_at=None):
    """The recipe's loop over `batches` on one GPU (dp_kw None) or through DataParallelSplitTrain; returns per batch the
    state after the gradient sum and the parameters after the step.  With enc_lr 0 the encoder keeps its weights and only
    the decoder's gradients are clipped, so that the decoder's trajectory depends on nothing the ranks sum in another order.
    With unfreeze_at, the encoder is frozen before the loop is built and unfrozen before batch `unfreeze_at`, as the
    recipe's freeze_net / unfreeze_net do."""
    dev = split.device
    if unfreeze_at is not None:
        enc.requires_grad_(False)
    K, M = split_edges(split, mbs)
    step = SplitTrainStep(dec, split, mbs, edge_capacity=K, max_edges=M, autocast_dtype=dt)
    params = list(dec.parameters()) + (list(enc.parameters()) if enc_lr else [])
    opt = optim.RAdam([{"params": [p for p in dec.parameters() if p.requires_grad]},
                       {"params": list(enc.parameters()), "lr": enc_lr}], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    dp = None if dp_kw is None else D.DataParallelSplitTrain(step, split, batch_size=dp_kw["bs"], micro_batch_size=mbs,
                                                             other_params=enc.parameters(), group=dp_kw.get("group"))
    rec = []
    for b, batch in enumerate(batches):
        if b == unfreeze_at:
            enc.requires_grad_(True)
        opt.zero_grad()
        micro = [batch[a:a + mbs] for a in range(0, len(batch), mbs)] if dp is None else dp.micro_batches(batch)
        for q in micro:
            with _autocast(dt):
                sv = enc(_inputs(q, dev))
            if dp is None:
                if len(q) == mbs:
                    loss = step(q, sv)
                else:
                    with _autocast(dt):
                        logits, _ = dec(sv, *split.batch(q, K))
                        loss = qagnn_b200.training.answer_loss(logits, split.labels[torch.from_numpy(q).to(dev)], NC)
                w = loss * len(q) / len(batch)
                (scaler.scale(w) if scaler is not None else w).backward()
            else:
                with dp.micro_step():
                    w = dp.loss(q, sv) * len(q) / len(batch)
                    (scaler.scale(w) if scaler is not None else w).backward()
        if dp is not None:
            if sync_check:
                torch.cuda.set_sync_debug_mode("error")
            try:
                dp.reduce_(len(batch))
            finally:
                torch.cuda.set_sync_debug_mode("default")
        r = _loop_state(dec, enc)
        if scaler is not None:
            scaler.unscale_(opt)
        optim.clip_grad_norm_([p for p in params if p.grad is not None], 1.0)
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        r.update(_params_state(dec, enc))
        rec.append(r)
    return rec


_EDGES = {}


def split_edges(split, mbs):
    return _EDGES[id(split)][mbs]


def _register(split_obj):
    _EDGES[id(split_obj.dev)] = {m: (split_obj.flat.max_batch_edges(m), split_obj.flat.max_graph_edges()) for m in (1, 2, 8)}
    return split_obj.dev


@pytest.mark.parametrize("mbs", [2, 8])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_one_rank_equals_the_one_gpu_loop_bit_for_bit(s48, deterministic, dt, mbs):
    split = _register(s48)
    order = np.random.default_rng(mbs).permutation(s48.Q)
    bs = 3 * mbs
    batches = [order[:bs], order[bs:bs + 2 * mbs + 1]]  # the second ends in a micro-batch of one question
    base = _decoder()
    ref = _run(copy.deepcopy(base), _encoder(DEV), split, batches, mbs, dt)
    got = _run(copy.deepcopy(base), _encoder(DEV), split, batches, mbs, dt, dp_kw={"bs": bs}, sync_check=True)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys(), (i, sorted(set(g) ^ set(r)))
        assert sum(k.startswith("grad ") for k in r) > 10
        for k in r:
            assert g[k].dtype == r[k].dtype and torch.equal(g[k], r[k]), f"batch {i}: {k}"


# ---- several ranks -------------------------------------------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _split(dev, n_questions=48, seed=51):
    """test_gpu_split_train.Split on `dev`."""
    s = Split.__new__(Split)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "s.graph.adj.pk")
        qagnn_b200.data.synth_adj_pickle(path, n_questions * NC, seed=seed)
        cids, ntypes, scores, lens, flat = qagnn_b200.data.load_flat_adj_cache(path, N, NC)
    s.flat = qagnn_b200.data.FlatAdjCache(np.array(flat.src), np.array(flat.tgt), np.array(flat.etype),
                                          np.array(flat.graph_ptr), NC, N)
    cids = torch.where(cids > 0, cids % N_CONCEPT + 1, 0)
    s.labels = torch.from_numpy(np.random.default_rng(seed).integers(0, NC, n_questions))
    s.host = (cids, ntypes, scores, lens)
    s.dev = qagnn_b200.data.DeviceSplit(s.flat, *s.host, dev, T, R, labels=s.labels)
    s.Q = n_questions
    return s


def _decoder_on(dev, seed=8):
    """test_gpu_split_train._decoder (dropout 0) on `dev`."""
    torch.manual_seed(seed)
    dec = qagnn_b200.QAGNN(None, 2, T, R, SENT_DIM, N_CONCEPT, D_, 32, 2, D_, 1, 0.0, 0.0, 0.0)
    dec.gnn.load_state_dict(O.random_state_dict(2, D_, T, R, "prod", seed=seed))
    for m in dec.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return dec.to(dev).train()


def _rank_main(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), CUBLAS_WORKSPACE_CONFIG=":4096:8")
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
    try:
        torch.use_deterministic_algorithms(True)
        split = _register(_split(dev, n_questions=128))
        mbs, bs = 2, 2 * world * 2  # M = 2 W micro-batches of a full batch
        order = np.random.default_rng(7).permutation(128)
        # a full batch with the encoder frozen, then unfrozen: a full batch, 5 questions (M = 3, a partial micro-batch on
        # some rank), 2 questions (M = 1 < W) and a full batch
        sizes, batches, at = [bs, bs, 2 * mbs + 1, mbs, bs], [], 0
        for n in sizes:
            batches.append(order[at:at + n])
            at += n
        base = _decoder_on(dev)
        got = _run(copy.deepcopy(base), _encoder(dev), split, batches, mbs, torch.float16, dp_kw={"bs": bs}, enc_lr=0.0,
                   unfreeze_at=1)
        torch.save([{k: v.cpu() for k, v in r.items()} for r in got], os.path.join(out_dir, f"rank{rank}.pt"))
        if rank == 0:
            ref = _run(copy.deepcopy(base), _encoder(dev), split, batches, mbs, torch.float16, enc_lr=0.0, unfreeze_at=1)
            torch.save([{k: v.cpu() for k, v in r.items()} for r in ref], os.path.join(out_dir, "one_gpu.pt"))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_several_ranks_equal_one_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"{world} ranks need {world} GPUs, {torch.cuda.device_count()} visible")
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(_rank_main, args=(world, _free_port(), tmp), nprocs=world, join=True)
        ranks = [torch.load(os.path.join(tmp, f"rank{r}.pt")) for r in range(world)]
        ref = torch.load(os.path.join(tmp, "one_gpu.pt"))
    for i, r in enumerate(ref):
        assert all(got[i].keys() == r.keys() for got in ranks), (i, sorted(set(ranks[0][i]) ^ set(r)))  # None as one GPU
        assert (i == 0) != any(k.startswith("enc grad ") for k in r)  # frozen for the first batch only
        for k in r:
            what = f"world {world}, batch {i}: {k}"
            for got in ranks:  # every rank holds the same bits
                assert torch.equal(got[i][k], ranks[0][i][k]), what
            g = ranks[0][i][k]
            if k.startswith("buffer ") and "num_batches" not in k:
                scale = float(r[k].abs().max())
                assert float((g - r[k]).abs().max()) <= BN_BAR * scale, what
            elif k.startswith("enc grad "):
                Hh.assert_close(g, r[k], what, atol=1e-5 * float(r[k].abs().max()), rtol=1e-5)
            else:
                assert torch.equal(g, r[k]), what
