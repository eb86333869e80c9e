"""Data-parallel training of a split on the CPU: the block partition of an optimiser batch's micro-batches over the ranks
(DataParallelSplitTrain.micro_batches), the BatchNorm fold (distributed.fold_running_stats) against a sequential fp64 EMA and
against nn.BatchNorm1d stepped micro-batch by micro-batch (BatchNormFold over mixed widths and momenta included), the
constructor's refusals, the slot layout, and the ordered-sum kernel's SASS (no floating-point atomics, no spills)."""
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

from qagnn_b200 import distributed as D

# The fold is exact in exact arithmetic; one process rounds every update to fp32 instead (each update's error is at most a
# few fp32 ulps of the statistic and decays by a = 0.9 per later update, so it sums to about 20 ulps), and the fold rounds once.
# The bar, relative to the largest magnitude of the buffer: 64 fp32 ulps.
BN_BAR = 64 * 2.0 ** -24


def _fake_step(batch_size, momentum=0.1):
    dec = torch.nn.Sequential(torch.nn.Linear(3, 4), torch.nn.BatchNorm1d(4, momentum=momentum))
    split = types.SimpleNamespace(device=torch.device("cpu"))
    return types.SimpleNamespace(batch_size=batch_size, split=split, decoder=dec)


@pytest.fixture
def world(monkeypatch):
    """Pretends torch.distributed is initialised with `set(W, r)`."""
    state = {"W": 1, "r": 0}
    monkeypatch.setattr(D.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(D.dist, "get_world_size", lambda group=None: state["W"])
    monkeypatch.setattr(D.dist, "get_rank", lambda group=None: state["r"])

    def set_(W, r=0):
        state.update(W=W, r=r)
    return set_


@pytest.mark.parametrize("W", [1, 2, 3, 8])
def test_every_rank_takes_its_contiguous_block_in_order(world, W):
    """Batches of M = 1 ... 70 micro-batches (odd M ending in a partial one) under a loop built for 70 full ones."""
    mbs = 2
    dps = []
    for r in range(W):
        world(W, r)
        step = _fake_step(mbs)
        dps.append(D.DataParallelSplitTrain(step, step.split, batch_size=70 * mbs, micro_batch_size=mbs))
    for M in range(1, 71):
        n = M * mbs - (M % 2)
        batch = np.arange(1000, 1000 + n)
        m = -(-M // W)
        got, empty = [], 0
        for r, dp in enumerate(dps):
            blocks = dp.micro_batches(batch)
            dp._batch = None  # the partition alone: no micro-step, no reduce_
            assert len(blocks) == max(0, min(M, (r + 1) * m) - r * m) <= m
            empty += not blocks
            got += [b.tolist() for b in blocks]
        assert got == [batch[a:a + mbs].tolist() for a in range(0, n, mbs)], (M, W)
        assert empty == W - -(-M // m)  # the ranks past the last block, and only those, have none


def test_a_rank_without_micro_batches_only_in_a_short_batch(world):
    world(2, 1)
    step = _fake_step(2)
    dp = D.DataParallelSplitTrain(step, step.split, batch_size=8, micro_batch_size=2)
    assert [b.tolist() for b in dp.micro_batches(np.arange(8))] == [[4, 5], [6, 7]]
    dp._batch = None
    assert dp.micro_batches(np.arange(2)) == []  # M = 1 < W


def _refuses(world, W, bs, mbs, step_bs=None, momentum=0.1, match=""):
    world(W, 0)
    step = _fake_step(mbs if step_bs is None else step_bs, momentum)
    with pytest.raises(ValueError, match=match):
        D.DataParallelSplitTrain(step, step.split, batch_size=bs, micro_batch_size=mbs)


def test_refusals(world):
    _refuses(world, 1, 8, 2, momentum=None, match="momentum=None")
    _refuses(world, 4, 6, 2, match="leaves rank 3 of 4 none")                 # M = 3 < W = 4
    _refuses(world, 4, 10, 2, match="leaves rank 3 of 4 none")                # M = 5, m = 2: rank 3 starts past M
    _refuses(world, 3, 5, 2, match="only the partial one")                    # rank 2's block is the 1-question micro-batch
    _refuses(world, 1, 8, 2, step_bs=4, match="step runs 4 questions")        # the step's batch size is not the loop's
    _refuses(world, 1, 1, 2, match="batch_size 1 < micro_batch_size 2")
    world(2, 0)
    step = _fake_step(2)
    D.DataParallelSplitTrain(step, step.split, batch_size=8, micro_batch_size=2)  # M = 4, W = 2 is fine


def test_slot_columns_start_on_16_byte_boundaries():
    cols, ld = D.slot_columns([1, 3, 8193, 0, 4])
    assert cols == [0, 4, 8, 8204, 8204] and ld == 8208
    assert D.slot_columns([]) == ([], 4)


# ---- the BatchNorm fold --------------------------------------------------------------------------------------------------

def _ema(start, xs, momentum):
    r = start.clone()
    for x in xs:
        r = (1 - momentum) * r + momentum * x
    return r


@pytest.mark.parametrize("counts", [[3, 0, 5], [1, 1], [0, 4, 0, 2, 7, 1, 1, 3], [10]])
def test_the_fold_is_the_sequential_fp64_ema(counts):
    g = torch.Generator().manual_seed(sum(counts))
    L = 17
    start = torch.randn(L, dtype=torch.float64, generator=g)
    xs = [[torch.randn(L, dtype=torch.float64, generator=g) * 3 + 1 for _ in range(n)] for n in counts]
    ends = torch.stack([_ema(start, x, 0.1) for x in xs])
    n = torch.tensor(counts, dtype=torch.float64)[:, None].expand(-1, L)
    got = D.fold_running_stats(start, ends, n, 0.1)
    ref = _ema(start, [x for r in xs for x in r], 0.1)
    assert torch.allclose(got, ref, rtol=0, atol=1e-13 * float(ref.abs().max()))


@pytest.mark.parametrize("W,micro", [(2, 4), (3, 7), (8, 32)])
def test_the_fold_of_batchnorm1d_is_within_the_bar(W, micro):
    """nn.BatchNorm1d(momentum=0.1) stepped micro-batch by micro-batch on one process against W copies, each stepping its
    block of micro-batches (each micro-batch makes k = 3 updates, as the shared edge encoder does), folded."""
    torch.manual_seed(W)
    C = 200
    data = [[torch.randn(40, C) * 5 + 3 for _ in range(3)] for _ in range(micro)]
    one = torch.nn.BatchNorm1d(C, momentum=0.1).train()
    one.running_mean.normal_(0, 2)
    one.running_var.uniform_(0.5, 4)
    start = {k: v.clone() for k, v in one.state_dict().items()}
    ranks = [torch.nn.BatchNorm1d(C, momentum=0.1).train() for _ in range(W)]
    for bn in ranks:
        bn.load_state_dict(start)
    for x in (x for mb in data for x in mb):
        one(x)
    for r, bn in enumerate(ranks):
        lo, hi = D.shard_bounds(micro, r, W)
        for mb in data[lo:hi]:
            for x in mb:
                bn(x)
    for name in ("running_mean", "running_var"):
        counts = torch.tensor([float(bn.num_batches_tracked - start["num_batches_tracked"]) for bn in ranks],
                              dtype=torch.float64)[:, None].expand(-1, C)
        folded = D.fold_running_stats(start[name], torch.stack([getattr(bn, name) for bn in ranks]), counts, 0.1).float()
        ref = getattr(one, name)
        assert float((folded - ref).abs().max()) <= BN_BAR * float(ref.abs().max()), name
    assert int(one.num_batches_tracked) == int(start["num_batches_tracked"]) + sum(
        int(bn.num_batches_tracked - start["num_batches_tracked"]) for bn in ranks)


@pytest.mark.parametrize("fp64", [False, True], ids=["rows", "gathered"])
@pytest.mark.parametrize("W,micro", [(2, 4), (3, 7), (8, 32)])
def test_the_fold_of_batchnorms_of_other_widths_and_momenta_is_within_the_bar(W, micro, fp64):
    """BatchNormFold over two BatchNorm1d of widths 200 and 48 and momenta 0.1 and 0.3, which a micro-batch updates 3 times and
    once: one process steps them micro-batch by micro-batch, W copies each step their block, and the fold of the copies'
    statistics (fp32 rows with int64 counts as SplitTrainBatch holds them, or the fp64 block DataParallelSplitTrain
    gathers) is within the bar of the one process, its num_batches_tracked equal."""
    torch.manual_seed(W)

    def make():
        return torch.nn.ModuleList([torch.nn.BatchNorm1d(200, momentum=0.1), torch.nn.BatchNorm1d(48, momentum=0.3)]).train()

    data = [([torch.randn(40, 200) * 5 + 3 for _ in range(3)], [torch.randn(40, 48) * 2 - 1]) for _ in range(micro)]
    one = make()
    for bn in one:
        bn.running_mean.normal_(0, 2)
        bn.running_var.uniform_(0.5, 4)
    start = {k: v.clone() for k, v in one.state_dict().items()}
    ranks = [make() for _ in range(W)]
    for m in ranks:
        m.load_state_dict(start)

    def step(m, micro_batches):
        for mb in micro_batches:
            for bn, xs in zip(m, mb):
                for x in xs:
                    bn(x)
    step(one, data)
    for r, m in enumerate(ranks):
        lo, hi = D.shard_bounds(micro, r, W)
        step(m, data[lo:hi])
    folded = make()
    folded.load_state_dict(start)
    fold = D.BatchNormFold(folded, "test", "ranks")
    ends = [D.BatchNormFold(m, "test", "ranks").read() for m in ranks]
    stats, counts = torch.stack([s for s, _ in ends]), torch.stack([c for _, c in ends])
    fold.fold_(fold.read(), (stats.double(), counts.double()) if fp64 else (stats, counts))
    for got, ref in zip(folded, one):
        for name in ("running_mean", "running_var"):
            a, b = getattr(got, name), getattr(ref, name)
            assert a.dtype == torch.float32
            assert float((a - b).abs().max()) <= BN_BAR * float(b.abs().max()), name
        assert torch.equal(got.num_batches_tracked, ref.num_batches_tracked)
    assert [int(bn.num_batches_tracked) for bn in folded] == [3 * micro, micro]


# ---- the kernel ----------------------------------------------------------------------------------------------------------

def _tool(name):
    for cand in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("no nvcc / cuobjdump")
    src = os.path.join(os.path.dirname(D.__file__), "csrc", "grad_reduce.cu")
    obj = str(tmp_path_factory.mktemp("grad_reduce") / "grad_reduce.o")
    r = subprocess.run([nvcc, "-c", src, "-o", obj, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xcompiler", "-fPIC", "-Xptxas", "-v"], capture_output=True, text=True, check=True)
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def test_the_kernel_does_not_spill(compiled):
    report, _ = compiled
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and all(a == "0" and b == "0" for a, b in spills)


def test_the_kernel_has_no_atomics_and_reads_float4(compiled):
    _, sass = compiled
    assert "ordered_grad_sum_kernel" in sass
    ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?P\d+\s+)?([A-Z][A-Z0-9_.]*)", sass)
    assert ops
    assert not [op for op in ops if op.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG", "ATOMS")]
    assert any(op.startswith("LDG.E.EF.128") or op.startswith("LDG.E.128") for op in ops), sorted(set(ops))


# ---- several ranks on the CPU (gloo): the encoder's gradients and the BatchNorm fold --------------------------------------

F_ = 6


class _CPUStep:
    """A stand-in for SplitTrainStep on the CPU: its decoder is one BatchNorm1d without trainable parameters, so the ranks
    exchange no decoder gradient; the loss is a function of sent_vecs only.  It "captures" on its first call."""

    def __init__(self, mbs):
        self.batch_size = mbs
        self.split = types.SimpleNamespace(device=torch.device("cpu"))
        self.decoder = torch.nn.Sequential(torch.nn.BatchNorm1d(F_, momentum=0.1)).train()
        self.decoder.requires_grad_(False)
        self._fwd, self._owned = None, []
        self._anchor = torch.zeros((), requires_grad=True)  # as SplitTrainStep's: backward() works with a frozen encoder

    def __call__(self, qids, sent_vecs):
        self._fwd = True
        return (self.decoder(sent_vecs) * sent_vecs).square().mean() + 0 * self._anchor


def _enc_inputs(q):
    g = torch.Generator().manual_seed(int(q[0]) * 100 + len(q))
    return torch.randn(len(q) * 5, F_, generator=g) * 3 + 1


def _schedule(bs):
    """Batch sizes and the encoder's requires-grad pattern before each batch: frozen at construction (freeze_net before the
    loop), unfrozen after the first batch (unfreeze_net), a short batch with fewer micro-batches than ranks, and the weight
    frozen again (a refreeze) for the last one."""
    return [(bs, (False, False)), (bs, (True, True)), (2, (True, True)), (bs - 2, (True, True)), (bs, (False, True))]


def _cpu_loop(world, dp_on):
    bs = 4 * world  # M = 2 W micro-batches of 2 questions
    torch.manual_seed(0)
    enc = torch.nn.Linear(F_, F_)
    step = _CPUStep(2)
    for p in enc.parameters():
        p.requires_grad_(False)
    dp = D.DataParallelSplitTrain(step, step.split, bs, 2, other_params=enc.parameters()) if dp_on else None
    order, at, rec = np.arange(100), 0, []
    for n, pattern in _schedule(bs):
        for p, t in zip(enc.parameters(), pattern):
            p.requires_grad_(t)
            p.grad = None
        batch = order[at:at + n]
        at += n
        micro = dp.micro_batches(batch) if dp_on else [batch[a:a + 2] for a in range(0, n, 2)]
        for q in micro:
            sv = enc(_enc_inputs(q))
            if dp_on:
                with dp.micro_step():
                    (dp.loss(q, sv) * len(q) / n).backward()
            else:
                (step(q, sv) * len(q) / n).backward()
        if dp_on:
            dp.reduce_(n)
        rec.append({"grads": [None if p.grad is None else p.grad.clone() for p in enc.parameters()],
                    "bn": {k: v.clone() for k, v in step.decoder.state_dict().items()}})
        with torch.no_grad():  # a plain SGD step on what requires grad and has a gradient, as every rank takes it
            for p in enc.parameters():
                if p.grad is not None:
                    p -= 0.1 * p.grad
    return rec


def _cpu_rank(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.save(_cpu_loop(world, True), os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_the_encoder_gradients_follow_freezing_and_unfreezing_across_ranks(world, tmp_path):
    """Built with the encoder frozen and unfrozen after the first batch, the ranks sum the encoder's gradients from then on:
    the same bits on every rank, within fp32 summation error of one process, and `.grad` None wherever one process leaves
    it None (the frozen batch, the refrozen weight).  The BatchNorm statistics are within the fold's bar."""
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_cpu_rank, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    ranks = [torch.load(str(tmp_path / f"rank{r}.pt")) for r in range(world)]
    ref = _cpu_loop(world, False)
    for b, r in enumerate(ref):
        for j, g in enumerate(r["grads"]):
            got = [rk[b]["grads"][j] for rk in ranks]
            if g is None:
                assert all(x is None for x in got), (b, j)
                continue
            assert all(x is not None and torch.equal(x, got[0]) for x in got), (b, j)
            assert torch.allclose(got[0], g, rtol=1e-5, atol=1e-6 * float(g.abs().max())), (b, j)
        for k, v in r["bn"].items():
            for rk in ranks:
                if "num_batches" in k:
                    assert torch.equal(rk[b]["bn"][k], v), (b, k)
                else:
                    assert float((rk[b]["bn"][k] - v).abs().max()) <= BN_BAR * float(v.abs().max()), (b, k)
    assert ref[0]["grads"] == [None, None] and ref[-1]["grads"][0] is None and ref[-1]["grads"][1] is not None
