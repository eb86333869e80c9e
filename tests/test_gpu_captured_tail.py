"""optim.CapturedTail against the eager tail it replaces, on the same GPU: `scaler.unscale_; optim.clip_grad_norm_;
scheduler.step; scaler.step; scaler.update` with optim.RAdam / optim.AdamW and torch's GradScaler, in the reference's order.
After every call, p, exp_avg, exp_avg_sq, step, .grad, the returned norm, the scaler's scale and growth tracker and every
group's lr equal the eager tail's bit for bit: both rules and their flags, weight decay, four groups, fp32 and fp16 with a
scaler, clipping on, off and inactive, three schedules, inf and NaN gradients, scale growth, sizes 0, 1, 3 and 8193,
odd-offset views, 700 tensors in 20 groups, 1100 steps, a state_dict round trip, eager steps in between, recaptures on
freezing, a call under sync-debug "error", and the recipe's loop through SplitTrainBatch and DataParallelSplitTrain.
Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

from qagnn_b200 import distributed as D
from qagnn_b200 import optim
from qagnn_b200.pipeline import SplitTrainBatch, train_chunks
from tests.test_gpu_split_train import NC, SENT_DIM, _decoder, deterministic, s48  # noqa: F401
from tests.test_gpu_split_train_batch import _sv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SCHEDULES = {  # the reference's --lr_schedule values as LambdaLR factors of the step count
    "fixed": lambda s: 1.0,
    "warmup_constant": lambda s: min(1.0, s / 7.5),
    "warmup_linear": lambda s: s / 7.5 if s < 7.5 else max(0.0, (60 - s) / (60 - 7.5)),
}


def _params(sizes, seed, offset=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if not offset:
        return [torch.randn(n, device=DEV, generator=g).requires_grad_() for n in sizes]
    base = torch.randn(sum(sizes) + 2 * len(sizes) + 1, device=DEV, generator=g)
    out, at = [], 1
    for n in sizes:
        out.append(base[at:at + n].detach().requires_grad_())  # starts at an odd float offset
        at += n + 2
    return out


def _opt(rule, params, n_groups, flag, wd):
    groups = [{"params": params[i::n_groups], "lr": 1e-3 * (1 + i), "weight_decay": wd if i % 2 == 0 else 0.0}
              for i in range(n_groups)]
    groups = [gr for gr in groups if gr["params"]]
    if rule == "radam":
        return optim.RAdam(groups, lr=1e-3, degenerated_to_sgd=flag)
    return optim.AdamW(groups, lr=1e-3, correct_bias=flag)


class Side:
    """One copy of the parameters, its optimiser, scaler and scheduler, stepped by the eager or the captured tail."""

    def __init__(self, sizes, rule, n_groups=4, flag=True, wd=0.01, fp16=False, growth_interval=2000, schedule=None,
                 max_norm=1.0, offset=False, captured=False):
        self.params = _params(sizes, 1, offset)
        self.opt = _opt(rule, self.params, n_groups, flag, wd)
        self.scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12, growth_interval=growth_interval) if fp16 else None
        if self.scaler is not None:
            self.scaler.scale(torch.ones((), device=DEV))  # creates the scale tensors
        self.sched = None if schedule is None else torch.optim.lr_scheduler.LambdaLR(self.opt, SCHEDULES[schedule])
        self.max_norm = max_norm
        self.tail = optim.CapturedTail(self.opt, scaler=self.scaler, scheduler=self.sched, max_grad_norm=max_norm,
                                       clip_parameters=self.params) if captured else None

    def set_grads(self, step, special=None, live=None):
        g = torch.Generator(device=DEV).manual_seed(1000 + step)
        scale = self.scaler._scale if self.scaler is not None else None
        for i, p in enumerate(self.params):
            if live is not None and not live[i]:
                p.grad = None
                continue
            x = torch.randn(p.shape, device=DEV, generator=g) * 0.3
            if scale is not None:
                x = x * scale
            if special is not None and i == 1 and p.numel():
                x.view(-1)[0] = special
            if p.grad is None:
                p.grad = torch.empty_like(p)
            p.grad.copy_(x)

    def run(self):
        if self.tail is not None:
            return self.tail()
        norm = None
        if self.max_norm > 0:
            if self.scaler is not None:
                self.scaler.unscale_(self.opt)
            norm = optim.clip_grad_norm_([p for p in self.params if p.grad is not None], self.max_norm)
        if self.sched is not None:
            self.sched.step()
        if self.scaler is not None:
            self.scaler.step(self.opt)
            self.scaler.update()
        else:
            self.opt.step()
        return norm

    def state(self, norm):
        r = {"norm": norm}
        for i, p in enumerate(self.params):
            r[f"p{i}"] = p.detach().clone()
            r[f"g{i}"] = None if p.grad is None else p.grad.clone()
            st = self.opt.state.get(p, {})
            for k in ("exp_avg", "exp_avg_sq", "step"):
                r[f"{k}{i}"] = st[k].clone() if k in st else None
        if self.scaler is not None:
            r["scale"] = self.scaler._scale.clone()
            r["tracker"] = self.scaler._growth_tracker.clone()
        r["lr"] = [g["lr"] for g in self.opt.param_groups]
        return r


def _same(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, torch.Tensor) or isinstance(y, torch.Tensor):
            assert x is not None and y is not None, (what, k)
            assert x.dtype == y.dtype and x.shape == y.shape, (what, k)
            assert torch.equal(x.view(-1).view(torch.int32 if x.dtype == torch.float32 else x.dtype),
                               y.view(-1).view(torch.int32 if y.dtype == torch.float32 else y.dtype)), (what, k)
        else:
            assert x == y, (what, k)


def _check(sizes, rule, steps=4, specials=None, live=None, between=None, **kw):
    ref, got = Side(sizes, rule, **kw), Side(sizes, rule, captured=True, **kw)
    for s in range(steps):
        sp = (specials or {}).get(s)
        lv = live(s) if live else None
        for side in (ref, got):
            side.set_grads(s, sp, lv)
        _same(ref.state(ref.run()), got.state(got.run()), f"step {s}")
        if between is not None:
            between(s, ref, got)
    return ref, got


SIZES = [3000, 1, 8193, 64, 3, 0, 20000, 17]


@pytest.mark.parametrize("rule", ["radam", "adamw"])
@pytest.mark.parametrize("flag", [True, False])
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_rules_flags_and_decay(rule, flag, wd):
    _check(SIZES, rule, steps=8, flag=flag, wd=wd, fp16=True)


@pytest.mark.parametrize("rule", ["radam", "adamw"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("max_norm", [1e6, 0.05, 0.0])
def test_precision_and_clipping(rule, fp16, max_norm):
    ref, got = _check(SIZES, rule, steps=6, fp16=fp16, max_norm=max_norm)
    assert got.tail.captures == 1


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
def test_schedules_over_60_steps(schedule):
    _check([500, 7, 9000], "radam", steps=60, fp16=True, schedule=schedule)


@pytest.mark.parametrize("max_norm", [1.0, 0.0])
@pytest.mark.parametrize("rule", ["radam", "adamw"])
def test_inf_and_nan_skip_the_step_and_back_off(rule, max_norm):
    ref, got = _check(SIZES, rule, steps=7, specials={1: float("inf"), 3: float("nan"), 4: float("-inf")}, fp16=True,
                      max_norm=max_norm, growth_interval=3)
    assert got.scaler.get_scale() < 2.0 ** 12  # backed off


def test_the_scale_grows():
    ref, got = _check([100, 5], "radam", steps=7, fp16=True, growth_interval=3)
    assert got.scaler.get_scale() == 2.0 ** 14


def test_odd_offset_views():
    _check([5, 8193, 3, 1, 4099], "adamw", steps=4, fp16=True, offset=True)


def test_700_tensors_in_20_groups_split_the_launch():
    sizes = [(i * 37) % 300 + (8193 if i % 97 == 0 else 0) for i in range(700)]
    _check(sizes, "radam", steps=3, n_groups=20, fp16=True)


def test_1100_steps_cross_the_table_regrowth():
    ref, got = _check([40, 3], "adamw", steps=1100, fp16=False, max_norm=0.5)
    assert got.opt._host_steps == 1100 and got.tail.captures == 1


def test_state_dict_round_trip_and_eager_steps_between_replays():
    def between(s, ref, got):
        if s == 2:  # an eager step in both
            for side in (ref, got):
                side.set_grads(100 + s)
                side.opt.step()
        if s == 4:
            for side in (ref, got):
                side.opt.load_state_dict(copy.deepcopy(side.opt.state_dict()))
    _, got = _check(SIZES, "radam", steps=8, between=between, fp16=True)
    assert got.tail.captures == 2  # the loaded state lives at new addresses


def test_freezing_recaptures_and_nothing_else_does():
    frozen = lambda s: [not (2 <= s < 5 and i < 3) and not (s >= 7 and i < 3) for i in range(len(SIZES))]  # noqa: E731
    ref, got = _check(SIZES, "radam", steps=9, live=frozen, fp16=True)
    assert got.tail.captures == 4  # the first call, frozen at 2, unfrozen at 5 (new .grad tensors), frozen at 7


def test_a_call_reads_nothing_on_the_host():
    side = Side(SIZES, "radam", fp16=True, captured=True)
    side.set_grads(0)
    side.run()
    side.set_grads(1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        side.run()
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_refusals():
    p = torch.zeros(4, device=DEV, requires_grad=True)
    with pytest.raises(ValueError, match="eager tail"):
        optim.CapturedTail(torch.optim.SGD([p], lr=0.1))
    with pytest.raises(ValueError, match="eager tail"):
        optim.CapturedTail(torch.optim.Adam([p], lr=0.1))
    opt = optim.RAdam([p])
    scaler = torch.amp.GradScaler("cuda")
    (scaler.scale(p.sum())).backward()
    scaler.unscale_(opt)
    with pytest.raises(RuntimeError, match="unscale_"):
        optim.CapturedTail(opt, scaler=scaler, max_grad_norm=1.0)()
    if torch.cuda.device_count() > 1:
        q = torch.zeros(4, device="cuda:1", requires_grad=True)
        q.grad = torch.ones_like(q)
        with pytest.raises(ValueError, match="one device"):
            optim.CapturedTail(optim.RAdam([p, q]))()


# ---- the recipe's loop -------------------------------------------------------------------------------------------------

def _loop(dec, s, batches, mbs, captured, dp=False):
    """Three fp16 optimiser batches through SplitTrainBatch (or DataParallelSplitTrain at one rank), then the tail."""
    kw = dict(edge_capacity=s.flat.max_batch_edges(mbs), max_edges=s.flat.max_graph_edges(), autocast_dtype=torch.float16)
    params = [p for p in dec.parameters() if p.requires_grad]
    opt = optim.RAdam([{"params": params[::2], "weight_decay": 0.01}, {"params": params[1::2], "weight_decay": 0.0}],
                      lr=1e-3)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, SCHEDULES["warmup_linear"])
    scaler = torch.amp.GradScaler("cuda")
    tail = optim.CapturedTail(opt, scaler=scaler, scheduler=sched, max_grad_norm=1.0, clip_parameters=dec.parameters())
    if dp:
        from qagnn_b200.pipeline import SplitTrainStep
        step = SplitTrainStep(dec, s.dev, mbs, **kw)
        runner = D.DataParallelSplitTrain(step, s.dev, batch_size=len(batches[0]), micro_batch_size=mbs)
    else:
        runner = SplitTrainBatch(dec, s.dev, mbs, branches=4, **kw)
    out = []
    for b, batch in enumerate(batches):
        opt.zero_grad(set_to_none=False)
        if dp:
            for q in runner.micro_batches(batch):
                with runner.micro_step():
                    scaler.scale(runner.loss(q, _sv(q)) * len(q) / len(batch)).backward()
            runner.reduce_(len(batch))
        else:
            for chunk in train_chunks(batch, mbs, 4):
                w = torch.tensor([len(q) / len(batch) for q in chunk], device=DEV)
                scaler.scale((runner(chunk, [_sv(q) for q in chunk]) * w).sum()).backward()
        if captured:
            norm = tail()
        else:
            scaler.unscale_(opt)
            norm = optim.clip_grad_norm_(dec.parameters(), 1.0)
            sched.step()
            scaler.step(opt)
            scaler.update()
        out.append({"norm": norm.clone(), "scale": scaler._scale.clone(),
                    **{k: p.detach().clone() for k, p in dec.named_parameters()}})
    return out


@pytest.mark.parametrize("dp", [False, True], ids=["split_train_batch", "data_parallel_1_rank"])
def test_the_recipe_loop_equals_the_eager_tail(s48, deterministic, dp):
    mbs = 2
    order = np.random.default_rng(3).permutation(s48.Q)
    batches = [order[i * 8:(i + 1) * 8] for i in range(3)]
    base = _decoder()
    ref = _loop(copy.deepcopy(base), s48, batches, mbs, captured=False, dp=dp)
    got = _loop(copy.deepcopy(base), s48, batches, mbs, captured=True, dp=dp)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys()
        for k in r:
            assert torch.equal(g[k], r[k]), f"batch {i}: {k}"
