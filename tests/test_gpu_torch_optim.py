"""optim.Adam and optim.SGD against torch.optim.Adam / SGD as torch steps them by default on CUDA (foreach), on the same GPU:
after every step p, every state tensor and .grad equal torch's bit for bit.  The reference's four param groups (weight decay
on for some), a LambdaLR schedule, gradients that are None at some steps, sizes 0, 1 and both sides of the 8192-element
chunk, both lerp branches of Adam, SGD with momentum 0, with dampening and with Nesterov, fp16 GradScaler with infs injected
(an SGD whose first step is skipped included), CapturedTail against the eager tail over replays and a recapture, a torch
state dict loaded mid-run, and a step and a tail replay under sync-debug "error".  Needs a GPU: run with -m gpu."""
import copy

import pytest
import torch

from qagnn_b200 import optim

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [0, 1, 3, 8191, 8192, 8193, 16387, 4 * 4096 + 5]
STEPS = 24


def _params(seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(n, device=DEV, generator=g).requires_grad_() for n in SIZES]


def _groups(params, wd):
    # the reference's layout: decayed and undecayed groups of two parameter sets, each at its own lr
    return [{"params": params[i::4], "lr": 1e-3 * (1 + i), "weight_decay": wd if i % 2 == 0 else 0.0} for i in range(4)]


def _make(kind, params, **kw):
    wd = kw.pop("wd", 0.01)
    groups = _groups(params, wd)
    if kind == "adam":
        return optim.Adam(groups, **kw), lambda ps: torch.optim.Adam(_groups(ps, wd), **kw)
    return optim.SGD(groups, **kw), lambda ps: torch.optim.SGD(_groups(ps, wd), **kw)


CONFIGS = [
    ("adam", {}),
    ("adam", {"betas": (0.3, 0.95), "eps": 1e-6}),  # 1 - beta1 >= 0.5: lerp's other branch
    ("adam", {"wd": 0.0}),
    ("sgd", {"momentum": 0.0}),
    ("sgd", {"momentum": 0.9, "dampening": 0.1}),
    ("sgd", {"momentum": 0.9, "nesterov": True}),
    ("sgd", {"momentum": 0.9, "nesterov": True, "wd": 0.0}),  # torch adds into .grad itself
]
IDS = [f"{k}-{'-'.join(f'{a}={b}' for a, b in kw.items()) or 'default'}" for k, kw in CONFIGS]


def _grads(params, step, scale=None, inf_at=None, live=None):
    g = torch.Generator(device=DEV).manual_seed(1000 + step)
    for i, p in enumerate(params):
        x = torch.randn(p.shape, device=DEV, generator=g) * 0.3
        if live is not None and not live(i, step):
            p.grad = None
            continue
        if scale is not None:
            x = x * scale
        if inf_at is not None and step in inf_at and i == 4:
            x[0] = float("inf")
        if p.grad is None:
            p.grad = x
        else:
            p.grad.copy_(x)  # in place, as backward accumulates: a captured tail keeps its graph


def _live(i, step):  # some parameters miss a gradient at some steps
    return not (i % 3 == 1 and step % 4 in (1, 2))


def _bits(a, b):
    """a and b hold the same bits (NaNs included)."""
    return a.shape == b.shape and torch.equal(a.detach().view(torch.int32), b.detach().view(torch.int32))


def _same(ours, opt, theirs, ref, what):
    for i, (p, q) in enumerate(zip(ours, theirs)):
        assert _bits(p, q), (what, "p", i)
        assert (p.grad is None) == (q.grad is None), (what, "grad", i)
        if p.grad is not None:
            assert _bits(p.grad, q.grad), (what, "grad", i)
        st, rt = opt.state.get(p, {}), ref.state.get(q, {})
        for k, v in rt.items():
            if k == "step":
                assert int(st["step"]) == int(v), (what, k, i)
            elif v is not None:
                assert _bits(st[k], v), (what, k, i)


@pytest.mark.parametrize("kind,kw", CONFIGS, ids=IDS)
def test_matches_torch_with_groups_schedule_and_missing_grads(kind, kw):
    ours, theirs = _params(), _params()
    opt, mk = _make(kind, ours, **dict(kw))
    ref = mk(theirs)
    lam = lambda s: min(1.0, (s + 1) / 5.0) * 0.97 ** s  # noqa: E731
    s1, s2 = torch.optim.lr_scheduler.LambdaLR(opt, lam), torch.optim.lr_scheduler.LambdaLR(ref, lam)
    for step in range(STEPS):
        _grads(ours, step, live=_live)
        _grads(theirs, step, live=_live)
        opt.step()
        ref.step()
        s1.step()
        s2.step()
        _same(ours, opt, theirs, ref, (kind, step))


@pytest.mark.parametrize("kind,kw", [CONFIGS[0], CONFIGS[4], CONFIGS[5]], ids=[IDS[0], IDS[4], IDS[5]])
def test_grad_scaler_skips_match_torch(kind, kw):
    ours, theirs = _params(), _params()
    opt, mk = _make(kind, ours, **dict(kw))
    ref = mk(theirs)
    sc1 = torch.amp.GradScaler("cuda", init_scale=2.0 ** 14, growth_interval=3)
    sc2 = torch.amp.GradScaler("cuda", init_scale=2.0 ** 14, growth_interval=3)
    for sc in (sc1, sc2):
        sc.scale(torch.ones((), device=DEV))
    inf_at = {0, 1, 7, 12}  # the first two steps skipped: SGD sets its buffers at the third
    for step in range(STEPS):
        _grads(ours, step, scale=sc1._scale, inf_at=inf_at)
        _grads(theirs, step, scale=sc2._scale, inf_at=inf_at)
        sc1.step(opt)
        sc2.step(ref)
        sc1.update()
        sc2.update()
        assert torch.equal(sc1._scale, sc2._scale) and torch.equal(sc1._growth_tracker, sc2._growth_tracker), step
        _same(ours, opt, theirs, ref, (kind, step))


@pytest.mark.parametrize("kind,kw", [CONFIGS[0], CONFIGS[4]], ids=[IDS[0], IDS[4]])
def test_torch_state_dict_loaded_mid_run(kind, kw):
    ours, theirs = _params(), _params()
    _, mk = _make(kind, ours, **dict(kw))
    ref = mk(theirs)
    for step in range(6):
        _grads(theirs, step)
        ref.step()
    with torch.no_grad():
        for p, q in zip(ours, theirs):
            p.copy_(q)
    opt, _ = _make(kind, ours, **dict(kw))
    opt.load_state_dict(copy.deepcopy(ref.state_dict()))  # a checkpoint: no tensor shared with ref
    for step in range(6, 6 + 10):
        _grads(ours, step)
        _grads(theirs, step)
        opt.step()
        ref.step()
        _same(ours, opt, theirs, ref, (kind, step))


def _eager_tail(opt, params, scaler, sched, max_norm):
    scaler.unscale_(opt)
    norm = optim.clip_grad_norm_([p for p in params if p.grad is not None], max_norm)
    sched.step()
    scaler.step(opt)
    scaler.update()
    return norm


@pytest.mark.parametrize("kind,kw", [CONFIGS[0], CONFIGS[1], CONFIGS[3], CONFIGS[4], CONFIGS[6]],
                         ids=[IDS[0], IDS[1], IDS[3], IDS[4], IDS[6]])
def test_captured_tail_matches_eager_tail(kind, kw):
    sides = []
    for captured in (False, True):
        params = _params()
        opt, _ = _make(kind, params, **dict(kw))
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12, growth_interval=4)
        scaler.scale(torch.ones((), device=DEV))
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: min(1.0, (s + 1) / 5.0))
        tail = optim.CapturedTail(opt, scaler=scaler, scheduler=sched, max_grad_norm=1.0) if captured else None
        sides.append((params, opt, scaler, sched, tail))
    (pa, oa, sa, ha, _), (pb, ob, sb, hb, tail) = sides
    for step in range(STEPS):
        if step == 13:  # a recapture: every .grad is reallocated, at new addresses while the old ones are held
            held = [p.grad for p in pa + pb]
            ob.zero_grad(set_to_none=True)
            oa.zero_grad(set_to_none=True)
        _grads(pa, step, scale=sa._scale, inf_at={0, 9})
        _grads(pb, step, scale=sb._scale, inf_at={0, 9})
        n1 = _eager_tail(oa, pa, sa, ha, 1.0)
        n2 = tail()
        assert _bits(n1, n2), step
        assert torch.equal(sa._scale, sb._scale) and torch.equal(sa._growth_tracker, sb._growth_tracker), step
        _same(pb, ob, pa, oa, (kind, step))
        assert [g["lr"] for g in oa.param_groups] == [g["lr"] for g in ob.param_groups]
    assert tail.captures == 2 and len(held) == 2 * len(SIZES)


def test_captured_tail_refuses_torch_optimizers():
    p = _params()
    for opt in (torch.optim.Adam(p), torch.optim.SGD(p, lr=0.1)):
        with pytest.raises(ValueError, match="run the eager tail"):
            optim.CapturedTail(opt)


@pytest.mark.parametrize("kind,kw", [CONFIGS[0], CONFIGS[5]], ids=[IDS[0], IDS[5]])
def test_step_and_tail_replay_read_nothing_on_the_host(kind, kw):
    params = _params()
    opt, _ = _make(kind, params, **dict(kw))
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    scaler.scale(torch.ones((), device=DEV))
    tail = optim.CapturedTail(opt, scaler=scaler, max_grad_norm=1.0)
    for step in range(3):
        _grads(params, step, scale=scaler._scale)
        if step == 0:
            scaler.step(opt)
            scaler.update()
        else:
            tail()  # the first call captures; the second replays
    _grads(params, 3, scale=scaler._scale)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.step()
        _grads(params, 4, scale=scaler._scale)
        tail()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert tail.captures == 1
