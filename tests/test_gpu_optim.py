"""qagnn_b200.optim.RAdam on the GPU against the eager restatement of the reference's update (tests/radam_oracle.py), bit for
bit: the kernel over sizes that exercise its vector and scalar paths, an unaligned view, more tensors than one launch holds;
the recipe's training loop (SplitTrainStep, clip_grad_norm_, GradScaler, a LambdaLR schedule) in fp32 / bf16 / fp16; GradScaler's
inf skip and its grad_scale route; no host synchronisation in the optimiser tail; one launch and no allocation per step;
state_dict round trips, from this optimiser's state and from the reference's.  Needs a GPU: run with -m gpu."""
import copy

import numpy as np
import pytest
import torch

from qagnn_b200 import _lib
from qagnn_b200.optim import RAdam
from qagnn_b200.pipeline import SplitTrainStep
from tests.radam_oracle import RAdamOracle
from tests.test_gpu_split_train import DT_IDS, DTYPES, NC, Split, _decoder, _plan, _sv, deterministic  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NO_DECAY = ("bias", "LayerNorm.bias", "LayerNorm.weight")


def _grads(shapes, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(s, device=DEV, generator=g) * scale * 10.0 ** (-(i % 4)) for i, s in enumerate(shapes)]


def _pairs(tensors, groups_of, opt_kw, group_kw):
    """The same parameters twice: for RAdam and for the oracle."""
    out = []
    for cls in (RAdam, RAdamOracle):
        ps = [torch.nn.Parameter(t.clone()) for t in tensors]
        groups = [dict(group_kw[gi], params=[p for p, g in zip(ps, groups_of) if g == gi]) for gi in range(len(group_kw))]
        out.append((ps, cls(groups, **opt_kw)))
    return out


def _assert_same_state(got, ref, what=""):
    (gp, gopt), (rp, ropt) = got, ref
    for i, (a, b) in enumerate(zip(gp, rp)):
        assert torch.equal(a.detach(), b.detach()), f"{what} param {i}"
        sa, sb = gopt.state[a], ropt.state[b]
        assert bool(sa) == bool(sb), f"{what} state {i}"
        if sb:
            assert sa["step"].dtype == torch.int64 and sa["step"].device == a.device
            assert int(sa["step"]) == sb["step"], f"{what} step {i}"
            for k in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(sa[k], sb[k]), f"{what} {k} {i}"


CONFIGS = {
    "recipe_dlr": (dict(lr=1e-3, weight_decay=0.01), [dict(), dict(weight_decay=0.0)]),
    "recipe_elr": (dict(lr=1e-5, weight_decay=0.01), [dict(), dict(weight_decay=0.0)]),
    "other_betas": (dict(lr=1e-3), [dict(betas=(0.8, 0.99), weight_decay=0.01), dict(eps=1e-6)]),
    "no_sgd": (dict(lr=1e-3, weight_decay=0.01, degenerated_to_sgd=False), [dict(), dict(weight_decay=0.0)]),
}


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_kernel_equals_the_eager_oracle_bit_for_bit(cfg):
    """numel 1, odd, not a multiple of 4, several chunks, over 2^24; 14 steps across the rho_t = 5 switch."""
    opt_kw, group_kw = CONFIGS[cfg]
    shapes = [(1,), (7,), (3, 5), (1001,), (8192 * 3 + 5,), (1 << 24) + 3]
    torch.manual_seed(1)
    tensors = [torch.randn(s, device=DEV) for s in shapes]
    groups_of = [i % 2 for i in range(len(shapes))]
    got, ref = _pairs(tensors, groups_of, opt_kw, group_kw)
    for t in range(14):
        gs = _grads(shapes, 10 + t)
        for (ps, opt) in (got, ref):
            for p, g in zip(ps, gs):
                p.grad = g.clone()
            opt.step()
        _assert_same_state(got, ref, f"{cfg} step {t + 1}")


def test_an_unaligned_view_takes_the_scalar_path_and_equals_the_oracle():
    """A parameter (and gradient) that is a view at a storage offset of one element is handled, not refused."""
    torch.manual_seed(2)
    base = torch.randn(4099, device=DEV)
    out = []
    for cls in (RAdam, RAdamOracle):
        b = base.clone()
        p = torch.nn.Parameter(b[1:])
        assert p.data_ptr() % 16 == 4 and p.is_contiguous()
        out.append(([p], cls([p], lr=1e-3, weight_decay=0.01)))
    gbase = torch.empty(4099, device=DEV)
    for t in range(12):
        g = _grads([(4098,)], 40 + t)[0]
        for ps, opt in out:
            gbase[1:].copy_(g)
            ps[0].grad = gbase[1:].clone() if opt.__class__ is RAdamOracle else gbase[1:]
            opt.step()
            if opt.__class__ is RAdam:
                ps[0].grad = None
        _assert_same_state(*out, f"step {t + 1}")


def test_more_tensors_than_one_launch_holds():
    rng = np.random.default_rng(3)
    shapes = [(int(n),) for n in rng.integers(1, 300, 700)]
    torch.manual_seed(3)
    tensors = [torch.randn(s, device=DEV) for s in shapes]
    groups_of = [i % 3 for i in range(len(shapes))]
    got, ref = _pairs(tensors, groups_of, dict(lr=1e-3, weight_decay=0.01),
                      [dict(), dict(weight_decay=0.0), dict(betas=(0.85, 0.995))])
    lib = _lib.load()
    for t in range(8):
        gs = _grads(shapes, 70 + t)
        for ps, opt in (got, ref):
            for p, g in zip(ps, gs):
                p.grad = g.clone()
            n0 = lib.qagnn_launch_count()
            opt.step()
            if opt is got[1]:
                assert lib.qagnn_launch_count() - n0 == 2  # 700 tensors: 512 + 188
        _assert_same_state(got, ref, f"step {t + 1}")


def test_a_parameter_without_grad_is_skipped_and_its_step_does_not_advance():
    shapes = [(33,), (5, 5)]
    tensors = [torch.randn(s, device=DEV) for s in shapes]
    got, ref = _pairs(tensors, [0, 0], dict(lr=1e-3, weight_decay=0.01), [dict()])
    for t in range(10):
        gs = _grads(shapes, 90 + t)
        for ps, opt in (got, ref):
            ps[0].grad = gs[0].clone()
            ps[1].grad = None if t in (0, 3, 4) else gs[1].clone()
            opt.step()
        _assert_same_state(got, ref, f"step {t + 1}")
    assert int(got[1].state[got[0][1]]["step"]) == 7


def test_refusals_on_the_gpu():
    p = torch.nn.Parameter(torch.zeros(4, 4, device=DEV))
    opt = RAdam([p])
    p.grad = torch.zeros(4, 4, device=DEV).t()
    with pytest.raises(ValueError, match="contiguous"):
        opt.step()
    q = torch.nn.Parameter(torch.zeros(4, 4, device=DEV, dtype=torch.bfloat16))
    q.grad = torch.zeros_like(q)
    with pytest.raises(TypeError, match="float32"):
        RAdam([q]).step()
    assert len(opt.state) == 0


# ---- the recipe's training loop (qagnn.py:249-278) through SplitTrainStep -------------------------------------------

@pytest.fixture(scope="module")
def s48():
    return Split(48, seed=51)


def _recipe_groups(dec):
    named = [(n, p) for n, p in dec.named_parameters() if p.requires_grad]
    return [{"params": [p for n, p in named if not any(nd in n for nd in NO_DECAY)], "weight_decay": 0.01, "lr": 1e-3},
            {"params": [p for n, p in named if any(nd in n for nd in NO_DECAY)], "weight_decay": 0.0, "lr": 1e-3}]


def _warmup_linear(warmup, total):
    return lambda step: step / max(1, warmup) if step < warmup else max(0.0, (total - step) / max(1.0, total - warmup))


def _train(dec, s, plan, dt, opt_cls, max_grad_norm=1.0):
    opt = opt_cls(_recipe_groups(dec))
    sched = torch.optim.lr_scheduler.LambdaLR(opt, _warmup_linear(1, 4))
    scaler = torch.amp.GradScaler("cuda") if dt == torch.float16 else None
    mbs = len(plan[0][0])
    K, M = s.flat.max_batch_edges(mbs), s.flat.max_graph_edges()
    step = SplitTrainStep(dec, s.dev, mbs, edge_capacity=K, max_edges=M, autocast_dtype=dt)
    rec = []
    for o, micro in enumerate(plan):
        opt.zero_grad()
        total = sum(len(q) for q in micro)
        for m, q in enumerate(micro):
            sv = _sv(mbs, 100 * o + m).requires_grad_(True)
            w = step(q, sv) * len(q) / total
            (scaler.scale(w) if scaler is not None else w).backward()
        if max_grad_norm > 0:
            if scaler is not None:
                scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(dec.parameters(), max_grad_norm)
        sched.step()
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        r = {}
        for k, p in dec.named_parameters():
            r[f"param {k}"] = p.detach().clone()
            st = opt.state[p]
            if st:
                r[f"step {k}"] = int(st["step"])
                r[f"exp_avg {k}"], r[f"exp_avg_sq {k}"] = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
        if scaler is not None:
            r["scale"], r["growth"] = scaler._scale.clone(), scaler._growth_tracker.clone()
        rec.append(r)
    return rec


def _same_records(got, ref):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys(), (i, sorted(set(g) ^ set(r)))
        assert sum(k.startswith("exp_avg ") for k in r) > 10
        for k in r:
            if isinstance(r[k], torch.Tensor):
                assert g[k].dtype == r[k].dtype and torch.equal(g[k], r[k]), f"batch {i}: {k}"
            else:
                assert g[k] == r[k], f"batch {i}: {k}"


@pytest.mark.parametrize("mbs", [2, 8])
@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_two_optimiser_batches_of_the_recipe_equal_the_eager_oracle(s48, deterministic, dt, mbs):  # noqa: F811
    dec = _decoder()
    plan = _plan(s48, mbs, seed=mbs)
    ref = _train(copy.deepcopy(dec), s48, plan, dt, RAdamOracle)
    got = _train(copy.deepcopy(dec), s48, plan, dt, RAdam)
    _same_records(got, ref)
    assert any(not torch.equal(got[1][k], ref[0][k]) for k in got[1] if k.startswith("param "))  # the step moved them


# ---- GradScaler ----------------------------------------------------------------------------------------------------

SHAPES = [(300, 64), (64,), (5,), (1000, 3)]


def _scaled_grads(seed, sc, inf_at=None):
    gs = [sc.scale(g) for g in _grads(SHAPES, seed)]
    if inf_at is not None:
        gs[inf_at][1] = float("inf")
    return gs


def _scaler_pair():
    torch.manual_seed(5)
    tensors = [torch.randn(s, device=DEV) for s in SHAPES]
    pairs = _pairs(tensors, [0, 1, 1, 0], dict(lr=1e-3, weight_decay=0.01), [dict(), dict(weight_decay=0.0)])
    return [(ps, opt, torch.amp.GradScaler("cuda", init_scale=2.0 ** 12, growth_interval=2)) for ps, opt in pairs]


def _scaler_state(sc):
    return sc._scale.clone(), sc._growth_tracker.clone()


@pytest.mark.parametrize("unscale", [True, False], ids=["unscale_clip", "grad_scale"])
def test_gradscaler_routes_and_an_overflowing_batch_equal_eager(unscale):
    """unscale_ + clip_grad_norm_ + step, or step straight from scaled grads (max_grad_norm 0: GradScaler hands RAdam the scale
    and the kernel unscales, writing the unscaled grads back); batch 3 overflows: nothing moves, the scale backs off."""
    got, ref = _scaler_pair()
    for t in range(8):
        before = [p.detach().clone() for p in got[0]]
        scale = float(got[2].get_scale())
        for ps, opt, sc in (got, ref):
            for p, g in zip(ps, _scaled_grads(20 + t, sc, inf_at=1 if t == 3 else None)):
                p.grad = g
            if unscale:
                sc.unscale_(opt)
                torch.nn.utils.clip_grad_norm_(ps, 1.0)
            sc.step(opt)
            sc.update()
        for a, b in zip(got[0], ref[0]):  # bit patterns: clipping an overflowed batch leaves NaN in both
            assert torch.equal(a.grad.view(torch.int32), b.grad.view(torch.int32)), t
        _assert_same_state(got[:2], ref[:2], f"step {t + 1}")
        for x, y in zip(_scaler_state(got[2]), _scaler_state(ref[2])):
            assert torch.equal(x, y), t
        if t == 3:
            assert all(torch.equal(a.detach(), b) for a, b in zip(got[0], before))
            assert all(int(got[1].state[p]["step"]) == 3 for p in got[0])
            assert float(got[2].get_scale()) == scale / 2  # backed off
    assert all(int(got[1].state[p]["step"]) == 7 for p in got[0])


def test_the_fp16_optimiser_tail_does_not_synchronise():
    (ps, opt, sc), _ = _scaler_pair()
    for t in range(3):
        gs = _scaled_grads(60 + t, sc)
        torch.cuda.synchronize()
        for p, g in zip(ps, gs):
            p.grad = g
        torch.cuda.set_sync_debug_mode("error")
        try:
            sc.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(ps, 1.0)
            sc.step(opt)
            sc.update()
            opt.zero_grad()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert all(int(opt.state[p]["step"]) == 3 for p in ps)


def test_one_launch_per_step_and_no_allocation_after_the_first():
    dec = _decoder()
    opt = RAdam(_recipe_groups(dec))
    params = [p for p in dec.parameters() if p.requires_grad]
    lib = _lib.load()
    mem = None
    for t in range(5):
        for p, g in zip(params, _grads([p.shape for p in params], 80 + t)):
            p.grad = g
        torch.cuda.synchronize()
        m0, n0 = torch.cuda.memory_allocated(DEV), lib.qagnn_launch_count()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            opt.step()
            torch.cuda.synchronize()
        assert lib.qagnn_launch_count() - n0 == 1
        kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "radam" in e.name]
        assert len(kernels) <= 1  # a profiler session can drop a record, never add one
        if t == 0:
            mem = torch.cuda.memory_allocated(DEV)
        else:
            assert torch.cuda.memory_allocated(DEV) == m0 == mem, t


# ---- state_dict ----------------------------------------------------------------------------------------------------

def test_state_dict_round_trip_continues_bit_for_bit():
    shapes = [(129,), (17, 3)]
    torch.manual_seed(6)
    tensors = [torch.randn(s, device=DEV) for s in shapes]
    (ps, opt), _ = _pairs(tensors, [0, 1], dict(lr=1e-3, weight_decay=0.01), [dict(), dict(weight_decay=0.0)])
    for t in range(4):
        for p, g in zip(ps, _grads(shapes, 100 + t)):
            p.grad = g
        opt.step()
    sd = copy.deepcopy(opt.state_dict())
    ps2 = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    opt2 = RAdam([dict(params=[ps2[0]]), dict(params=[ps2[1]])], lr=5.0)
    opt2.load_state_dict(sd)
    assert opt2.param_groups[1]["weight_decay"] == 0.0 and opt2.param_groups[0]["lr"] == 1e-3
    for t in range(4, 10):
        gs = _grads(shapes, 100 + t)
        for q, o in ((ps, opt), (ps2, opt2)):
            for p, g in zip(q, gs):
                p.grad = g.clone()
            o.step()
    for a, b in zip(ps, ps2):
        assert torch.equal(a, b)
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(opt.state[a][k], opt2.state[b][k]), k


def test_a_reference_form_state_loads_and_continues_bit_for_bit():
    """The reference's state: 'step' a Python int, tensors on the CPU, its per-group step-size cache in the groups."""
    shapes = [(257,), (9, 9)]
    torch.manual_seed(7)
    tensors = [torch.randn(s, device=DEV) for s in shapes]
    got, ref = _pairs(tensors, [0, 1], dict(lr=1e-3, weight_decay=0.01), [dict(), dict(weight_decay=0.0)])
    for t in range(7):
        for p, g in zip(ref[0], _grads(shapes, 120 + t)):
            p.grad = g
        ref[1].step()
    sd = copy.deepcopy(ref[1].state_dict())
    for st in sd["state"].values():
        assert isinstance(st["step"], int)
        st["exp_avg"], st["exp_avg_sq"] = st["exp_avg"].cpu(), st["exp_avg_sq"].cpu()
    for g in sd["param_groups"]:
        g["buffer"] = [[None, None, None] for _ in range(10)]
    for a, b in zip(got[0], ref[0]):
        a.data.copy_(b.detach())
    got[1].load_state_dict(sd)
    _assert_same_state(got, ref, "loaded")
    for t in range(7, 14):
        gs = _grads(shapes, 120 + t)
        for ps, opt in (got, ref):
            for p, g in zip(ps, gs):
                p.grad = g.clone()
            opt.step()
        _assert_same_state(got, ref, f"step {t + 1}")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_parameters_on_two_devices_get_one_launch_each_and_equal_the_oracle():
    shapes = [(1000,), (33,)]
    tensors = [torch.randn(shapes[0], device="cuda:0"), torch.randn(shapes[1], device="cuda:1")]
    got, ref = _pairs(tensors, [0, 1], dict(lr=1e-3, weight_decay=0.01), [dict(), dict(weight_decay=0.0)])
    scalers = [torch.amp.GradScaler("cuda", init_scale=256.0) for _ in range(2)]
    lib = _lib.load()
    for t in range(8):
        gs = [torch.randn(s, generator=torch.Generator().manual_seed(t)) for s in shapes]
        for (ps, opt), sc in zip((got, ref), scalers):
            for p, g in zip(ps, gs):
                p.grad = (g * 256.0).to(p.device)
            n0 = lib.qagnn_launch_count()
            sc.step(opt)
            sc.update()
            if opt is got[1]:
                assert lib.qagnn_launch_count() - n0 == 2
        _assert_same_state(got, ref, f"step {t + 1}")
