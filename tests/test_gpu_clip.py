"""qagnn_b200.optim.clip_grad_norm_ on the GPU: the norm equals the restated summation order (tests/clip_oracle.py) bit for bit
over sizes, unaligned views, several launches, the decoder's real gradients and a RoBERTa-large-sized set; it repeats, sits
within one fp32 ulp of the exact norm and within 1e-5 of torch's; from its norm on, the coefficient and every gradient are
torch's ops bit for bit; non-finite gradients; the recipe's optimiser tail without host synchronisation; and three optimiser
batches of the recipe through SplitTrainStep against torch's clip.  Needs a GPU: run with -m gpu."""
import copy
import math

import numpy as np
import pytest
import torch

from qagnn_b200 import _lib, optim
from tests import clip_oracle as CO
from tests import helpers as Hh
from tests.test_gpu_optim import _grads, _same_records, _train
from tests.test_gpu_split_train import DT_IDS, DTYPES, NC, _decoder, _eager, _plan, _sv, deterministic, s48  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _params(grads):
    ps = []
    for g in grads:
        p = torch.nn.Parameter(torch.zeros_like(g))
        p.grad = g.clone()
        ps.append(p)
    return ps


def _coef():
    return optim._clip_workspace[torch.device(DEV)][2].reshape(())


def _bits(t):
    return t.detach().reshape(-1).view(torch.int32)


def _check_against_oracle_and_torch(grads, max_norm):
    """Runs the clip on copies of grads; returns (total_norm, clipped grads) after checking the norm against the oracle bit
    for bit and torch's within 1e-5, and the coefficient and gradients against torch's ops fed this norm."""
    ps = _params(grads)
    norm = optim.clip_grad_norm_(ps, max_norm)
    assert norm.dtype == torch.float32 and norm.dim() == 0 and norm.device == torch.device(DEV)
    want = CO.total_norm([g.cpu().numpy() for g in grads])
    assert np.float32(norm.item()).view(np.int32) == want.view(np.int32), (norm.item(), want)
    ref = _params(grads)
    torch_norm = torch.nn.utils.clip_grad_norm_(ref, max_norm, foreach=True)
    torch.testing.assert_close(norm, torch_norm, rtol=1e-5, atol=0)
    # torch's own coefficient ops and _foreach_mul_ on this kernel's norm
    ref = _params(grads)
    coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
    assert torch.equal(_bits(_coef()), _bits(coef))
    torch._foreach_mul_([p.grad for p in ref], coef)
    for i, (a, b) in enumerate(zip(ps, ref)):
        assert torch.equal(_bits(a.grad), _bits(b.grad)), i
    return norm, [p.grad for p in ps]


def _exact_norm(grads):
    return math.sqrt(math.fsum(float(v) for g in grads for v in g.double().square().reshape(-1).cpu().numpy()))


def _within_one_ulp(norm, grads):
    exact = _exact_norm(grads)
    assert abs(norm.item() - exact) <= float(np.spacing(np.float32(norm.item()))), (norm.item(), exact)


def _random(sizes, seed):
    return _grads([(n,) for n in sizes], seed)


def test_sizes_0_1_3_8193_clip_and_do_not_clip():
    grads = _random([0, 1, 3, 8193], 1)
    for max_norm in (0.05, 1e6):
        norm, out = _check_against_oracle_and_torch(grads, max_norm)
        _within_one_ulp(norm, grads)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(out, grads))  # max_norm above the norm: untouched
    for n in (0, 1, 3, 8193):
        _check_against_oracle_and_torch(_random([n], 10 + n), 1e-3)


def test_views_at_odd_storage_offsets_take_the_scalar_path():
    base = torch.randn(3 * 8192 + 11, device=DEV)
    spans = [(1, 8193), (8195, 5003), (13199, 1)]  # element offsets 1, 3 and 3 mod 4: no view is 16-byte aligned
    grads = [base[o:o + n] for o, n in spans]
    assert all(g.data_ptr() % 16 != 0 and g.is_contiguous() for g in grads)
    for max_norm in (0.5, 1e6):
        work = base.clone()
        ps = [torch.nn.Parameter(torch.zeros(n, device=DEV)) for _, n in spans]
        for p, (o, n) in zip(ps, spans):
            p.grad = work[o:o + n]
        norm = optim.clip_grad_norm_(ps, max_norm)
        want = CO.total_norm([g.cpu().numpy() for g in grads])
        assert np.float32(norm.item()).view(np.int32) == want.view(np.int32)
        # the same values through the vector path: the order does not depend on alignment
        assert torch.equal(_bits(optim.clip_grad_norm_(_params(grads), 1e6)), _bits(norm))
        coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
        expect = base.clone()
        for o, n in spans:
            expect[o:o + n] *= coef
        assert torch.equal(_bits(work), _bits(expect))  # every view scaled, nothing between them written


def test_700_tensors_take_two_launches_of_each_kernel():
    rng = np.random.default_rng(3)
    grads = _random([int(n) for n in rng.integers(1, 20000, 700)], 4)
    lib = _lib.load()
    n0 = lib.qagnn_launch_count()
    norm, _ = _check_against_oracle_and_torch(grads, 1.0)
    assert lib.qagnn_launch_count() - n0 == 4  # 512 + 188 tensors, norm and scale
    _within_one_ulp(norm, grads)


def test_two_launches_no_sync_and_no_workspace_allocation_after_the_first_call():
    grads = _random([300 * 64, 64, 5, 3000], 5)
    ps = _params(grads)
    lib = _lib.load()
    optim.clip_grad_norm_(ps, 1.0)
    for t in range(3):
        for p, g in zip(ps, _random([300 * 64, 64, 5, 3000], 6 + t)):
            p.grad.copy_(g)
        torch.cuda.synchronize()
        m0, n0 = torch.cuda.memory_allocated(DEV), lib.qagnn_launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            norm = optim.clip_grad_norm_(ps, 1.0)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert lib.qagnn_launch_count() - n0 == 2
        assert torch.cuda.memory_allocated(DEV) - m0 <= 512  # the returned norm alone
        del norm
        assert torch.cuda.memory_allocated(DEV) == m0


def test_two_calls_give_the_same_bits_and_the_norm_is_a_new_tensor():
    grads = _random([100_003, 7, 8192 * 5], 7)
    a = optim.clip_grad_norm_(_params(grads), 1e6)
    b = optim.clip_grad_norm_(_params(grads), 1e6)
    assert a.data_ptr() != b.data_ptr() and torch.equal(_bits(a), _bits(b))
    _within_one_ulp(a, grads)


def test_the_decoders_real_gradients(s48):
    dec = _decoder()
    K = s48.flat.max_batch_edges(2)
    q = _plan(s48, 2, seed=4)[0][0]
    loss, _, _ = _eager(dec, s48, q, _sv(2, 3).requires_grad_(True), K, None)
    loss.backward()
    grads = [p.grad.detach().clone() for p in dec.parameters() if p.grad is not None]
    assert len(grads) > 20
    norm = torch.nn.utils.clip_grad_norm_(_params(grads), 1e6)
    for max_norm in (0.5 * norm.item(), 2.0 * norm.item()):
        got, _ = _check_against_oracle_and_torch(grads, max_norm)
        _within_one_ulp(got, grads)


def _roberta_large_sizes():
    H, F, V = 1024, 4096, 50265
    layer = [H * H, H] * 4 + [H, H, F * H, F, H * F, H, H, H]
    return [V * H, 514 * H, H, H, H] + layer * 24 + [H * H, H]


def test_a_roberta_large_set_of_355m_parameters():
    sizes = _roberta_large_sizes()
    assert len(sizes) == 391 and sum(sizes) > 355_000_000
    g = torch.Generator(device=DEV).manual_seed(8)
    grads = [torch.randn(n, device=DEV, generator=g) * 1e-3 for n in sizes]
    norm = optim.clip_grad_norm_(_params(grads), 1e9)
    want = CO.total_norm([x.cpu().numpy() for x in grads])
    assert np.float32(norm.item()).view(np.int32) == want.view(np.int32)
    torch_norm = torch.nn.utils.clip_grad_norm_(_params(grads), 1e9, foreach=True)
    torch.testing.assert_close(norm, torch_norm, rtol=1e-5, atol=0)
    ps = _params(grads)
    norm2 = optim.clip_grad_norm_(ps, 1.0)
    assert torch.equal(_bits(norm2), _bits(norm))
    coef = torch.clamp(1.0 / (norm + 1e-6), max=1.0)
    assert coef.item() < 1
    for p, x in zip(ps, grads):
        assert torch.equal(_bits(p.grad), _bits(x * coef))


@pytest.mark.parametrize("bad", ["inf", "nan"])
def test_non_finite_gradients_give_torchs_result(bad):
    grads = _random([1000, 33, 8192 * 2 + 1], 9)
    grads[2][5000] = float(bad)
    ps, ref = _params(grads), _params(grads)
    norm = optim.clip_grad_norm_(ps, 1.0)
    want = torch.nn.utils.clip_grad_norm_(ref, 1.0)
    assert (norm.isinf().item() and want.isinf().item()) if bad == "inf" else (norm.isnan().item() and want.isnan().item())
    assert _coef().item() == 0.0 if bad == "inf" else _coef().isnan().item()
    for a, b in zip(ps, ref):
        assert torch.equal(a.grad.isnan(), b.grad.isnan())
        keep = ~b.grad.isnan()
        assert torch.equal(_bits(a.grad[keep]), _bits(b.grad[keep]))


def test_refusals_on_the_gpu():
    p = torch.nn.Parameter(torch.zeros(4, 4, device=DEV))
    p.grad = torch.ones(4, 4, device=DEV).t()
    with pytest.raises(ValueError, match=r"clip_grad_norm_: the gradient must be contiguous"):
        optim.clip_grad_norm_([p], 1.0)
    q = torch.nn.Parameter(torch.zeros(3, device=DEV, dtype=torch.float16))
    q.grad = torch.ones_like(q)
    with pytest.raises(TypeError, match=r"clip_grad_norm_: the gradient must be float32 \(got torch.float16\)"):
        optim.clip_grad_norm_([q], 1.0)
    if torch.cuda.device_count() > 1:
        r = torch.nn.Parameter(torch.zeros(3, device="cuda:1"))
        r.grad = torch.ones_like(r)
        p.grad = torch.ones(4, 4, device=DEV)
        with pytest.raises(ValueError, match="all must be on one device"):
            optim.clip_grad_norm_([p, r], 1.0)


# ---- the recipe's optimiser tail -------------------------------------------------------------------------------------

@pytest.mark.parametrize("cls", [optim.RAdam, optim.AdamW], ids=["radam", "adamw"])
def test_the_fp16_optimiser_tail_does_not_synchronise(cls):
    shapes = [(300, 64), (64,), (5,), (1000, 3)]
    torch.manual_seed(5)
    ps = [torch.nn.Parameter(torch.randn(s, device=DEV)) for s in shapes]
    opt, sc = cls(ps, lr=1e-3), torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
    for t in range(3):
        gs = [sc.scale(g) for g in _grads(shapes, 60 + t)]
        torch.cuda.synchronize()
        for p, g in zip(ps, gs):
            p.grad = g
        torch.cuda.set_sync_debug_mode("error")
        try:
            sc.unscale_(opt)
            optim.clip_grad_norm_(ps, 1.0)
            sc.step(opt)
            sc.update()
            opt.zero_grad()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert all(int(opt.state[p]["step"]) == 3 for p in ps)


def _split_train(monkeypatch, s, plan, dt, clip, max_norm):
    """test_gpu_optim._train (the recipe's loop with RAdam through SplitTrainStep) with `clip` as clip_grad_norm_; returns
    its records and the norms the clip returned."""
    norms = []

    def recorded(params, _max_norm):
        norms.append(clip(params, max_norm).item())

    with monkeypatch.context() as m:
        m.setattr(torch.nn.utils, "clip_grad_norm_", recorded)
        return _train(copy.deepcopy(_decoder()), s, plan, dt, optim.RAdam, max_grad_norm=max_norm), norms


TORCH_CLIP = torch.nn.utils.clip_grad_norm_


def _within_training_bars(got, ref):
    assert len(got) == len(ref) == 3
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.keys() == r.keys()
        for k in r:
            what = f"batch {i}: {k}"
            if k.startswith("step "):
                assert g[k] == r[k], what
            elif k in ("scale", "growth"):
                assert torch.equal(g[k], r[k]), what
            elif k.startswith("param "):  # tests/test_gpu_split_train.py's bars
                Hh.assert_close(g[k], r[k], what, atol=1e-4 * float(r[k].abs().max()) + 2e-3, rtol=1e-4)
            else:
                Hh.assert_close(g[k], r[k], what, atol=1e-4 * max(float(r[k].abs().max()), 1e-6), rtol=1e-4)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_three_optimiser_batches_of_the_recipe_against_torchs_clip(monkeypatch, s48, deterministic, dt):  # noqa: F811
    plan = _plan(s48, 2, seed=5, n_opt=3)
    # a max_norm that never clips: every parameter and optimiser state equals torch's clip's bit for bit
    got, norms = _split_train(monkeypatch, s48, plan, dt, optim.clip_grad_norm_, 1e9)
    ref, ref_norms = _split_train(monkeypatch, s48, plan, dt, TORCH_CLIP, 1e9)
    assert len(norms) == 3 and max(norms) < 1e9
    np.testing.assert_allclose(norms, ref_norms, rtol=1e-5)
    _same_records(got, ref)
    # the recipe's max_norm of 1.0 (half the first batch's norm if that is smaller, so the clip scales at least once):
    # within the training bars
    max_norm = min(1.0, 0.5 * norms[0])
    got, norms = _split_train(monkeypatch, s48, plan, dt, optim.clip_grad_norm_, max_norm)
    ref, ref_norms = _split_train(monkeypatch, s48, plan, dt, TORCH_CLIP, max_norm)
    assert norms[0] > max_norm
    np.testing.assert_allclose(norms, ref_norms, rtol=1e-5)
    _within_training_bars(got, ref)
