"""qagnn_b200.optim.RAdam without a GPU: the eager restatement of the reference's update (tests/radam_oracle.py) against the
reference's own trajectories (tests/golden/ref/radam.pt) bit for bit, the step-size table against the reference's formula,
the hyperparameter refusals and the refusal of CPU tensors."""
import os

import pytest
import torch

from qagnn_b200 import optim
from tests.radam_oracle import RAdamOracle, step_size

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "radam.pt")
CASES = torch.load(GOLDEN, weights_only=False)


def test_goldens_cover_the_cases_the_recipes_need():
    assert set(CASES) == {"two_groups_dlr", "two_groups_elr", "other_betas", "no_sgd", "grad_none"}
    assert CASES["two_groups_dlr"]["kwargs"]["lr"] == 1e-3 and CASES["two_groups_elr"]["kwargs"]["lr"] == 1e-5
    assert CASES["no_sgd"]["kwargs"]["degenerated_to_sgd"] is False
    assert any(g is None for step in CASES["grad_none"]["grads"] for g in step)
    assert all(len(c["after"]) == 12 for c in CASES.values())


def _groups(case, params):
    out, i = [], 0
    for gk, n in zip(case["groups"], case["group_sizes"]):
        out.append(dict(gk, params=params[i:i + n]))
        i += n
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_the_reference_bit_for_bit(name):
    case = CASES[name]
    params = [torch.nn.Parameter(p.clone()) for p in case["init"]]
    opt = RAdamOracle(_groups(case, params), **case["kwargs"])
    for t, (grads, after) in enumerate(zip(case["grads"], case["after"])):
        for p, g in zip(params, grads):
            p.grad = None if g is None else g.clone()
        opt.step()
        for i, (p, want) in enumerate(zip(params, after)):
            assert torch.equal(p.detach(), want["param"]), (name, t, i, "param")
            st = opt.state[p]
            assert (st["step"] if st else 0) == want["step"], (name, t, i, "step")
            for k in ("exp_avg", "exp_avg_sq"):
                assert (k in st) == (k in want), (name, t, i, k)
                if k in want:
                    assert torch.equal(st[k], want[k]), (name, t, i, k)


def test_the_trajectories_cross_the_rectification_switch_and_skip_missing_grads():
    assert step_size(0.9, 0.999, 5)[0] < 5 <= step_size(0.9, 0.999, 6)[0]
    after = CASES["grad_none"]["after"]
    assert [a[1]["step"] for a in after] == [1, 2, 2, 2, 3, 4, 5, 5, 6, 7, 8, 9]
    assert after[0][2]["step"] == 0 and "exp_avg" not in after[0][2]
    # without degenerated_to_sgd the first steps leave p as it is
    case = CASES["no_sgd"]
    assert torch.equal(case["after"][4][0]["param"], case["init"][0])
    assert not torch.equal(case["after"][5][0]["param"], case["init"][0])


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.8, 0.99), (0.0, 0.5), (0.95, 0.9999), (0.9, 0.0)])
def test_step_size_table_equals_the_reference_formula(betas):
    n = 100_001
    table = optim.step_size_table(*betas, n)
    assert table.dtype == torch.float64 and table.shape == (n, 2)
    rect, s = table[:, 0].tolist(), table[:, 1].tolist()
    for t in range(1, n):
        rho_t, want = step_size(*betas, t)
        assert rect[t] == (1.0 if rho_t >= 5 else 0.0), (betas, t)
        assert s[t] == want, (betas, t)  # exact: the same doubles


def test_hyperparameters_are_refused_as_the_reference_refuses_them():
    p = [torch.nn.Parameter(torch.zeros(3))]
    for kw, msg in [(dict(lr=-1e-3), "Invalid learning rate"), (dict(eps=-1.0), "Invalid epsilon value"),
                    (dict(betas=(1.0, 0.999)), "Invalid beta parameter at index 0"),
                    (dict(betas=(-0.1, 0.999)), "Invalid beta parameter at index 0"),
                    (dict(betas=(0.9, 1.0)), "Invalid beta parameter at index 1")]:
        with pytest.raises(ValueError, match=msg):
            optim.RAdam(p, **kw)
    optim.RAdam(p, lr=0.0, eps=0.0, betas=(0.0, 0.0), weight_decay=0.01)


def test_a_group_with_bad_betas_is_refused_at_step():
    p = torch.nn.Parameter(torch.zeros(3))
    opt = optim.RAdam([dict(params=[p], betas=(0.9, 1.0))])
    p.grad = torch.zeros(3)
    with pytest.raises(ValueError, match="index 1"):
        opt.step()


def test_cpu_tensors_and_sparse_grads_are_refused():
    p = torch.nn.Parameter(torch.zeros(3))
    opt = optim.RAdam([p])
    opt.step()  # no gradient: nothing to do
    p.grad = torch.zeros(3)
    with pytest.raises(TypeError, match="CUDA"):
        opt.step()
    p.grad = torch.zeros(3).to_sparse()
    with pytest.raises(RuntimeError, match="sparse"):
        opt.step()
    assert len(opt.state) == 0


def test_optimizer_contract():
    assert optim.RAdam._step_supports_amp_scaling is True
    assert issubclass(optim.RAdam, torch.optim.Optimizer)
