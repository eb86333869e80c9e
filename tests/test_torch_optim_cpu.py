"""optim.Adam and optim.SGD without a GPU: the constructors' checks and messages against torch's, the refusals, the param
groups, the Adam step table against torch's Python formulas, the state-dict conversion of torch's steps, the C entries in the
header and the ctypes binding, and the compiled kernels (vector loads, no floating-point atomics)."""
import collections
import os
import re
import shutil
import subprocess

import pytest
import torch

from qagnn_b200 import _lib, build, optim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _param():
    return torch.nn.Parameter(torch.zeros(3))


def _error(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return type(e), str(e)
    return None


ADAM_BAD = [dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)), dict(weight_decay=-0.1),
            dict(betas=(0, 0.999))]
SGD_BAD = [dict(lr=-0.1), dict(momentum=-0.5), dict(weight_decay=-1.0), dict(nesterov=True),
           dict(nesterov=True, momentum=0.9, dampening=0.1)]


@pytest.mark.parametrize("kw", ADAM_BAD)
def test_adam_checks_as_torch(kw):
    ours, theirs = _error(lambda: optim.Adam([_param()], **kw)), _error(lambda: torch.optim.Adam([_param()], **kw))
    assert theirs is not None and ours == theirs


@pytest.mark.parametrize("kw", SGD_BAD)
def test_sgd_checks_as_torch(kw):
    ours, theirs = _error(lambda: optim.SGD([_param()], **kw)), _error(lambda: torch.optim.SGD([_param()], **kw))
    assert theirs is not None and ours == theirs


def test_defaults_and_groups_are_torchs():
    for ours, theirs in ((optim.Adam, torch.optim.Adam), (optim.SGD, torch.optim.SGD)):
        a, b = ours([_param()]), theirs([_param()])
        assert a.defaults == b.defaults
        ga, gb = dict(a.param_groups[0]), dict(b.param_groups[0])
        ga.pop("params"), gb.pop("params")
        assert ga == gb


@pytest.mark.parametrize("kw", [dict(amsgrad=True), dict(maximize=True), dict(foreach=True), dict(fused=True),
                                dict(capturable=True), dict(differentiable=True), dict(decoupled_weight_decay=True)])
def test_adam_refuses_what_it_does_not_implement(kw):
    with pytest.raises(ValueError, match=r"use torch\.optim\.Adam"):
        optim.Adam([_param()], **kw)


@pytest.mark.parametrize("kw", [dict(maximize=True), dict(fused=True)])
def test_sgd_refuses_what_it_does_not_implement(kw):
    with pytest.raises(ValueError, match=r"use torch\.optim\.SGD"):
        optim.SGD([_param()], lr=0.1, **kw)


def test_a_group_added_later_is_checked_at_step():
    p, q = _param(), _param()
    opt = optim.Adam([p])
    opt.add_param_group({"params": [q], "amsgrad": True})
    q.grad = torch.zeros(3)
    with pytest.raises(ValueError, match="amsgrad=True"):
        opt.step()


def test_sparse_gradients_get_torchs_message():
    p = _param()
    p.grad = torch.zeros(3).to_sparse()
    with pytest.raises(RuntimeError, match="Adam does not support sparse gradients, please consider SparseAdam instead"):
        optim.Adam([p]).step()
    with pytest.raises(RuntimeError, match="sparse"):
        optim.SGD([p], lr=0.1).step()


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.3, 0.95), (0.0, 0.5), (0.95, 0.98)])
def test_adam_table_rows_are_torchs_formulas(betas):
    b1, b2 = betas
    table = optim.adam_bias_correction_table(b1, b2, 3000)
    for t in (1, 2, 3, 7, 100, 1023, 2999):
        step = torch.tensor(float(t))  # torch's fp32 CPU step, read with .item()
        bc1 = 1 - b1 ** step.item()
        bc2 = 1 - b2 ** step.item()
        assert table[t, 0].item() == bc2 ** 0.5 and table[t, 1].item() == bc1, t


def test_torch_state_is_converted_on_load():
    p, q = _param(), _param()
    ref = torch.optim.SGD([p], lr=0.1, momentum=0.9)
    ref.state[p]["momentum_buffer"] = torch.ones(3)
    opt = optim.SGD([q], lr=0.1, momentum=0.9)
    opt.load_state_dict(ref.state_dict())
    st = opt.state[q]
    assert st["step"].dtype == torch.int64 and int(st["step"]) == 1  # a saved buffer has been set
    assert torch.equal(st["momentum_buffer"], torch.ones(3))
    ref = torch.optim.Adam([p])
    ref.state[p].update(step=torch.tensor(5.0), exp_avg=torch.ones(3), exp_avg_sq=torch.ones(3))
    opt = optim.Adam([q])
    opt.load_state_dict(ref.state_dict())
    assert opt.state[q]["step"].dtype == torch.int64 and int(opt.state[q]["step"]) == 5 and opt._host_steps == 5


def test_device_table_maps_the_reference_names():
    assert optim.OPTIMIZER_CLASSES == {"sgd": torch.optim.SGD, "adam": torch.optim.Adam, "adamw": optim.AdamW,
                                       "radam": optim.RAdam}
    assert optim.DEVICE_OPTIMIZER_CLASSES == {"sgd": optim.SGD, "adam": optim.Adam, "adamw": optim.AdamW,
                                              "radam": optim.RAdam}


def test_captured_tail_takes_both():
    for opt in (optim.Adam([_param()]), optim.SGD([_param()], lr=0.1)):
        assert optim.CapturedTail(opt)._rule == opt._rule


def test_one_entry_is_declared_and_bound_for_every_rule():
    header = open(os.path.join(ROOT, "include", "qagnn_b200.h")).read()
    assert re.search(r"\bint32_t qagnn_optim_step\s*\(int32_t rule,", header)
    assert "qagnn_optim_step" in _lib.EXPORTS
    for name in ("qagnn_radam_step", "qagnn_adamw_step", "qagnn_adam_step", "qagnn_sgd_step"):
        assert name not in header and name not in _lib.EXPORTS, name
    assert "QAGNN_RULE_RADAM = 0, QAGNN_RULE_ADAMW = 1, QAGNN_RULE_ADAM = 2, QAGNN_RULE_SGD = 3" in header


def _tool(name):
    for cand in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def kernels(tmp_path_factory):
    """csrc/optim.cu and csrc/tail.cu cross-compiled with the library's flags: {kernel: opcode counts} of the Adam and SGD
    kernels."""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("no nvcc / cuobjdump")
    out = {}
    for src in ("optim.cu", "tail.cu"):
        obj = str(tmp_path_factory.mktemp("optim") / (src + ".o"))
        subprocess.run([nvcc, "-c", os.path.join(build.CSRC, src), "-o", obj] + build.NVCC_FLAGS,
                       capture_output=True, text=True, check=True)
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        for body in re.split(r"\n\s*Function : ", sass)[1:]:
            name = re.search(r"\d+((?:tail_)?(?:adam|sgd)_kernel)", body.split("\n", 1)[0])
            if name is None:
                continue
            ops = collections.Counter()
            for line in body.split("\n"):
                m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
                if m:
                    ops[m.group(1)] += 1
            out[name.group(1)] = ops
    return out


def test_adam_and_sgd_kernels_take_vector_loads_and_no_float_atomics(kernels):
    assert set(kernels) == {"adam_kernel", "sgd_kernel", "tail_adam_kernel", "tail_sgd_kernel"}
    for name, ops in kernels.items():
        atomics = [op for op in ops if op.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG", "ATOMS")]
        assert not [op for op in atomics if re.search(r"\.F(16|32|64)", op)], (name, atomics)
        assert sum(ops[op] for op in atomics) == 1, (name, atomics)  # the arrival counter
    for name in ("adam_kernel", "tail_adam_kernel"):
        assert kernels[name]["LDG.E.128"] == 4 and kernels[name]["STG.E.128"] >= 3, name
    for name in ("sgd_kernel", "tail_sgd_kernel"):  # p, g and the momentum buffer
        assert kernels[name]["LDG.E.128"] == 3 and kernels[name]["STG.E.128"] >= 2, name
