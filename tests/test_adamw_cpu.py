"""qagnn_b200.optim.AdamW without a GPU: the eager restatement of transformers' AdamW (tests/adamw_oracle.py) against the
closed form of its update in fp64, and against torch.optim.AdamW, which it must not be; the bias-correction table against
transformers' formula bit for bit and its growth; the argument checks; the reference's optimiser table built on its
grouped_parameters; loading transformers' state; and the compiled kernels (0 spills for both rules, RAdam's SASS unchanged)."""
import collections
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from qagnn_b200 import build, optim
from tests.adamw_oracle import AdamWOracle


def _grad_seq(shape, steps, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(shape, generator=g, dtype=torch.float64).to(dtype) * 10.0 ** (-(t % 3)) for t in range(steps)]


@pytest.mark.parametrize("correct_bias", [True, False])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("eps", [1e-6, 1e-8])
def test_oracle_is_bias_corrected_adam_with_eps_outside_and_decay_after(correct_bias, wd, eps):
    """fp64: m and v as weighted sums of every gradient so far, eps added to sqrt(v) unscaled, the step size
    lr sqrt(1 - b2^t) / (1 - b1^t), and the decay p (1 - lr wd) applied to the updated p."""
    lr, b1, b2, steps = 1e-2, 0.9, 0.999, 30
    p0 = torch.randn(257, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    grads = _grad_seq(p0.shape, steps, 2, torch.float64)
    p = torch.nn.Parameter(p0.clone())
    opt = AdamWOracle([p], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, correct_bias=correct_bias)
    want = p0.numpy().copy()
    G = np.stack([g.numpy() for g in grads])
    for t in range(1, steps + 1):
        p.grad = grads[t - 1].clone()
        opt.step()
        w1 = (1 - b1) * b1 ** np.arange(t - 1, -1, -1.0)
        w2 = (1 - b2) * b2 ** np.arange(t - 1, -1, -1.0)
        m = (w1[:, None] * G[:t]).sum(0)
        v = (w2[:, None] * G[:t] ** 2).sum(0)
        c = math.sqrt(1 - b2 ** t) / (1 - b1 ** t) if correct_bias else 1.0
        want = (want - lr * c * m / (np.sqrt(v) + eps)) * (1 - lr * wd)
        np.testing.assert_allclose(opt.state[p]["exp_avg"].numpy(), m, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(opt.state[p]["exp_avg_sq"].numpy(), v, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(p.detach().numpy(), want, rtol=1e-12, atol=1e-15)
        assert opt.state[p]["step"] == t


def test_oracle_is_not_torch_adamw():
    """torch decays first (p (1 - lr wd)) and divides sqrt(v) by sqrt(bc2) before adding eps: another fp32 trajectory."""
    kw = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01)
    p0 = torch.randn(4096, generator=torch.Generator().manual_seed(3))
    grads = _grad_seq(p0.shape, 20, 4, torch.float32)
    out = []
    for cls in (AdamWOracle, torch.optim.AdamW):
        p = torch.nn.Parameter(p0.clone())
        opt = cls([p], **kw)
        for g in grads:
            p.grad = g.clone()
            opt.step()
        out.append(p.detach())
    assert not torch.equal(out[0], out[1])
    torch.testing.assert_close(out[0], out[1], rtol=1e-3, atol=1e-4)  # the same optimiser family all the same


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.8, 0.99), (0.0, 0.5), (0.95, 0.9999), (0.9, 0.0)])
def test_bias_correction_table_equals_transformers_formula(betas):
    b1, b2 = betas
    n = 100_001
    table = optim.bias_correction_table(b1, b2, n)
    assert table.dtype == torch.float64 and table.shape == (n, 2)
    sq, bc1 = table[:, 0].tolist(), table[:, 1].tolist()
    for t in range(1, n):
        assert sq[t] == math.sqrt(1.0 - b2 ** t) and bc1[t] == 1.0 - b1 ** t, (betas, t)  # exact: the same doubles
    # the kernel forms the step size as (lr * sq) / bc1 in IEEE fp64: transformers' `lr * math.sqrt(bc2) / bc1`
    for lr in (1e-3, 2e-5, 0.1, 3.7e-4):
        for t in (1, 2, 7, 150, 10_000):
            assert lr * sq[t] / bc1[t] == lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)


def test_the_table_grows_ahead_of_the_host_step_count(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)  # no CUDA host allocator here
    opt = optim.AdamW([torch.nn.Parameter(torch.zeros(3))])
    first = opt._table("cpu", 0.9, 0.999)
    assert first.shape[0] == 1024 and opt._table("cpu", 0.9, 0.999) is first
    opt._host_steps = 1024
    grown = opt._table("cpu", 0.9, 0.999)
    assert grown.shape[0] > 1024 and grown is not first
    assert torch.equal(grown, optim.bias_correction_table(0.9, 0.999, grown.shape[0]))
    assert grown[1500].tolist() == [math.sqrt(1.0 - 0.999 ** 1500), 1.0 - 0.9 ** 1500]


def test_arguments_are_checked_as_transformers_checks_them():
    p = [torch.nn.Parameter(torch.zeros(3))]
    for kw, msg in [(dict(lr=-1e-3), r"Invalid learning rate: -0.001 - should be >= 0.0"),
                    (dict(eps=-1.0), r"Invalid epsilon value: -1.0 - should be >= 0.0"),
                    (dict(betas=(1.0, 0.999)), r"Invalid beta parameter: 1.0 - should be in \[0.0, 1.0\["),
                    (dict(betas=(-0.1, 0.999)), r"Invalid beta parameter: -0.1 - should be in \[0.0, 1.0\["),
                    (dict(betas=(0.9, 1.0)), r"Invalid beta parameter: 1.0 - should be in \[0.0, 1.0\[")]:
        with pytest.raises(ValueError, match=msg):
            optim.AdamW(p, **kw)
    opt = optim.AdamW(p, lr=0.0, eps=0.0, betas=(0.0, 0.0), weight_decay=0.01, correct_bias=False)
    assert opt.defaults == dict(lr=0.0, betas=(0.0, 0.0), eps=0.0, weight_decay=0.01, correct_bias=False)
    assert optim.AdamW(p).defaults == dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True)


def test_a_group_with_bad_betas_is_refused_at_step():
    p = torch.nn.Parameter(torch.zeros(3))
    opt = optim.AdamW([dict(params=[p], betas=(0.9, 1.0))])
    p.grad = torch.zeros(3)
    with pytest.raises(ValueError, match="Invalid beta parameter: 1.0"):
        opt.step()


def test_cpu_tensors_and_sparse_grads_are_refused():
    p = torch.nn.Parameter(torch.zeros(3))
    opt = optim.AdamW([p])
    opt.step()  # no gradient: nothing to do
    p.grad = torch.zeros(3)
    with pytest.raises(TypeError, match=r"qagnn_b200\.optim\.AdamW: the parameter must live on a CUDA device"):
        opt.step()
    p.grad = torch.zeros(3).to_sparse()
    with pytest.raises(RuntimeError, match="Adam does not support sparse gradients"):
        opt.step()
    assert len(opt.state) == 0
    # RAdam keeps its own name in the messages it shares with AdamW
    r = optim.RAdam([p])
    p.grad = torch.zeros(3)
    with pytest.raises(TypeError, match=r"qagnn_b200\.optim\.RAdam: the parameter must live on a CUDA device"):
        r.step()


def test_optimizer_contract():
    assert optim.AdamW._step_supports_amp_scaling is True and optim.RAdam._step_supports_amp_scaling is True
    assert issubclass(optim.AdamW, torch.optim.Optimizer)


class _Model(torch.nn.Module):
    """An encoder and a decoder with weights, biases and LayerNorms, named as qagnn.py's grouping expects."""

    def __init__(self):
        super().__init__()
        self.encoder = torch.nn.Sequential(torch.nn.Linear(8, 8), torch.nn.Linear(8, 8))
        self.encoder.add_module("LayerNorm", torch.nn.LayerNorm(8))
        self.decoder = torch.nn.Sequential(torch.nn.Linear(8, 4), torch.nn.Linear(4, 1, bias=False))
        self.decoder.add_module("LayerNorm", torch.nn.LayerNorm(4))


def _grouped_parameters(model, weight_decay=0.01, encoder_lr=2e-5, decoder_lr=1e-3):
    # qagnn.py:172-178
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
    return [
        {'params': [p for n, p in model.encoder.named_parameters() if not any(nd in n for nd in no_decay)], 'weight_decay': weight_decay, 'lr': encoder_lr},
        {'params': [p for n, p in model.encoder.named_parameters() if any(nd in n for nd in no_decay)], 'weight_decay': 0.0, 'lr': encoder_lr},
        {'params': [p for n, p in model.decoder.named_parameters() if not any(nd in n for nd in no_decay)], 'weight_decay': weight_decay, 'lr': decoder_lr},
        {'params': [p for n, p in model.decoder.named_parameters() if any(nd in n for nd in no_decay)], 'weight_decay': 0.0, 'lr': decoder_lr},
    ]


def test_the_reference_optimiser_table_builds_every_optim_value():
    from qagnn_b200.optim import OPTIMIZER_CLASSES
    assert OPTIMIZER_CLASSES == {"sgd": torch.optim.SGD, "adam": torch.optim.Adam, "adamw": optim.AdamW, "radam": optim.RAdam}
    model = _Model()
    for name in ("sgd", "adam", "adamw", "radam"):
        gp = _grouped_parameters(model)
        opt = OPTIMIZER_CLASSES[name](gp)  # qagnn.py:180
        assert isinstance(opt, torch.optim.Optimizer), name
        assert [len(g["params"]) for g in opt.param_groups] == [len(g["params"]) for g in gp] == [2, 4, 2, 3], name
        assert [g["lr"] for g in opt.param_groups] == [2e-5, 2e-5, 1e-3, 1e-3], name
        assert [g["weight_decay"] for g in opt.param_groups] == [0.01, 0.0, 0.01, 0.0], name
    assert OPTIMIZER_CLASSES["adamw"](_grouped_parameters(model)).param_groups[0]["eps"] == 1e-6


def test_transformers_state_with_an_int_step_loads():
    """transformers' state_dict: 'step' a Python int, its group keys (correct_bias included) as AdamW keeps them."""
    torch.manual_seed(5)
    ps = [torch.nn.Parameter(torch.randn(7)), torch.nn.Parameter(torch.randn(2, 3))]
    ref = AdamWOracle([dict(params=[ps[0]]), dict(params=[ps[1]], weight_decay=0.0, correct_bias=False)], lr=1e-3,
                      weight_decay=0.01)
    for t in range(5):
        for p in ps:
            p.grad = torch.randn_like(p)
        if t == 2:
            ps[1].grad = None
        ref.step()
    sd = ref.state_dict()
    assert all(isinstance(st["step"], int) for st in sd["state"].values())
    qs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    opt = optim.AdamW([dict(params=[qs[0]]), dict(params=[qs[1]])], lr=5.0)
    opt.load_state_dict(sd)
    assert opt.param_groups[0]["lr"] == 1e-3 and opt.param_groups[1]["correct_bias"] is False
    assert opt.param_groups[1]["weight_decay"] == 0.0
    for p, q in zip(ps, qs):
        st = opt.state[q]
        assert st["step"].dtype == torch.int64 and st["step"].dim() == 0 and int(st["step"]) == ref.state[p]["step"]
        for k in ("exp_avg", "exp_avg_sq"):
            assert st[k].dtype == torch.float32 and torch.equal(st[k], ref.state[p][k])
    assert [int(opt.state[q]["step"]) for q in qs] == [5, 4] and opt._host_steps == 5


# ---- the compiled kernels ------------------------------------------------------------------------------------------

# radam_kernel's SASS opcode counts as CUDA 12.9's nvcc compiles csrc/optim.cu (-O3, sm_90a) before the update rule became a
# template parameter: the RAdam instantiation must compile to the same code.
RADAM_OPCODES = {
    "ATOMG.E.ADD.STRONG.GPU": 1, "BAR.SYNC.DEFER_BLOCKING": 2, "BRA": 122, "BSSY": 30, "BSYNC": 30, "CALL.REL.NOINC": 23,
    "CCTL.IVALL": 2, "CGAERRBAR": 2, "DFMA": 18, "DMUL": 4, "DSETP.GTU.AND": 1, "DSETP.NEU.AND": 1, "ERRBAR": 2, "EXIT": 3,
    "F2F.F32.F64": 2, "F2F.F64.F32": 1, "FADD": 11, "FADD.FTZ": 4, "FCHK": 11, "FFMA": 144, "FFMA.RM": 1, "FFMA.RP": 1,
    "FFMA.RZ": 1, "FMUL": 44, "FMUL.FTZ": 25, "FSETP.GEU.AND": 1, "FSETP.GEU.FTZ.AND": 1, "FSETP.GTU.FTZ.AND": 3,
    "FSETP.NEU.AND": 1, "FSETP.NEU.FTZ.AND": 5, "HFMA2.MMA": 4, "IADD3": 47, "IADD3.X": 22, "IMAD": 4, "IMAD.IADD": 2,
    "IMAD.MOV": 1, "IMAD.MOV.U32": 38, "IMAD.SHL.U32": 2, "IMAD.U32": 5, "IMAD.WIDE": 5, "IMAD.WIDE.U32": 4, "IMAD.X": 10,
    "ISETP.GE.AND": 7, "ISETP.GE.AND.EX": 3, "ISETP.GE.U32.AND": 8, "ISETP.GE.U32.AND.EX": 1, "ISETP.GT.AND": 1,
    "ISETP.GT.AND.EX": 3, "ISETP.GT.U32.AND": 14, "ISETP.GT.U32.OR": 1, "ISETP.LT.AND.EX": 1, "ISETP.LT.U32.AND": 2,
    "ISETP.NE.AND": 38, "ISETP.NE.AND.EX": 5, "ISETP.NE.OR": 1, "ISETP.NE.U32.AND": 5, "LDC": 3, "LDC.64": 9, "LDG.E": 30,
    "LDG.E.128": 4, "LDG.E.64": 8, "LDS.U8": 1, "LEA": 2, "LEA.HI": 1, "LEA.HI.X": 1, "LOP3.LUT": 27, "MEMBAR.SC.GPU": 2,
    "MOV": 69, "MUFU.RCP": 12, "MUFU.RCP64H": 3, "MUFU.RSQ": 13, "NOP": 15, "PLOP3.LUT": 20, "PRMT": 5, "R2UR": 3,
    "RET.REL.NODEC": 3, "S2R": 2, "S2UR": 4, "SEL": 10, "SHF.L.U32": 1, "SHF.L.U64.HI": 2, "SHF.R.U32.HI": 5,
    "SHF.R.U64": 1, "STG.E": 29, "STG.E.128": 4, "STG.E.64": 5, "STS.U8": 1, "UIADD3": 12, "UIADD3.X": 2, "UIMAD": 2,
    "UIMAD.WIDE": 5, "UISETP.EQ.OR": 1, "UISETP.GE.AND": 3, "UISETP.GT.AND": 1, "UISETP.LT.AND.EX": 1,
    "UISETP.LT.U32.AND": 1, "UISETP.NE.AND": 12, "UISETP.NE.AND.EX": 1, "UISETP.NE.U32.AND": 1, "ULDC": 8, "ULDC.64": 16,
    "ULDC.U8": 2, "ULEA": 9, "ULOP3.LUT": 5, "UMOV": 17, "USEL": 3, "USHF.L.U32": 1, "USHF.R.S32.HI": 2, "USHF.R.S64": 1,
    "USHF.R.U32.HI": 1, "VIADD": 17, "VIADDMNMX": 1, "VOTEU.ANY": 1,
}


def _tool(name):
    for cand in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """csrc/optim.cu cross-compiled with the library's flags: (ptxas report, {kernel: opcode counts}, nvcc version text)."""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("no nvcc / cuobjdump")
    obj = str(tmp_path_factory.mktemp("optim") / "optim.o")
    r = subprocess.run([nvcc, "-c", os.path.join(build.CSRC, "optim.cu"), "-o", obj] + build.NVCC_FLAGS,
                       capture_output=True, text=True, check=True)
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        ops = collections.Counter()
        for line in body.split("\n"):
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                ops[m.group(1)] += 1
        kernels[body.split("\n", 1)[0].strip()] = ops
    version = subprocess.run([nvcc, "--version"], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, kernels, version


def _kernel(kernels, name):
    found = [ops for k, ops in kernels.items() if f"{name}E" in k]
    assert len(found) == 1, (name, list(kernels))
    return found[0]


def test_radam_and_adamw_compile_without_spills_among_four_kernels(compiled):
    report, _, _ = compiled
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\n.*?Used (\d+) registers", report)
    got = {re.search(r"(?:radam|adamw|adam|sgd)_kernel", n).group(0): tuple(int(x) for x in rest) for n, *rest in props}
    assert set(got) == {"radam_kernel", "adamw_kernel", "adam_kernel", "sgd_kernel"}, report
    got = {name: got[name] for name in ("radam_kernel", "adamw_kernel")}
    for name, (stack, stores, loads, regs) in got.items():
        assert stack == stores == loads == 0, (name, report)
    assert got["radam_kernel"][3] == 40


def test_radam_compiles_to_the_same_code(compiled):
    _, kernels, version = compiled
    if "release 12.9" not in version:
        pytest.skip("the opcode counts are CUDA 12.9's")
    assert dict(_kernel(kernels, "12radam_kernel")) == RADAM_OPCODES


def test_both_rules_take_vector_loads_and_no_float_atomics(compiled):
    _, kernels, _ = compiled
    for name in ("12radam_kernel", "12adamw_kernel"):
        ops = _kernel(kernels, name)
        assert ops["LDG.E.128"] == 4 and ops["STG.E.128"] >= 3, name
        assert not [op for op in ops if op.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG") and re.search(r"\.F(16|32|64)", op)]
