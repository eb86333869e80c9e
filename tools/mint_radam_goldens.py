"""Mints tests/golden/ref/radam.pt: trajectories of the reference's OWN RAdam (utils/optimization_utils.py) on the CPU.

    python tools/mint_radam_goldens.py            # writes tests/golden/ref/radam.pt
    python tools/mint_radam_goldens.py --check    # re-mints in memory and compares with the committed file, writes nothing

Needs the reference tree (QAGNN_REFERENCE_ROOT, see oracle/ref_shim.py).  Its module imports `transformers.AdamW`, which the
installed transformers no longer has, so the import runs with that one name stubbed; RAdam itself runs verbatim.

Each case records the initial parameters, the gradient of every parameter at every step (None where the parameter gets no
gradient) and, after every step, each parameter with its exp_avg, exp_avg_sq and step.  tests/test_optim_cpu.py replays the
gradients through tests/radam_oracle.py and requires every recorded tensor bit for bit.
"""
import importlib
import os
import sys
import types
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.ref_shim import REFERENCE_ROOT  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref", "radam.pt")
STEPS = 12  # across rho_t = 5 at beta2 = 0.999 (steps 1-5 take the SGD branch)

# name -> (constructor kwargs, [(group kwargs, [param shapes])], {param index: steps without a gradient})
CASES = {
    "two_groups_dlr": (dict(lr=1e-3, weight_decay=0.01), [(dict(weight_decay=0.01), [(7, 5), (3,)]),
                                                          (dict(weight_decay=0.0), [(5,), (2, 2)])], {}),
    "two_groups_elr": (dict(lr=1e-5, weight_decay=0.01), [(dict(weight_decay=0.01), [(6, 4)]),
                                                          (dict(weight_decay=0.0), [(4,)])], {}),
    "other_betas": (dict(lr=1e-3, weight_decay=0.01), [(dict(betas=(0.8, 0.99)), [(5, 3)]),
                                                       (dict(weight_decay=0.0), [(3,)])], {}),
    "no_sgd": (dict(lr=1e-3, weight_decay=0.01, degenerated_to_sgd=False), [(dict(), [(4, 4)]),
                                                                             (dict(weight_decay=0.0), [(4,)])], {}),
    "grad_none": (dict(lr=1e-3, weight_decay=0.01), [(dict(), [(3, 3), (5,)]), (dict(weight_decay=0.0), [(2,)])],
                  {1: {2, 3, 7}, 2: {0}}),
}


def _reference_radam():
    stub = types.ModuleType("transformers")
    stub.AdamW = type("AdamW", (), {})
    saved = sys.modules.get("transformers")
    sys.modules["transformers"] = stub
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        return importlib.import_module("utils.optimization_utils").RAdam
    finally:
        sys.path.remove(REFERENCE_ROOT)
        if saved is None:
            del sys.modules["transformers"]
        else:
            sys.modules["transformers"] = saved


def mint_case(radam_cls, name, spec, seed):
    kwargs, groups, missing = spec
    g = torch.Generator().manual_seed(seed)
    params, param_groups = [], []
    for gk, shapes in groups:
        ps = [torch.nn.Parameter(torch.randn(*s, generator=g)) for s in shapes]
        params += ps
        param_groups.append(dict(gk, params=ps))
    rec = {"kwargs": kwargs, "groups": [gk for gk, _ in groups], "group_sizes": [len(s) for _, s in groups],
           "init": [p.detach().clone() for p in params], "grads": [], "after": []}
    opt = radam_cls(param_groups, **kwargs)
    for t in range(STEPS):
        grads = []
        for i, p in enumerate(params):
            gr = None if t in missing.get(i, ()) else torch.randn(p.shape, generator=g) * 10.0 ** float(torch.randint(-4, 1, (1,), generator=g))
            p.grad = gr
            grads.append(None if gr is None else gr.clone())
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # the reference's deprecated add_ / addcmul_ overloads
            opt.step()
        rec["grads"].append(grads)
        rec["after"].append([{"param": p.detach().clone(),
                              **({k: opt.state[p][k].clone() for k in ("exp_avg", "exp_avg_sq")} if opt.state[p] else {}),
                              "step": opt.state[p]["step"] if opt.state[p] else 0} for p in params])
    return rec


def mint():
    radam = _reference_radam()
    return {name: mint_case(radam, name, spec, seed) for seed, (name, spec) in enumerate(CASES.items())}


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def main():
    got = mint()
    if "--check" in sys.argv[1:]:
        have = torch.load(GOLDEN, weights_only=False)
        bad = [n for n in got if n not in have or not _same(got[n], have[n])]
        print("radam.pt: " + ("identical" if not bad and have.keys() == got.keys() else f"differs in {bad or 'its case list'}"))
        sys.exit(1 if bad or have.keys() != got.keys() else 0)
    os.makedirs(os.path.dirname(GOLDEN), exist_ok=True)
    torch.save(got, GOLDEN)
    print("wrote", GOLDEN, {n: len(r["after"]) for n, r in got.items()})


if __name__ == "__main__":
    main()
