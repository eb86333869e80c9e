"""The reference's RAdam (utils/optimization_utils.py) as one multi-tensor sm_90a launch per device (qagnn_radam_step).

`RAdam` takes the reference's arguments and param groups and reproduces its update bit for bit: the same fp32 operations in
the same order, with the same rounding of every Python scalar (csrc/optim.cu).  It differs from the reference in how it runs:
- one kernel launch per device per `step()` (one per 512 tensors), instead of about ten element-wise ops per tensor;
- `state[p]['step']` is an int64 0-dim tensor on p's device, advanced by the kernel, so `step()` never reads the GPU;
- it declares `_step_supports_amp_scaling`: `GradScaler.step` hands it `found_inf` and, when `unscale_` was not called,
  `grad_scale`, and the kernel skips the step or unscales the gradients on the device instead of the scaler's `.item()`.
The step size s and the branch (rectified when rho_t >= 5) depend only on (beta1, beta2, t).  The host builds them in Python
doubles with the reference's formula into a device fp64 table per (device, beta1, beta2), and the kernel indexes it with the
device step.  The host counts its own `step()` calls, which bounds every device step, and grows the table ahead of that count.
"""
import ctypes as C
import math

import torch

from . import _lib

_TABLE_MIN = 1024


def step_size_row(beta1, beta2, t):
    """(rectified, s) of the reference's RAdam at step t >= 1: rectified is 1.0 when rho_t >= 5, and s is then the rectified
    step size, else 1 / (1 - beta1^t), its SGD step size.  The reference's formula and evaluation order, in Python doubles."""
    beta2_t = beta2 ** t
    n_sma_max = 2 / (1 - beta2) - 1
    n_sma = n_sma_max - 2 * t * beta2_t / (1 - beta2_t)
    if n_sma >= 5:
        return 1.0, math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_sma_max - 4) * (n_sma - 2) / n_sma * n_sma_max / (n_sma_max - 2)) / (
            1 - beta1 ** t)
    return 0.0, 1.0 / (1 - beta1 ** t)


def step_size_table(beta1, beta2, length):
    """fp64 [length, 2]: row t is step_size_row(beta1, beta2, t); row 0 (never indexed) is (0, 0)."""
    rows = [(0.0, 0.0)] + [step_size_row(beta1, beta2, t) for t in range(1, length)]
    return torch.tensor(rows, dtype=torch.float64)


def _check_hyper(lr, betas, eps):
    # the reference's checks and messages
    if not 0.0 <= lr:
        raise ValueError("Invalid learning rate: {}".format(lr))
    if not 0.0 <= eps:
        raise ValueError("Invalid epsilon value: {}".format(eps))
    if not 0.0 <= betas[0] < 1.0:
        raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
    if not 0.0 <= betas[1] < 1.0:
        raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))


def _check_tensor(t, what):
    if not t.is_cuda:
        raise TypeError(f"qagnn_b200.optim.RAdam: the {what} must live on a CUDA device (got {t.device}); there is no CPU path")
    if t.dtype != torch.float32:
        raise TypeError(f"qagnn_b200.optim.RAdam: the {what} must be float32 (got {t.dtype})")
    if not t.is_contiguous():
        raise ValueError(f"qagnn_b200.optim.RAdam: the {what} must be contiguous")


class RAdam(torch.optim.Optimizer):
    """RAdam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, degenerated_to_sgd=True): the reference's
    `utils.optimization_utils.RAdam`, stepped on the GPU.  Parameters and their gradients must be contiguous fp32 CUDA
    tensors; a parameter whose `.grad` is None is skipped and its step does not advance.  `lr` (and every other
    hyperparameter) is read from each group at every `step()`, so LambdaLR schedules work as with the reference."""

    _step_supports_amp_scaling = True

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, degenerated_to_sgd=True):
        _check_hyper(lr, betas, eps)
        self.degenerated_to_sgd = degenerated_to_sgd
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._host_steps = 0  # step() calls: no device step counter exceeds it
        self._tables = {}  # (device, beta1, beta2) -> (device table, its pinned staging copy)
        self._counters = {}  # device -> int32 arrival counter of the kernel

    def _table(self, device, beta1, beta2):
        key = (device, beta1, beta2)
        have = self._tables.get(key)
        if have is not None and have[0].shape[0] > self._host_steps:
            return have[0]
        length = max(_TABLE_MIN, 1 << (2 * self._host_steps + 1).bit_length())
        # a fresh pinned buffer per upload, written before its copy is enqueued and never written again
        staging = step_size_table(beta1, beta2, length).pin_memory()
        table = staging.to(device, non_blocking=True)
        self._tables[key] = (table, staging)
        return table

    def _counter(self, device):
        c = self._counters.get(device)
        if c is None:
            c = self._counters[device] = torch.zeros(1, dtype=torch.int32, device=device)
        return c

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        work = {}  # device -> [(group index, p)]
        for gi, group in enumerate(self.param_groups):
            _check_hyper(group["lr"], group["betas"], group["eps"])
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("RAdam does not support sparse gradients")
                _check_tensor(p, "parameter")
                _check_tensor(p.grad, "gradient")
                if p.grad.shape != p.shape or p.grad.device != p.device:
                    raise ValueError(f"qagnn_b200.optim.RAdam: a gradient of shape {tuple(p.grad.shape)} on {p.grad.device} "
                                     f"for a parameter of shape {tuple(p.shape)} on {p.device}")
                work.setdefault(p.device, []).append((gi, p))
        if not work:
            return loss
        self._host_steps += 1
        found_inf = getattr(self, "found_inf", None)
        grad_scale = getattr(self, "grad_scale", None)
        lib = _lib.load()
        n_groups = len(self.param_groups)
        hyper = [(float(g["lr"]), float(g["weight_decay"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]))
                 for g in self.param_groups]
        arr = lambda ct, vals: (ct * len(vals))(*vals)  # noqa: E731
        lr, wd, b1, b2, eps = (arr(C.c_double, col) for col in zip(*hyper))
        degenerated = arr(C.c_int32, [int(bool(self.degenerated_to_sgd))] * n_groups)
        for device, items in work.items():
            states = []
            for _, p in items:
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.zeros((), dtype=torch.int64, device=device)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                states.append(st)
            tables = [None] * n_groups
            for gi in {gi for gi, _ in items}:
                tables[gi] = self._table(device, hyper[gi][2], hyper[gi][3])
            length = min(t.shape[0] for t in tables if t is not None)
            # GradScaler keeps found_inf and the scale on its own device: the copies to this one are enqueued, never read
            fi = None if found_inf is None else found_inf.to(device, torch.float32, non_blocking=True)
            gs = None if grad_scale is None else grad_scale.to(device, torch.float32, non_blocking=True)
            n = len(items)
            ptrs = lambda ts: arr(C.c_void_p, [t.data_ptr() for t in ts])  # noqa: E731
            with torch.cuda.device(device):
                _lib.check(lib.qagnn_radam_step(
                    n, ptrs([p for _, p in items]), ptrs([p.grad for _, p in items]), ptrs([s["exp_avg"] for s in states]),
                    ptrs([s["exp_avg_sq"] for s in states]), ptrs([s["step"] for s in states]),
                    arr(C.c_int64, [p.numel() for _, p in items]), arr(C.c_int32, [gi for gi, _ in items]), n_groups,
                    lr, wd, b1, b2, eps, degenerated,
                    arr(C.c_void_p, [0 if t is None else t.data_ptr() for t in tables]), length,
                    _lib.ptr(fi), _lib.ptr(gs), _lib.ptr(self._counter(device)), _lib.stream_ptr(device)), "qagnn_radam_step")
        return loss

    def load_state_dict(self, state_dict):
        """Loads this optimiser's state_dict or the reference RAdam's, whose 'step' is a Python int.  Every step becomes an
        int64 0-dim tensor on its parameter's device, and the step counts are read once to bound the step-size tables."""
        super().load_state_dict(state_dict)
        top = self._host_steps
        steps = {}
        for group in self.param_groups:
            group.pop("buffer", None)  # the reference's host cache of step sizes
            for p in group["params"]:
                st = self.state.get(p)
                if not st:
                    continue
                step = st["step"]
                if isinstance(step, torch.Tensor):
                    step = step.to(device=p.device, dtype=torch.int64).reshape(())
                else:
                    step = torch.tensor(int(step), dtype=torch.int64, device=p.device)
                st["step"] = step
                for k in ("exp_avg", "exp_avg_sq"):
                    st[k] = st[k].to(device=p.device, dtype=torch.float32).contiguous()
                steps.setdefault(p.device, []).append(step)
        for ss in steps.values():
            top = max(top, int(torch.stack(ss).max()))
        self._host_steps = top
