"""The reference's optimisers as one multi-tensor sm_90a launch per device (csrc/optim.cu, qagnn_optim_step).

`RAdam` is the reference's `utils.optimization_utils.RAdam` and `AdamW` is transformers' `AdamW` (3.4.0, the version the
reference pins).  `Adam` and `SGD` are torch.optim's, as torch 2.11 steps them by default on CUDA.  Each takes its
original's arguments and param groups and reproduces its update bit for bit: the same fp32 operations in the same order,
with the same rounding of every Python scalar.  They differ from the originals in how they run:
- one kernel launch per device per `step()` (one per 512 tensors), instead of about ten element-wise ops per tensor;
- `state[p]['step']` is an int64 0-dim tensor on p's device, advanced by the kernel, so `step()` never reads the GPU;
- they declare `_step_supports_amp_scaling`: `GradScaler.step` hands them `found_inf` and, when `unscale_` was not called,
  `grad_scale`, and the kernel skips the step or unscales the gradients on the device instead of the scaler's `.item()`.
What depends on the step t alone (RAdam's step size and branch, AdamW's and Adam's bias corrections) is computed on the host in Python
doubles with the original's formula, into a device fp64 table per (device, beta1, beta2) that the kernel indexes with the
device step.  The host counts its own `step()` calls, which bounds every device step, and grows the table ahead of that count.

`OPTIMIZER_CLASSES` is the reference's `--optim` table, so `from qagnn_b200.optim import OPTIMIZER_CLASSES` replaces the
reference's import, whose module no longer loads with current `transformers`; `DEVICE_OPTIMIZER_CLASSES` maps the same names
to the four device optimisers.  `clip_grad_norm_` is the recipe's
`torch.nn.utils.clip_grad_norm_` in two launches per device (csrc/clip.cu) instead of torch's three foreach passes, so
the optimiser tail `scaler.unscale_; clip_grad_norm_; scaler.step; scaler.update` never reads the GPU.  `CapturedTail` runs
that whole tail, scheduler step included, as one CUDA graph replay of two launches (csrc/tail.cu).
"""
import ctypes as C
import functools
import math

import torch
from torch.amp.grad_scaler import OptState

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


def bias_correction_row(beta1, beta2, t):
    """(math.sqrt(bias_correction2), bias_correction1) of transformers' AdamW at step t >= 1, in Python doubles as it forms
    them; its step size is lr * row[0] / row[1]."""
    return math.sqrt(1.0 - beta2 ** t), 1.0 - beta1 ** t


def adam_bias_correction_row(beta1, beta2, t):
    """(bias_correction2_sqrt, bias_correction1) of torch.optim.Adam's default CUDA step at step t >= 1, in Python doubles as
    torch forms them from its fp32 step count; its step size is (lr / row[1]) * -1."""
    t = float(t)
    return (1 - beta2 ** t) ** 0.5, 1 - beta1 ** t


def step_table(row, beta1, beta2, length):
    """fp64 [length, 2]: row t is row(beta1, beta2, t), one of the *_row functions above; row 0 (never indexed) is (0, 0)."""
    rows = [(0.0, 0.0)] + [row(beta1, beta2, t) for t in range(1, length)]
    return torch.tensor(rows, dtype=torch.float64)


# each rule's table(beta1, beta2, length)
step_size_table = functools.partial(step_table, step_size_row)
bias_correction_table = functools.partial(step_table, bias_correction_row)
adam_bias_correction_table = functools.partial(step_table, adam_bias_correction_row)


def _arr(ct, vals):
    return (ct * len(vals))(*vals)


def _ptrs(ts):
    """A void* array of the tensors' addresses, None a null pointer."""
    return _arr(C.c_void_p, [None if t is None else t.data_ptr() for t in ts])


def _tensor_arrays(items, states, moments):
    """The per-tensor arrays of qagnn_optim_step and qagnn_step_tail for [(group index, p)], their states and
    [(exp_avg, exp_avg_sq)]: params, grads, exp_avgs, exp_avg_sqs, steps, numels and group_index."""
    return (_ptrs([p for _, p in items]), _ptrs([p.grad for _, p in items]), _ptrs([m for m, _ in moments]),
            _ptrs([v for _, v in moments]), _ptrs([s["step"] for s in states]),
            _arr(C.c_int64, [p.numel() for _, p in items]), _arr(C.c_int32, [gi for gi, _ in items]))


def _refuse(name, options):
    """ValueError for options set to what the device step does not implement: [(option, value)] that must be falsy."""
    on = [k for k, v in options if v]
    if on:
        raise ValueError(f"qagnn_b200.optim.{name}: {', '.join(f'{k}=True' for k in on)} is not implemented on the device; "
                         f"use torch.optim.{name} for it")


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


def _check_adamw_hyper(lr, betas, eps):
    # transformers' checks and messages
    if lr < 0.0:
        raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
    if not 0.0 <= betas[0] < 1.0:
        raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[0]))
    if not 0.0 <= betas[1] < 1.0:
        raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[1]))
    if not 0.0 <= eps:
        raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(eps))


def _check_tensor(t, what, name):
    if not t.is_cuda:
        raise TypeError(f"qagnn_b200.optim.{name}: the {what} must live on a CUDA device (got {t.device}); there is no CPU path")
    if t.dtype != torch.float32:
        raise TypeError(f"qagnn_b200.optim.{name}: the {what} must be float32 (got {t.dtype})")
    if not t.is_contiguous():
        raise ValueError(f"qagnn_b200.optim.{name}: the {what} must be contiguous")


class _DeviceStepOptimizer(torch.optim.Optimizer):
    """What RAdam, AdamW, Adam and SGD share: the per-device work lists, the state, the step tables, the kernel's arrival
    counter, the GradScaler hand-off and state_dict loading.  A subclass names its update rule (`_rule`, QAGNN_RULE_*), its
    table builder (`_table_rows`, fp64 [length, 2] for (beta1, beta2); None for no table), its state tensors (`_state_keys`: the entry's
    exp_avgs and exp_avg_sqs), its original's sparse-gradient message and host caches in the groups, and supplies
    `_check_group` and `_rule_flags` (one int32 per group: the entry's per-group flag)."""

    _step_supports_amp_scaling = True
    _rule = None
    _table_rows = None
    _state_keys = ("exp_avg", "exp_avg_sq")
    _sparse_message = None
    _host_caches = ()

    @staticmethod
    def _hyper(group):
        """The entry's per-group doubles (lr, weight_decay, beta1, beta2, eps)."""
        return float(group["lr"]), float(group["weight_decay"]), float(group["betas"][0]), float(group["betas"][1]), float(
            group["eps"])

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
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
        staging = self._table_rows(beta1, beta2, length).pin_memory()
        table = staging.to(device, non_blocking=True)
        self._tables[key] = (table, staging)
        return table

    def _counter(self, device):
        c = self._counters.get(device)
        if c is None:
            c = self._counters[device] = torch.zeros(1, dtype=torch.int32, device=device)
        return c

    def _state_for(self, p, group):
        st = self.state[p]
        if len(st) == 0:
            st["step"] = torch.zeros((), dtype=torch.int64, device=p.device)
            for k in self._state_keys:
                st[k] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        return st

    def _state_tensors(self, st):
        """The entry's exp_avgs[i] and exp_avg_sqs[i] of one parameter's state (None: a null pointer)."""
        return st["exp_avg"], st["exp_avg_sq"]

    def _group_tables(self, device, hyper, groups):
        """Each listed group's step table on device (None for the others, and for a rule without tables) and the shortest
        table's length."""
        tables = [None] * len(hyper)
        if self._table_rows is None:
            return tables, 0
        for gi in groups:
            tables[gi] = self._table(device, hyper[gi][2], hyper[gi][3])
        return tables, min(t.shape[0] for t in tables if t is not None)

    def _items(self, name, check_dense):
        """[(group index, p)] of the parameters with a gradient, every group checked with `_check_group` and every gradient
        against its parameter, in the messages of `name`.  check_dense(grad) raises the caller's error for a gradient that
        is not dense."""
        items = []
        for gi, group in enumerate(self.param_groups):
            self._check_group(group)
            for p in group["params"]:
                if p.grad is None:
                    continue
                check_dense(p.grad)
                _check_tensor(p, "parameter", name)
                _check_tensor(p.grad, "gradient", name)
                if p.grad.shape != p.shape or p.grad.device != p.device:
                    raise ValueError(f"qagnn_b200.optim.{name}: a gradient of shape {tuple(p.grad.shape)} on {p.grad.device} "
                                     f"for a parameter of shape {tuple(p.shape)} on {p.device}")
                items.append((gi, p))
        return items

    def _check_sparse(self, grad):
        if grad.is_sparse:
            raise RuntimeError(self._sparse_message)

    def _group_columns(self):
        """Each group's (lr, weight_decay, beta1, beta2, eps), and the entries' per-group host arrays: those five columns
        and rule_flag."""
        hyper = [self._hyper(g) for g in self.param_groups]
        return hyper, [_arr(C.c_double, col) for col in zip(*hyper)] + [_arr(C.c_int32, self._rule_flags())]

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        work = {}  # device -> [(group index, p)]
        for gi, p in self._items(type(self).__name__, self._check_sparse):
            work.setdefault(p.device, []).append((gi, p))
        if not work:
            return loss
        self._host_steps += 1
        found_inf = getattr(self, "found_inf", None)
        grad_scale = getattr(self, "grad_scale", None)
        lib = _lib.load()
        n_groups = len(self.param_groups)
        hyper, columns = self._group_columns()
        for device, items in work.items():
            states = [self._state_for(p, self.param_groups[gi]) for gi, p in items]
            moments = [self._state_tensors(st) for st in states]
            tables, length = self._group_tables(device, hyper, {gi for gi, _ in items})
            # GradScaler keeps found_inf and the scale on its own device: the copies to this one are enqueued, never read
            fi = None if found_inf is None else found_inf.to(device, torch.float32, non_blocking=True)
            gs = None if grad_scale is None else grad_scale.to(device, torch.float32, non_blocking=True)
            with torch.cuda.device(device):
                _lib.check(lib.qagnn_optim_step(
                    self._rule, len(items), *_tensor_arrays(items, states, moments), n_groups, *columns, _ptrs(tables),
                    length, _lib.ptr(fi), _lib.ptr(gs), _lib.ptr(self._counter(device)), _lib.stream_ptr(device)),
                    "qagnn_optim_step")
        return loss

    def _missing_step(self, st):
        """The step of an original's state that keeps none (torch's SGD)."""
        raise KeyError("step")

    def load_state_dict(self, state_dict):
        """Loads this optimiser's state_dict or its original's, whose 'step' is a Python int or a CPU tensor.  Every step
        becomes an int64 0-dim tensor on its parameter's device, and the step counts are read once to bound the step
        tables."""
        super().load_state_dict(state_dict)
        top = self._host_steps
        steps = {}
        for group in self.param_groups:
            for k in self._host_caches:
                group.pop(k, None)
            for p in group["params"]:
                st = self.state.get(p)
                if not st:
                    continue
                step = st["step"] if "step" in st else self._missing_step(st)
                if isinstance(step, torch.Tensor):
                    step = step.to(device=p.device, dtype=torch.int64).reshape(())
                else:
                    step = torch.tensor(int(step), dtype=torch.int64, device=p.device)
                st["step"] = step
                for k in self._state_keys:
                    st[k] = (torch.zeros_like(p, memory_format=torch.contiguous_format) if st.get(k) is None else
                             st[k].to(device=p.device, dtype=torch.float32).contiguous())
                steps.setdefault(p.device, []).append(step)
        for ss in steps.values():
            top = max(top, int(torch.stack(ss).max()))
        self._host_steps = top


class RAdam(_DeviceStepOptimizer):
    """RAdam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, degenerated_to_sgd=True): the reference's
    `utils.optimization_utils.RAdam`, stepped on the GPU.  Parameters and their gradients must be contiguous fp32 CUDA
    tensors; a parameter whose `.grad` is None is skipped and its step does not advance.  `lr` (and every other
    hyperparameter) is read from each group at every `step()`, so LambdaLR schedules work as with the reference."""

    _rule = 0
    _table_rows = staticmethod(step_size_table)
    _sparse_message = "RAdam does not support sparse gradients"
    _host_caches = ("buffer",)  # the reference's host cache of step sizes

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, degenerated_to_sgd=True):
        _check_hyper(lr, betas, eps)
        self.degenerated_to_sgd = degenerated_to_sgd
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def _check_group(self, group):
        _check_hyper(group["lr"], group["betas"], group["eps"])

    def _rule_flags(self):
        return [int(bool(self.degenerated_to_sgd))] * len(self.param_groups)


class AdamW(_DeviceStepOptimizer):
    """AdamW(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True): transformers' `AdamW`
    (3.4.0), the reference's `--optim adamw`, stepped on the GPU.  It is not `torch.optim.AdamW`: it adds eps to sqrt(v)
    before any bias correction, folds both corrections into one step size, and decays the weights after the Adam update
    (p += (-lr * weight_decay) * p, only when weight_decay > 0).  Parameters and their gradients must be contiguous fp32 CUDA
    tensors; a parameter whose `.grad` is None is skipped and its step does not advance.  Every hyperparameter, `correct_bias`
    included, is read from each group at every `step()`."""

    _rule = 1
    _table_rows = staticmethod(bias_correction_table)
    _sparse_message = "Adam does not support sparse gradients, please consider SparseAdam instead"

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True):
        _check_adamw_hyper(lr, betas, eps)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias))

    def _check_group(self, group):
        _check_adamw_hyper(group["lr"], group["betas"], group["eps"])

    def _rule_flags(self):
        return [int(bool(g["correct_bias"])) for g in self.param_groups]


class Adam(_DeviceStepOptimizer):
    """Adam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None, maximize=False,
    capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False): torch.optim.Adam, the reference's
    `--optim adam`, stepped on the GPU bit for bit as torch 2.11 steps it by default on CUDA (its foreach
    implementation).  The constructor, defaults, checks and param-group keys are torch's; amsgrad, maximize,
    decoupled_weight_decay and foreach / fused / capturable / differentiable set to True are refused (torch.optim.Adam has
    them).  The state keeps torch's keys, with `step` an int64 0-dim tensor on the parameter's device; `load_state_dict`
    takes torch's own state dict, whose fp32 CPU steps it converts.  Parameters and their gradients must be contiguous fp32
    CUDA tensors; a parameter whose `.grad` is None is skipped and its step does not advance."""

    _rule = 2
    _table_rows = staticmethod(adam_bias_correction_table)
    _sparse_message = "Adam does not support sparse gradients, please consider SparseAdam instead"

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        if isinstance(lr, torch.Tensor) or any(isinstance(b, torch.Tensor) for b in betas):
            raise ValueError("qagnn_b200.optim.Adam: a Tensor lr or betas is not implemented on the device; use "
                             "torch.optim.Adam for it")
        # torch's checks and messages
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if not (isinstance(betas[0], float) and isinstance(betas[1], float)):
            raise ValueError("betas must be either both floats or both Tensors")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize,
                        foreach=foreach, capturable=capturable, differentiable=differentiable, fused=fused,
                        decoupled_weight_decay=decoupled_weight_decay)
        self._check_group(defaults)
        super().__init__(params, defaults)

    def _check_group(self, group):
        _refuse("Adam", [(k, group.get(k)) for k in ("amsgrad", "maximize", "decoupled_weight_decay", "foreach", "fused",
                                                      "capturable", "differentiable")])
        _check_hyper(group["lr"], group["betas"], group["eps"])

    def _rule_flags(self):
        return [0] * len(self.param_groups)


class SGD(_DeviceStepOptimizer):
    """SGD(params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False, *, maximize=False, foreach=None,
    differentiable=False, fused=None): torch.optim.SGD, the reference's `--optim sgd`, stepped on the GPU
    bit for bit as torch 2.11 steps it by default on CUDA (its foreach implementation).  The constructor, defaults, checks and
    param-group keys are torch's; maximize, fused and differentiable set to True are refused (torch.optim.SGD has them).  With
    momentum the state keeps torch's `momentum_buffer`, allocated as zeros, plus `step`, an int64 0-dim tensor on the
    parameter's device: the buffer is set from the gradient where the device step is 0, so a first step that GradScaler
    skips on the device is handled as torch handles it.  `load_state_dict` takes torch's own state dict (a buffer counts as
    set).  Parameters and their gradients must be contiguous fp32 CUDA tensors; a parameter whose `.grad` is None is
    skipped."""

    _rule = 3
    _state_keys = ("momentum_buffer",)
    _sparse_message = "qagnn_b200.optim.SGD does not support sparse gradients; use torch.optim.SGD for them"

    def __init__(self, params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False, *, maximize=False,
                 foreach=None, differentiable=False, fused=None):
        if isinstance(lr, torch.Tensor):
            raise ValueError("qagnn_b200.optim.SGD: a Tensor lr is not implemented on the device; use torch.optim.SGD for it")
        # torch's checks and messages
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                        maximize=maximize, foreach=foreach, differentiable=differentiable, fused=fused)
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        self._check_group(defaults)
        super().__init__(params, defaults)

    @staticmethod
    def _hyper(group):
        # SGD's beta1 and beta2 are the momentum and the dampening
        return float(group["lr"]), float(group["weight_decay"]), float(group["momentum"]), float(group["dampening"]), 0.0

    def _check_group(self, group):
        _refuse("SGD", [(k, group.get(k)) for k in ("maximize", "fused", "differentiable")])
        if not 0.0 <= group["lr"]:
            raise ValueError(f"Invalid learning rate: {group['lr']}")
        if not 0.0 <= group["momentum"] < math.inf:
            raise ValueError(f"Invalid momentum value: {group['momentum']}")

    def _rule_flags(self):
        return [int(bool(g["nesterov"])) for g in self.param_groups]

    def _state_for(self, p, group):
        st = self.state[p]
        if "step" not in st:
            st["step"] = torch.zeros((), dtype=torch.int64, device=p.device)
        if group["momentum"] != 0 and st.get("momentum_buffer") is None:
            st["momentum_buffer"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            st["step"].zero_()  # a fresh buffer is set from the next gradient, as torch sets a missing one
        return st

    def _state_tensors(self, st):
        return st.get("momentum_buffer"), None

    def _missing_step(self, st):
        # torch's SGD keeps no step: a buffer it saved has been set
        return 0 if st.get("momentum_buffer") is None else 1


_clip_workspace = {}  # device -> [fp64 slots, int32 arrival counter, fp32 clip coefficient]


def _clip_buffers(device, n_slots):
    ws = _clip_workspace.get(device)
    if ws is None:
        ws = _clip_workspace[device] = [torch.empty(0, dtype=torch.float64, device=device),
                                        torch.zeros(1, dtype=torch.int32, device=device),
                                        torch.empty(1, dtype=torch.float32, device=device)]
    if ws[0].numel() < n_slots:
        ws[0] = torch.empty(max(n_slots, 2 * ws[0].numel()), dtype=torch.float64, device=device)
    return ws


@torch.no_grad()
def clip_grad_norm_(parameters, max_norm, norm_type=2.0, error_if_nonfinite=False, foreach=None):
    """torch.nn.utils.clip_grad_norm_ as the reference calls it, in two sm_90a launches on one device (csrc/clip.cu): the
    L2 norm of every `.grad` (parameters without one are skipped) and `.grad *= min(max_norm / (norm + 1e-6), 1)` in place.
    Returns the norm as a new 0-dim fp32 tensor on the gradients' device without reading it on the host, or
    `torch.tensor(0.0)` when no parameter has a gradient.

    The norm is summed in fp64 in an order fixed by the gradients' sizes alone, so it is reproducible bit for bit and within
    one fp32 ulp of the exact norm; torch's fp32 sum is neither, and its squares overflow (an inf norm) for gradients past
    about 1.8e19, where this one stays finite.  From the norm on, the coefficient and every gradient are torch's fp32
    operations bit for bit, and a coefficient of 1 leaves the gradients untouched without rewriting them.  An inf norm gives
    a coefficient of 0 and a NaN norm a NaN one, as in torch.  Gradients must be dense, contiguous fp32 CUDA tensors on one
    device.  `norm_type` must be 2 and `error_if_nonfinite` False, which would need a host read; `foreach` is accepted and
    ignored.  One fp64 slot per 8192 gradient elements is kept per device between calls."""
    name = "clip_grad_norm_"
    if float(norm_type) != 2.0:
        raise ValueError(f"qagnn_b200.optim.{name}: only the L2 norm (norm_type=2) is implemented (got {norm_type})")
    if error_if_nonfinite:
        raise ValueError(f"qagnn_b200.optim.{name}: error_if_nonfinite=True needs a host read of the norm; it is not "
                         f"supported")
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    grads = [p.grad for p in parameters if p.grad is not None]
    if not grads:
        return torch.tensor(0.0)
    for g in grads:
        if g.layout != torch.strided:
            raise TypeError(f"qagnn_b200.optim.{name}: the gradient must be dense (got {g.layout})")
        _check_tensor(g, "gradient", name)
    device = grads[0].device
    if any(g.device != device for g in grads):
        raise ValueError(f"qagnn_b200.optim.{name}: gradients on {sorted({str(g.device) for g in grads})}; all must be on "
                         f"one device")
    lib = _lib.load()
    n = len(grads)
    numels = (C.c_int64 * n)(*[g.numel() for g in grads])
    slots, counter, coef = _clip_buffers(device, lib.qagnn_clip_grad_norm_slots(n, numels))
    total_norm = torch.empty((), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.qagnn_clip_grad_norm(n, (C.c_void_p * n)(*[g.data_ptr() for g in grads]), numels, float(max_norm),
                                            _lib.ptr(slots), slots.numel(), _lib.ptr(counter), _lib.ptr(total_norm),
                                            _lib.ptr(coef), _lib.stream_ptr(device)), "qagnn_clip_grad_norm")
    return total_norm


class CapturedTail:
    """The recipe's optimiser tail as one CUDA graph replay per optimiser batch (csrc/tail.cu).  `tail()` does what

        scaler.unscale_(optimizer); clip_grad_norm_(clip_parameters, max_grad_norm)   # both only when max_grad_norm > 0
        scheduler.step(); scaler.step(optimizer); scaler.update()

    does with this module's `optimizer` and `clip_grad_norm_` and torch's GradScaler, bit for bit in the parameters, their
    state, `.grad`, the norm and the scaler's scale and growth tracker, in two sm_90a launches (two more per 512 tensors or
    16 groups) and with no host read.  It returns the norm as a new 0-dim device tensor, or None when max_grad_norm <= 0.

    `optimizer` is a `RAdam`, `AdamW`, `Adam` or `SGD`; `scaler` a `torch.amp.GradScaler` or None (a disabled one counts as None);
    `scheduler` any LR scheduler or None.  `clip_parameters` defaults to the optimizer's parameters; those with a `.grad` must
    be the optimizer's parameters with a `.grad`, in any order.  Every call first steps the scheduler on the host, then
    writes what a replay must not freeze (each group's hyperparameters, the step tables, max_grad_norm and the scaler's
    factors) into a device block through a fresh pinned buffer, replays the graph and counts the step on the host, so eager
    `optimizer.step()` calls can be mixed in.  The graph holds the tensors' addresses: a call whose parameters, gradients,
    optimiser state or scaler tensors moved (a frozen or unfrozen encoder, `zero_grad(set_to_none=True)`,
    `load_state_dict`) first runs its kernels directly and captures them again; `captures` counts the captures.  The
    scaler's Python bookkeeping is not touched, so `scaler.scale`, `get_scale` and `state_dict` keep working.  Gradients
    must be dense, contiguous fp32 tensors on one CUDA device, as for the optimiser."""

    def __init__(self, optimizer, scaler=None, scheduler=None, max_grad_norm=0.0, clip_parameters=None):
        if not isinstance(optimizer, (RAdam, AdamW, Adam, SGD)):
            raise ValueError(f"qagnn_b200.optim.CapturedTail: {type(optimizer).__module__}.{type(optimizer).__name__} is not "
                             f"qagnn_b200.optim.RAdam, AdamW, Adam or SGD; run the eager tail (scaler.unscale_, clip_grad_norm_, "
                             f"scheduler.step, scaler.step, scaler.update) for it")
        if scaler is not None and not scaler.is_enabled():
            scaler = None
        self.optimizer, self.scaler, self.scheduler = optimizer, scaler, scheduler
        self.max_grad_norm = float(max_grad_norm)
        if isinstance(clip_parameters, torch.Tensor):
            clip_parameters = [clip_parameters]
        self._clip_parameters = None if clip_parameters is None else list(clip_parameters)
        self._rule = optimizer._rule
        self.captures = 0
        self._key = None
        self._graph = None
        self._bufs = self._bufs_key = self._graph_bufs = None

    @staticmethod
    def _check_dense(grad):
        if grad.layout != torch.strided:
            raise TypeError(f"qagnn_b200.optim.CapturedTail: the gradient must be dense (got {grad.layout})")

    def _work(self):
        """[(group index, p)] of the parameters with a gradient, checked as the optimiser and the clip check them."""
        name = "CapturedTail"
        items = self.optimizer._items(name, self._check_dense)
        if not items:
            raise RuntimeError(f"qagnn_b200.optim.{name}: no parameter has a gradient")
        devices = {p.device for _, p in items}
        if len(devices) != 1:
            raise ValueError(f"qagnn_b200.optim.{name}: parameters on {sorted(str(d) for d in devices)}; all must be on one "
                             f"device (the eager tail handles several)")
        return items, items[0][1].device

    def _norm_grads(self, items):
        if self._clip_parameters is None:
            return [p.grad for _, p in items]
        grads = [p.grad for p in self._clip_parameters if p.grad is not None]
        if {id(g) for g in grads} != {id(p.grad) for _, p in items} or len(grads) != len(items):
            raise ValueError("qagnn_b200.optim.CapturedTail: the clip_parameters with a .grad must be the optimizer's "
                             "parameters with a .grad; run the eager tail for other sets")
        return grads

    def _scaler_tensors(self, device):
        scaler = self.scaler
        if scaler is None:
            return None, None
        if scaler._scale is None or scaler._growth_tracker is None:
            raise RuntimeError("qagnn_b200.optim.CapturedTail: the scaler has no scale yet; call scaler.scale(loss) first")
        if scaler._scale.device != device:
            raise ValueError(f"qagnn_b200.optim.CapturedTail: the scaler's scale is on {scaler._scale.device}, the "
                             f"parameters on {device}")
        return scaler._scale, scaler._growth_tracker

    @torch.no_grad()
    def __call__(self):
        key, launcher = self.prepare()
        if self._graph is not None and self._key == key and self._graph_bufs is self._bufs:
            self._graph.replay()
        else:
            # this call's step runs directly, which also loads the kernels; the capture then records the same launches
            self._graph = None
            launch = launcher()
            launch()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                launch()
            self._graph, self._key, self._graph_bufs = graph, key, self._bufs
            self.captures += 1
        return self._bufs["total_norm"].clone() if self.max_grad_norm > 0 else None

    @torch.no_grad()
    def prepare(self):
        """The host half of a call, which a graph holding the tail's launches runs before every replay: the checks, the
        scheduler step, the optimiser's host step count and the upload of the per-call block, enqueued on the current stream.
        Returns (key, launcher): `key` names what the launches bake in (the device, the clip, and the addresses and sizes of
        the parameters, gradients, optimiser state and scaler tensors), and `launcher()` returns a function that enqueues the
        tail's kernels on the current stream.  The device buffers they use, `self._bufs`, are replaced when the key changes;
        a graph that holds the launches is valid while the key and that dict are the ones it was captured with."""
        opt = self.optimizer
        st = None if self.scaler is None else self.scaler._per_optimizer_states.get(id(opt))
        if st is not None and st["stage"] is OptState.UNSCALED:
            raise RuntimeError("qagnn_b200.optim.CapturedTail: scaler.unscale_(optimizer) was already called since the last "
                               "update(); the tail unscales the gradients itself")
        items, device = self._work()
        clip = self.max_grad_norm > 0
        scale, tracker = self._scaler_tensors(device)
        norm_grads = self._norm_grads(items) if clip else [p.grad for _, p in items]
        states = [opt._state_for(p, opt.param_groups[gi]) for gi, p in items]
        moments = [opt._state_tensors(st) for st in states]
        addr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        key = (device, clip, None if scale is None else (scale.data_ptr(), tracker.data_ptr()), len(opt.param_groups),
               tuple((gi, p.data_ptr(), p.grad.data_ptr(), addr(m), addr(v), s["step"].data_ptr(), p.numel())
                     for (gi, p), s, (m, v) in zip(items, states, moments)),
               tuple((g.data_ptr(), g.numel()) for g in norm_grads))

        if self.scheduler is not None:
            self.scheduler.step()
        opt._host_steps += 1
        lib = _lib.load()
        hyper, columns = opt._group_columns()
        tables, table_len = opt._group_tables(device, hyper, range(len(hyper)))
        n_groups = len(hyper)
        n_bytes = lib.qagnn_step_tail_block_bytes(n_groups)
        if self._bufs_key != key:
            self._bufs, self._bufs_key = self._buffers(device, n_bytes, norm_grads, lib), key
        bufs = self._bufs
        # a fresh pinned buffer per call from the caching host allocator, which keeps it until its copy has run
        staging = torch.empty(n_bytes, dtype=torch.uint8, pin_memory=True)
        sc = self.scaler
        _lib.check(lib.qagnn_step_tail_fill(
            self._rule, n_groups, *columns, _ptrs(tables), table_len, self.max_grad_norm,
            float(sc._growth_factor) if sc else 2.0, float(sc._backoff_factor) if sc else 0.5,
            int(sc._growth_interval) if sc else 1, C.c_void_p(staging.data_ptr()), n_bytes), "qagnn_step_tail_fill")
        bufs["block"].copy_(staging, non_blocking=True)
        return key, lambda: self._launcher(lib, device, items, states, moments, norm_grads, clip, scale, tracker, n_groups)

    def _buffers(self, device, n_bytes, norm_grads, lib):
        n = len(norm_grads)
        n_slots = lib.qagnn_clip_grad_norm_slots(n, (C.c_int64 * n)(*[g.numel() for g in norm_grads]))
        z = lambda dt: torch.zeros(1, dtype=dt, device=device)  # noqa: E731
        return dict(block=torch.empty(n_bytes, dtype=torch.uint8, device=device),
                    slots=torch.empty(max(n_slots, 1), dtype=torch.float64, device=device),
                    counter=z(torch.int32), found_inf=z(torch.float32), coef=z(torch.float32),
                    total_norm=torch.zeros((), dtype=torch.float32, device=device))

    def _launcher(self, lib, device, items, states, moments, norm_grads, clip, scale, tracker, n_groups):
        b = self._bufs
        args = (self._rule, len(items), *_tensor_arrays(items, states, moments), n_groups, len(norm_grads), _ptrs(norm_grads),
                _arr(C.c_int64, [g.numel() for g in norm_grads]), int(clip), _lib.ptr(b["block"]),
                _lib.ptr(b["slots"]), b["slots"].numel(), _lib.ptr(b["counter"]), _lib.ptr(b["total_norm"]),
                _lib.ptr(b["coef"]), _lib.ptr(b["found_inf"]), _lib.ptr(scale), _lib.ptr(tracker))

        def launch():
            with torch.cuda.device(device):
                _lib.check(lib.qagnn_step_tail(*args, _lib.stream_ptr(device)), "qagnn_step_tail")
        return launch


# The reference's --optim table (utils/optimization_utils.py).  'sgd' and 'adam' are torch's own classes, as the reference
# imports them: they do not declare `_step_supports_amp_scaling`, so under GradScaler `scaler.step` still reads found_inf on
# the host for them, and CapturedTail refuses them.
OPTIMIZER_CLASSES = {
    "sgd": torch.optim.SGD,
    "adam": torch.optim.Adam,
    "adamw": AdamW,
    "radam": RAdam,
}

# The same table stepped on the device throughout: this module's Adam and SGD step as torch's do, bit for bit, take
# GradScaler's inf skip on the device and run in CapturedTail.
DEVICE_OPTIMIZER_CLASSES = {
    "sgd": SGD,
    "adam": Adam,
    "adamw": AdamW,
    "radam": RAdam,
}
