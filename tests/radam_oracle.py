"""The reference's RAdam update (utils/optimization_utils.py) restated as eager torch ops in the reference's order, for the tests
of qagnn_b200.optim.RAdam.  Pure torch: on the CPU it reproduces the reference's trajectories (tests/golden/ref/radam.pt), and
on a GPU it is the eager op sequence the kernel must equal bit for bit.  `state['step']` is a Python int, as the reference keeps
it, and GradScaler drives it the eager way (unscale_, a host read of found_inf, then step())."""
import math

import torch


def step_size(beta1, beta2, t, degenerated_to_sgd=True):
    """(rho_t, s) at step t in Python doubles; s = -1 when rho_t < 5 and the step does not degenerate to SGD."""
    beta2_t = beta2 ** t
    rho_inf = 2 / (1 - beta2) - 1
    rho_t = rho_inf - 2 * t * beta2_t / (1 - beta2_t)
    if rho_t >= 5:
        s = math.sqrt((1 - beta2_t) * (rho_t - 4) / (rho_inf - 4) * (rho_t - 2) / rho_t * rho_inf / (rho_inf - 2)) / (1 - beta1 ** t)
    elif degenerated_to_sgd:
        s = 1.0 / (1 - beta1 ** t)
    else:
        s = -1
    return rho_t, s


class RAdamOracle(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, degenerated_to_sgd=True):
        self.degenerated_to_sgd = degenerated_to_sgd
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            lr, wd = group["lr"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad.float()
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                m, v = st["exp_avg"], st["exp_avg_sq"]
                v.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                m.mul_(beta1).add_(grad, alpha=1 - beta1)
                st["step"] += 1
                rho_t, s = step_size(beta1, beta2, st["step"], self.degenerated_to_sgd)
                if rho_t >= 5:
                    if wd != 0:
                        p.add_(p, alpha=-wd * lr)
                    denom = v.sqrt().add_(group["eps"])
                    p.addcdiv_(m, denom, value=-s * lr)
                elif s > 0:
                    if wd != 0:
                        p.add_(p, alpha=-wd * lr)
                    p.add_(m, alpha=-s * lr)
        return None
