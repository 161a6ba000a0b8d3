"""Host-side schedule of the reference's `PLMSSampler` (ldm/models/diffusion/plms.py): the loop's time bookkeeping
(`time_range`, `index`, `t_next`, :139-149) and the per-step scalars of `get_x_prev_and_pred_x0` (:205-223).

The tables are DDIM's (`make_schedule`, :25-55).  Every scalar is formed with torch CPU fp32 ops in the reference's
order, on the values its `torch.full` calls take (:207-210), and handed to `ctrlora_plms_update` /
`ctrlora_ddim_update` as a float kernel argument: no per-step device tensor, no host sync.  The values equal the
reference's as it computes them on a CPU.  torch's CPU `sqrt` is not always correctly rounded, so the reference run on a
GPU, whose `sqrt` is, can differ by one ulp (t = 701 of the 20-step plan, DESIGN §7).
"""
import numpy as np
import torch


class Step:
    """Step i of plms_sampling: the model is evaluated at (x, t) (and at t_next on step 0); `index` selects the table
    entries.  a_t, a_prev, sigma_t, sqrt_one_minus_at are the fp32 values of :207-210 (what ctrlora_ddim_update takes);
    sqrt_a_t, sqrt_a_prev and dir_coef are a_t.sqrt(), a_prev.sqrt() and (1 - a_prev - sigma_t**2).sqrt()."""
    __slots__ = ("index", "t", "t_next", "a_t", "a_prev", "sigma_t", "sqrt_one_minus_at", "sqrt_a_t", "sqrt_a_prev",
                 "dir_coef")

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)

    def kernel_args(self):
        return dict(sqrt_a_t=self.sqrt_a_t, sqrt_one_minus_at=self.sqrt_one_minus_at, sqrt_a_prev=self.sqrt_a_prev,
                    dir_coef=self.dir_coef)


def time_range(ddim_timesteps):
    """The steps plms_sampling walks (:139): the DDIM timesteps, flipped."""
    return [int(v) for v in np.flip(ddim_timesteps)]


def plan(steps, alphas, alphas_prev, sqrt_one_minus_alphas, sigmas):
    """`Step`s for the walk `steps` (time_range's result) over the given tables, which are indexed by
    index = len(steps) - i - 1 (:147); t_next = steps[min(i + 1, len(steps) - 1)] (:149)."""
    n = len(steps)
    full = lambda v: torch.full((1,), v, dtype=torch.float32)   # torch.full((b, 1, 1, 1), table[index]), :207-210
    out = []
    for i, t in enumerate(steps):
        index = n - i - 1
        a_t, a_prev = full(float(alphas[index])), full(float(alphas_prev[index]))
        sigma_t, s1m = full(float(sigmas[index])), full(float(sqrt_one_minus_alphas[index]))
        f = lambda v: float(v[0])
        out.append(Step(index=index, t=int(t), t_next=int(steps[min(i + 1, n - 1)]), a_t=f(a_t), a_prev=f(a_prev),
                        sigma_t=f(sigma_t), sqrt_one_minus_at=f(s1m), sqrt_a_t=f(a_t.sqrt()),
                        sqrt_a_prev=f(a_prev.sqrt()), dir_coef=f((1. - a_prev - sigma_t ** 2).sqrt())))
    return out
