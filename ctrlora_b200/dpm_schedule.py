"""Host-side schedule of the reference's `DPMSolverSampler` (ldm/models/diffusion/dpm_solver/sampler.py:72-85):
DPM-Solver++ (data prediction), multistep, order 2, `time_uniform` steps, `lower_order_final`.

Every per-step scalar is formed with torch CPU fp32 ops in the reference's order (dpm_solver.py), on one-element
tensors, and handed to `ctrlora_dpm_multistep_update` as a float kernel argument.  The reference forms the same
scalars on `[B]` tensors; its unary ops (exp, log, expm1) take torch's scalar CPU loop for batches below two SIMD
vectors (16 images with AVX2), so the values agree bit for bit there.
"""
import torch


class DiscreteVPSchedule:
    """NoiseScheduleVP('discrete', alphas_cumprod=...) (dpm_solver.py:60-160): log(alpha_t) is piecewise linear in the
    continuous time t over the keypoints t_n = (n + 1) / N, N = len(alphas_cumprod); T = 1."""

    def __init__(self, alphas_cumprod):
        ac = torch.as_tensor(alphas_cumprod).detach().cpu().to(torch.float32)
        self.total_N = ac.shape[0]
        self.T = 1.
        self.t_array = torch.linspace(0., 1., self.total_N + 1)[1:]
        self.log_alpha_array = 0.5 * torch.log(ac)

    def marginal_log_mean_coeff(self, t):
        return _interp(t, self.t_array, self.log_alpha_array)

    def marginal_alpha(self, t):
        return torch.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):
        lmc = self.marginal_log_mean_coeff(t)
        return lmc - 0.5 * torch.log(1. - torch.exp(2. * lmc))

    def model_time(self, t):
        """the discrete model's input time for continuous t (model_wrapper, dpm_solver.py:246-253): fractional"""
        return (t - 1. / self.total_N) * 1000.


def _interp(x, xp, yp):
    """Piecewise-linear y(x) through ascending keypoints (xp, yp), continued linearly past both ends (interpolate_fn,
    dpm_solver.py:1104-1142).  An x equal to a keypoint is ranked before it, and the segment is chosen from that rank
    (rank 0 -> first segment, rank K -> last); the value is start_y + (x - start_x) * (end_y - start_y) / (end_x - start_x)
    with the reference's rounding order."""
    k = xp.shape[0]
    rank = torch.searchsorted(xp, x, right=False)
    lo = torch.clamp(rank - 1, 0, k - 2)
    sx, ex, sy, ey = xp[lo], xp[lo + 1], yp[lo], yp[lo + 1]
    return sy + (x - sx) * (ey - sy) / (ex - sx)


class Step:
    """One sampler step i: the model is evaluated at (x_i, t[i]); the update kernel forms the data prediction with
    (sigma_s, alpha_s) and moves x to t[i + 1] with order `order` and coefficients (c_x, c_m, c_d, inv_r0)."""
    __slots__ = ("order", "t", "model_time", "sigma_s", "alpha_s", "c_x", "c_m", "c_d", "inv_r0")

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)

    def kernel_args(self):
        return dict(sigma_s=self.sigma_s, alpha_s=self.alpha_s, c_x=self.c_x, c_m=self.c_m, c_d=self.c_d,
                    inv_r0=self.inv_r0)


def time_steps(ns, steps):
    """get_time_steps('time_uniform', t_T = T, t_0 = 1 / N) (dpm_solver.py:376-403, :1037-1038): fp32 [steps + 1]"""
    return torch.linspace(ns.T, 1. / ns.total_N, steps + 1)


def step_orders(steps, order=2, lower_order_final=True):
    """DPM_Solver.sample(method='multistep') (dpm_solver.py:1044-1074): order 1 for the first step, then `order`,
    and with lower_order_final and steps < 15 the last steps drop to the order they have history for."""
    if steps < order:
        raise ValueError(f"DPM-Solver multistep needs steps >= order ({steps} < {order})")
    out = [1]
    for step in range(order, steps + 1):
        out.append(min(order, steps + 1 - step) if lower_order_final and steps < 15 else order)
    return out


def multistep_plan(alphas_cumprod, steps):
    """The reference sampler's `steps` steps as `Step`s, every scalar a Python float holding an fp32 value."""
    ns = DiscreteVPSchedule(alphas_cumprod)
    ts = time_steps(ns, steps)
    f = lambda v: float(v[0])
    plan = []
    for i, order in enumerate(step_orders(steps)):
        s, t = ts[i:i + 1], ts[i + 1:i + 2]
        sigma_s, sigma_t = ns.marginal_std(s), ns.marginal_std(t)
        alpha_t = torch.exp(ns.marginal_log_mean_coeff(t))
        lambda_s, lambda_t = ns.marginal_lambda(s), ns.marginal_lambda(t)
        h = lambda_t - lambda_s
        if order == 1:   # dpm_solver_first_update, predict_x0 (:484-497)
            c_m = alpha_t * torch.expm1(-h)
            c_d = inv_r0 = torch.zeros(1)
        else:            # multistep_dpm_solver_second_update, predict_x0, 'dpm_solver' (:742-758)
            h_0 = lambda_s - ns.marginal_lambda(ts[i - 1:i])
            r0 = h_0 / h
            inv_r0 = 1. / r0
            c_m = alpha_t * (torch.exp(-h) - 1.)
            c_d = 0.5 * (alpha_t * (torch.exp(-h) - 1.))
        plan.append(Step(order=order, t=f(s), model_time=f(ns.model_time(s)), sigma_s=f(sigma_s),
                         alpha_s=f(ns.marginal_alpha(s)), c_x=f(sigma_t / sigma_s), c_m=f(c_m), c_d=f(c_d),
                         inv_r0=f(inv_r0)))
    return plan
