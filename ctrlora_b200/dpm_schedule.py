"""Host-side schedule of the reference's `DPMSolverSampler` (ldm/models/diffusion/dpm_solver/sampler.py:72-85):
DPM-Solver++ (data prediction), multistep, order 2, `time_uniform` steps, `lower_order_final`.

Every per-step scalar is formed with torch CPU fp32 ops in the reference's order (dpm_solver.py), on one-element
tensors, and handed to `ctrlora_dpm_multistep_update` as a float kernel argument.  The reference forms the same
scalars on `[B]` tensors; its unary ops (exp, log, expm1) take torch's scalar CPU loop for batches below two SIMD
vectors (16 images with AVX2), so the values agree bit for bit there.

The second half of the module serves the full DPM_Solver drop-in (ldm/models/diffusion/dpm_solver/dpm_solver.py):
`NoiseScheduleVP` for the three schedules, the time steps of the three skip types and every update's scalars.
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


# ---- the full DPM_Solver (ldm/models/diffusion/dpm_solver/dpm_solver.py) --------------------------------------------
# Everything below takes and returns CPU fp32 tensors of the shapes the reference uses ([B] times, 0-dim r1 / r2 where
# the reference has them), evaluated with the reference's torch ops in its order; the kernel scalars are read from
# element 0 (every image of a batch shares its times).

import math

import numpy as np


def interpolate_fn(x, xp, yp):
    """y(x) piecewise linear through the keypoints (xp, yp) per channel, continued linearly past both ends
    (dpm_solver.py:1104-1142); x [N, C], xp / yp [C, K] with xp ascending.  Same segment choice and rounding as
    `_interp` (an x equal to a keypoint is ranked before it)."""
    n, k = x.shape[0], xp.shape[1]
    rank = torch.searchsorted(xp.contiguous(), x.t().contiguous(), right=False).t()
    lo = torch.clamp(rank - 1, 0, k - 2)
    at = lambda arr, idx: torch.gather(arr.unsqueeze(0).expand(n, -1, -1), 2, idx.unsqueeze(2)).squeeze(2)
    sx, ex, sy, ey = at(xp, lo), at(xp, lo + 1), at(yp, lo), at(yp, lo + 1)
    return sy + (x - sx) * (ey - sy) / (ex - sx)


class NoiseScheduleVP:
    """The reference's VP noise schedule (dpm_solver.py:7-158): 'discrete' (log alpha piecewise linear over
    t_n = (n + 1) / N, from `betas` or `alphas_cumprod`), 'linear' and 'cosine' (continuous time).  The discrete
    tables are held at fp32 on the CPU and moved to the device of the argument, as the reference moves its own."""

    def __init__(self, schedule='discrete', betas=None, alphas_cumprod=None, continuous_beta_0=0.1,
                 continuous_beta_1=20.):
        if schedule not in ('discrete', 'linear', 'cosine'):
            raise ValueError("Unsupported noise schedule {}. The schedule needs to be 'discrete' or 'linear' or "
                             "'cosine'".format(schedule))
        self.schedule = schedule
        if schedule == 'discrete':
            if betas is not None:
                b = torch.as_tensor(betas).detach().cpu().to(torch.float32)
                log_alphas = 0.5 * torch.log(1 - b).cumsum(dim=0)
            else:
                assert alphas_cumprod is not None
                log_alphas = 0.5 * torch.log(torch.as_tensor(alphas_cumprod).detach().cpu().to(torch.float32))
            self.total_N = len(log_alphas)
            self.T = 1.
            self.t_array = torch.linspace(0., 1., self.total_N + 1)[1:].reshape((1, -1))
            self.log_alpha_array = log_alphas.reshape((1, -1))
        else:
            self.total_N = 1000
            self.beta_0, self.beta_1 = continuous_beta_0, continuous_beta_1
            self.cosine_s, self.cosine_beta_max = 0.008, 999.
            self.cosine_t_max = (math.atan(self.cosine_beta_max * (1. + self.cosine_s) / math.pi) * 2.
                                 * (1. + self.cosine_s) / math.pi - self.cosine_s)
            self.cosine_log_alpha_0 = math.log(math.cos(self.cosine_s / (1. + self.cosine_s) * math.pi / 2.))
            self.T = 0.9946 if schedule == 'cosine' else 1.   # the reference's end time for the cosine schedule

    def marginal_log_mean_coeff(self, t):
        """log alpha_t"""
        if self.schedule == 'discrete':
            y = interpolate_fn(t.reshape((-1, 1)), self.t_array.to(t.device), self.log_alpha_array.to(t.device))
            return y.reshape((-1,))
        if self.schedule == 'linear':
            return -0.25 * t ** 2 * (self.beta_1 - self.beta_0) - 0.5 * t * self.beta_0
        return torch.log(torch.cos((t + self.cosine_s) / (1. + self.cosine_s) * math.pi / 2.)) - self.cosine_log_alpha_0

    def marginal_alpha(self, t):
        return torch.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):
        """lambda_t = log alpha_t - log sigma_t (the half log-SNR)"""
        lmc = self.marginal_log_mean_coeff(t)
        return lmc - 0.5 * torch.log(1. - torch.exp(2. * lmc))

    def inverse_lambda(self, lamb):
        """t of a half log-SNR"""
        zero = torch.zeros((1,)).to(lamb)
        if self.schedule == 'linear':
            tmp = 2. * (self.beta_1 - self.beta_0) * torch.logaddexp(-2. * lamb, zero)
            delta = self.beta_0 ** 2 + tmp
            return tmp / (torch.sqrt(delta) + self.beta_0) / (self.beta_1 - self.beta_0)
        if self.schedule == 'discrete':
            log_alpha = -0.5 * torch.logaddexp(torch.zeros((1,)).to(lamb.device), -2. * lamb)
            t = interpolate_fn(log_alpha.reshape((-1, 1)), torch.flip(self.log_alpha_array.to(lamb.device), [1]),
                               torch.flip(self.t_array.to(lamb.device), [1]))
            return t.reshape((-1,))
        log_alpha = -0.5 * torch.logaddexp(-2. * lamb, zero)
        return (torch.arccos(torch.exp(log_alpha + self.cosine_log_alpha_0)) * 2. * (1. + self.cosine_s) / math.pi
                - self.cosine_s)

    def model_input_time(self, t_continuous):
        """model_wrapper's get_model_input_time (dpm_solver.py:246-255)"""
        if self.schedule == 'discrete':
            return (t_continuous - 1. / self.total_N) * 1000.
        return t_continuous


SKIP_TYPES = ('logSNR', 'time_uniform', 'time_quadratic')


def get_time_steps(ns, skip_type, t_T, t_0, N):
    """DPM_Solver.get_time_steps (dpm_solver.py:376-403) on the CPU: fp32 [N + 1]"""
    if skip_type == 'logSNR':
        lambda_T = ns.marginal_lambda(torch.tensor(t_T))
        lambda_0 = ns.marginal_lambda(torch.tensor(t_0))
        return ns.inverse_lambda(torch.linspace(lambda_T.item(), lambda_0.item(), N + 1))
    if skip_type == 'time_uniform':
        return torch.linspace(t_T, t_0, N + 1)
    if skip_type == 'time_quadratic':
        return torch.linspace(t_T ** 0.5, t_0 ** 0.5, N + 1).pow(2)
    raise ValueError("Unsupported skip_type {}, need to be 'logSNR' or 'time_uniform' or 'time_quadratic'"
                     .format(skip_type))


def singlestep_orders(steps, order):
    """the orders of DPM-Solver-fast (dpm_solver.py:435-454): all `steps` evaluations used, highest order first"""
    if order == 3:
        k = steps // 3 + 1
        return {0: [3] * (k - 2) + [2, 1], 1: [3] * (k - 1) + [1], 2: [3] * (k - 1) + [2]}[steps % 3]
    if order == 2:
        return [2] * (steps // 2) + [1] * (steps % 2)
    if order == 1:
        return [1] * steps
    raise ValueError("'order' must be '1' or '2' or '3'.")


def get_orders_and_timesteps_for_singlestep_solver(ns, steps, order, skip_type, t_T, t_0):
    """(outer time steps, orders) of DPM-Solver-fast (dpm_solver.py:405-461), CPU fp32"""
    orders = singlestep_orders(steps, order)
    if skip_type == 'logSNR':   # K outer intervals; the reference takes K = 1 for order 1
        return get_time_steps(ns, skip_type, t_T, t_0, 1 if order == 1 else len(orders)), orders
    return get_time_steps(ns, skip_type, t_T, t_0, steps)[torch.cumsum(torch.tensor([0] + orders), 0)], orders


def quantile_rank(n, q=0.995):
    """torch.quantile's order statistics for `n` values: (floor, ceil, lerp weight) of fp32(q) * (n - 1) in fp32"""
    rank = np.float32(q) * np.float32(n - 1)
    lo = int(rank)
    return lo, int(np.ceil(rank)), float(np.float32(rank - np.float32(lo)))


def _s(v):
    """a kernel scalar: element 0 of an fp32 tensor, or a Python number rounded to fp32 as torch rounds it"""
    if torch.is_tensor(v):
        assert v.dtype == torch.float32
        return float(v.reshape(-1)[0])
    return float(np.float32(v))


class Update:
    """One kernel update: `mode` of ops.dpm_solver_update and its coefficients (a, b, c, d, k0, k1, k2, k3, rd)."""
    __slots__ = ("mode", "coef")

    def __init__(self, mode, a, b, c=0., d=0., k0=0., k1=0., k2=0., k3=0., rd=0.):
        self.mode = mode
        self.coef = tuple(_s(v) for v in (a, b, c, d, k0, k1, k2, k3, rd))


def _check_solver_type(solver_type):
    if solver_type not in ('dpm_solver', 'taylor'):
        raise ValueError("'solver_type' must be either 'dpm_solver' or 'taylor', got {}".format(solver_type))


def first_update(ns, s, t, predict_x0):
    """dpm_solver_first_update (dpm_solver.py:469-513)"""
    h = ns.marginal_lambda(t) - ns.marginal_lambda(s)
    log_alpha_s, log_alpha_t = ns.marginal_log_mean_coeff(s), ns.marginal_log_mean_coeff(t)
    sigma_s, sigma_t = ns.marginal_std(s), ns.marginal_std(t)
    if predict_x0:
        return Update("first", sigma_t / sigma_s, torch.exp(log_alpha_t) * torch.expm1(-h))
    return Update("first", torch.exp(log_alpha_t - log_alpha_s), sigma_t * torch.expm1(h))


def singlestep_second_update(ns, s, t, r1, predict_x0, solver_type):
    """singlestep_dpm_solver_second_update (dpm_solver.py:515-597): (s1, x_s1 update, x_t update with m1 = model_s1)"""
    _check_solver_type(solver_type)
    r1 = 0.5 if r1 is None else r1
    lambda_s, lambda_t = ns.marginal_lambda(s), ns.marginal_lambda(t)
    h = lambda_t - lambda_s
    s1 = ns.inverse_lambda(lambda_s + r1 * h)
    log_alpha_s, log_alpha_s1, log_alpha_t = (ns.marginal_log_mean_coeff(v) for v in (s, s1, t))
    sigma_s, sigma_s1, sigma_t = ns.marginal_std(s), ns.marginal_std(s1), ns.marginal_std(t)
    alpha_s1, alpha_t = torch.exp(log_alpha_s1), torch.exp(log_alpha_t)
    if predict_x0:
        phi_11, phi_1 = torch.expm1(-r1 * h), torch.expm1(-h)
        mid = Update("first", sigma_s1 / sigma_s, alpha_s1 * phi_11)
        if solver_type == 'dpm_solver':
            c = -((0.5 / r1) * (alpha_t * phi_1))
        else:
            c = (1. / r1) * (alpha_t * ((torch.exp(-h) - 1.) / h + 1.))
        return s1, mid, Update("diff", sigma_t / sigma_s, alpha_t * phi_1, c)
    phi_11, phi_1 = torch.expm1(r1 * h), torch.expm1(h)
    mid = Update("first", torch.exp(log_alpha_s1 - log_alpha_s), sigma_s1 * phi_11)
    if solver_type == 'dpm_solver':
        c = -((0.5 / r1) * (sigma_t * phi_1))
    else:
        c = -((1. / r1) * (sigma_t * ((torch.exp(h) - 1.) / h - 1.)))
    return s1, mid, Update("diff", torch.exp(log_alpha_t - log_alpha_s), sigma_t * phi_1, c)


def singlestep_third_update(ns, s, t, r1, r2, predict_x0, solver_type):
    """singlestep_dpm_solver_third_update (dpm_solver.py:599-721): (s1, s2, x_s1 update, x_s2 update (m1 = model_s1),
    x_t update ('dpm_solver': DIFF with m1 = model_s2; 'taylor': m1 = model_s1, m2 = model_s2))"""
    _check_solver_type(solver_type)
    r1 = 1. / 3. if r1 is None else r1
    r2 = 2. / 3. if r2 is None else r2
    lambda_s, lambda_t = ns.marginal_lambda(s), ns.marginal_lambda(t)
    h = lambda_t - lambda_s
    s1, s2 = ns.inverse_lambda(lambda_s + r1 * h), ns.inverse_lambda(lambda_s + r2 * h)
    log_alpha_s, log_alpha_s1, log_alpha_s2, log_alpha_t = (ns.marginal_log_mean_coeff(v) for v in (s, s1, s2, t))
    sigma_s, sigma_s1, sigma_s2, sigma_t = (ns.marginal_std(v) for v in (s, s1, s2, t))
    alpha_s1, alpha_s2, alpha_t = torch.exp(log_alpha_s1), torch.exp(log_alpha_s2), torch.exp(log_alpha_t)
    taylor = dict(k0=1. / r1, k1=1. / r2, k2=r1, k3=r2, rd=r2 - r1)
    if predict_x0:
        phi_11, phi_12, phi_1 = torch.expm1(-r1 * h), torch.expm1(-r2 * h), torch.expm1(-h)
        phi_22 = torch.expm1(-r2 * h) / (r2 * h) + 1.
        phi_2 = phi_1 / h + 1.
        phi_3 = phi_2 / h - 0.5
        mid1 = Update("first", sigma_s1 / sigma_s, alpha_s1 * phi_11)
        mid2 = Update("diff", sigma_s2 / sigma_s, alpha_s2 * phi_12, r2 / r1 * (alpha_s2 * phi_22))
        a, b = sigma_t / sigma_s, alpha_t * phi_1
        if solver_type == 'dpm_solver':
            last = Update("diff", a, b, (1. / r2) * (alpha_t * phi_2))
        else:
            last = Update("singlestep3_taylor", a, b, alpha_t * phi_2, -(alpha_t * phi_3), **taylor)
        return s1, s2, mid1, mid2, last
    phi_11, phi_12, phi_1 = torch.expm1(r1 * h), torch.expm1(r2 * h), torch.expm1(h)
    phi_22 = torch.expm1(r2 * h) / (r2 * h) - 1.
    phi_2 = phi_1 / h - 1.
    phi_3 = phi_2 / h - 0.5
    mid1 = Update("first", torch.exp(log_alpha_s1 - log_alpha_s), sigma_s1 * phi_11)
    mid2 = Update("diff", torch.exp(log_alpha_s2 - log_alpha_s), sigma_s2 * phi_12, -(r2 / r1 * (sigma_s2 * phi_22)))
    a, b = torch.exp(log_alpha_t - log_alpha_s), sigma_t * phi_1
    if solver_type == 'dpm_solver':
        last = Update("diff", a, b, -((1. / r2) * (sigma_t * phi_2)))
    else:
        last = Update("singlestep3_taylor", a, b, -(sigma_t * phi_2), -(sigma_t * phi_3), **taylor)
    return s1, s2, mid1, mid2, last


def multistep_second_update(ns, t_prev_list, t, predict_x0, solver_type):
    """multistep_dpm_solver_second_update (dpm_solver.py:723-778): m0 = model_prev_0 (newest), m1 = model_prev_1"""
    _check_solver_type(solver_type)
    t_prev_1, t_prev_0 = t_prev_list
    lambda_prev_1, lambda_prev_0, lambda_t = (ns.marginal_lambda(v) for v in (t_prev_1, t_prev_0, t))
    log_alpha_prev_0, log_alpha_t = ns.marginal_log_mean_coeff(t_prev_0), ns.marginal_log_mean_coeff(t)
    sigma_prev_0, sigma_t = ns.marginal_std(t_prev_0), ns.marginal_std(t)
    alpha_t = torch.exp(log_alpha_t)
    h_0 = lambda_prev_0 - lambda_prev_1
    h = lambda_t - lambda_prev_0
    k0 = 1. / (h_0 / h)
    if predict_x0:
        a, b = sigma_t / sigma_prev_0, alpha_t * (torch.exp(-h) - 1.)
        c = -(0.5 * (alpha_t * (torch.exp(-h) - 1.))) if solver_type == 'dpm_solver' else \
            alpha_t * ((torch.exp(-h) - 1.) / h + 1.)
    else:
        a, b = torch.exp(log_alpha_t - log_alpha_prev_0), sigma_t * (torch.exp(h) - 1.)
        c = -(0.5 * (sigma_t * (torch.exp(h) - 1.))) if solver_type == 'dpm_solver' else \
            -(sigma_t * ((torch.exp(h) - 1.) / h - 1.))
    return Update("multistep2", a, b, c, k0=k0)


def multistep_third_update(ns, t_prev_list, t, predict_x0):
    """multistep_dpm_solver_third_update (dpm_solver.py:780-825; one form for both solver types): m0 newest, m1, m2"""
    t_prev_2, t_prev_1, t_prev_0 = t_prev_list
    lambda_prev_2, lambda_prev_1, lambda_prev_0, lambda_t = (ns.marginal_lambda(v)
                                                             for v in (t_prev_2, t_prev_1, t_prev_0, t))
    log_alpha_prev_0, log_alpha_t = ns.marginal_log_mean_coeff(t_prev_0), ns.marginal_log_mean_coeff(t)
    sigma_prev_0, sigma_t = ns.marginal_std(t_prev_0), ns.marginal_std(t)
    alpha_t = torch.exp(log_alpha_t)
    h_1 = lambda_prev_1 - lambda_prev_2
    h_0 = lambda_prev_0 - lambda_prev_1
    h = lambda_t - lambda_prev_0
    r0, r1 = h_0 / h, h_1 / h
    ks = dict(k0=1. / r0, k1=1. / r1, k2=r0 / (r0 + r1), k3=1. / (r0 + r1))
    if predict_x0:
        return Update("multistep3", sigma_t / sigma_prev_0, alpha_t * (torch.exp(-h) - 1.),
                      alpha_t * ((torch.exp(-h) - 1.) / h + 1.),
                      -(alpha_t * ((torch.exp(-h) - 1. + h) / h ** 2 - 0.5)), **ks)
    return Update("multistep3", torch.exp(log_alpha_t - log_alpha_prev_0), sigma_t * (torch.exp(h) - 1.),
                  -(sigma_t * ((torch.exp(h) - 1.) / h - 1.)),
                  -(sigma_t * ((torch.exp(h) - 1. - h) / h ** 2 - 0.5)), **ks)
