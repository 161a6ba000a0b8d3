"""Drop-in for the reference's `ldm/models/diffusion/dpm_solver/dpm_solver.py`: `NoiseScheduleVP`, `model_wrapper`,
`DPM_Solver`, `interpolate_fn` and `expand_dims` with the reference's names, signatures and defaults.

Every method of `DPM_Solver.sample` runs: 'multistep', 'singlestep' (DPM-Solver-fast), 'singlestep_fixed' and
'adaptive', orders 1-3, `predict_x0` False (DPM-Solver) or True (DPM-Solver++), the 'dpm_solver' and 'taylor' solver
types, the three skip types, `t_start` / `t_end`, `denoise_to_zero` and dynamic thresholding.  The split of the work:
  * host: every per-update scalar (times, h, r1 / r2, phi terms, sigma / alpha ratios) is formed by
    ctrlora_b200.dpm_schedule with torch CPU fp32 ops in the reference's order;
  * device: each model value (guidance combine, model-type conversion, data prediction) is one
    `ctrlora_dpm_model_output` launch, thresholding one `ctrlora_dpm_threshold`, each update (and each singlestep
    intermediate state) one `ctrlora_dpm_solver_update`, the adaptive error one `ctrlora_dpm_adaptive_error`.
  Given the same model values, x is the reference's to the bit; only the adaptive solver's error norm is summed in a
  different order (DESIGN.md §7).
Model evaluations:
  * `model_wrapper(model.apply_model, ...)` on a ControlLDM evaluates through `DDIMSampler`'s eps pair, as
    `DPMSolverSampler` does: batched classifier-free guidance, CUDA-graph replay and the context cache for a
    `sample()` run; the guidance combine is fused into the model-output kernel.  Any other callable (a lambda around
    apply_model included) is called eagerly: classifier-free guidance concatenates tensor conditions as the reference
    does (:308-311) and calls dict or list conditions once per half;
  * 'classifier' guidance differentiates the user's classifier only (torch autograd); the diffusion model is not
    differentiated.
Differences from the reference: CUDA tensors only (a CPU tensor raises); the schedule is held at fp32; times are
uniform over the batch, as every reference code path makes them; an unknown `method` raises ValueError instead of
returning x unchanged; no tqdm bars.  Two reference failures run here: DPM-Solver-fast with the 'time_uniform' or
'time_quadratic' skip type (the reference's `torch.cumsum` without `dim`, :459-460, raises TypeError) takes the outer
steps that code means, and order-3 multistep with `lower_order_final` and steps < 15 (the reference hands its final
second-order update three history entries, :1066 -> :740, and raises ValueError) gives that update the newest two.
"""
import contextlib
import inspect

import torch

from ctrlora_b200 import dpm_schedule as S
from ctrlora_b200 import ops
from ctrlora_b200.dpm_schedule import NoiseScheduleVP, interpolate_fn  # noqa: F401  (the reference's names)

__all__ = ["NoiseScheduleVP", "model_wrapper", "DPM_Solver", "interpolate_fn", "expand_dims"]


def expand_dims(v, dims):
    """v [N] -> [N, 1, ..., 1] with `dims` dimensions"""
    return v[(...,) + (None,) * (dims - 1)]


def _check_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("ctrlora_b200: DPM_Solver runs on the sm_90a kernels and needs CUDA tensors "
                               "(there is no CPU path)")


def _host_t(t, batch):
    """a time argument as the CPU fp32 [batch] vector the host scalars are formed from"""
    t = torch.as_tensor(t).detach().reshape(-1).to("cpu", torch.float32)
    return t.expand(batch) if t.shape[0] == 1 else t


def _f32(t):
    return t if t.dtype == torch.float32 and t.is_contiguous() else t.float().contiguous()


class _ModelFn:
    """What model_wrapper returns: the reference's `model_fn(x, t_continuous) -> noise`, and `output()`, which writes
    a (data) prediction into a history slot with one kernel launch."""

    def __init__(self, model, noise_schedule, model_type, model_kwargs, guidance_type, condition,
                 unconditional_condition, guidance_scale, classifier_fn, classifier_kwargs, batched_cfg,
                 use_cuda_graph):
        self.model, self.ns, self.model_type = model, noise_schedule, model_type
        self.model_kwargs, self.guidance_type = dict(model_kwargs), guidance_type
        self.condition, self.unconditional_condition = condition, unconditional_condition
        self.guidance_scale, self.classifier_fn, self.classifier_kwargs = guidance_scale, classifier_fn, classifier_kwargs
        self.eps = None
        owner = getattr(model, "__self__", None)
        graphable = guidance_type == "classifier-free" and not self.model_kwargs or set(self.model_kwargs) == {"cond"}
        if inspect.ismethod(model) and model.__name__ == "apply_model" and hasattr(owner, "control_model") and graphable:
            from cldm.ddim_hacked import DDIMSampler
            self.eps = DDIMSampler(owner, batched_cfg=batched_cfg, use_cuda_graph=use_cuda_graph)

    def run(self):
        """a sampling run: constant conditioning, so the graph path caches the text context's projections"""
        return contextlib.nullcontext() if self.eps is None else self.eps._run_mode(self.eps)

    def _cfg(self):
        return self.guidance_type == "classifier-free" and not (self.guidance_scale == 1. or
                                                                self.unconditional_condition is None)

    def _evaluate(self, x, t_in):
        """(out_cond, out_uncond | None): the model's raw outputs at the model input time t_in (device [B])"""
        cond = self.condition if self.guidance_type == "classifier-free" else self.model_kwargs.get("cond")
        if self.eps is not None:
            return self.eps._eps_pair(x, t_in, cond, self.unconditional_condition, self._cfg())
        kw = self.model_kwargs
        if self._cfg():
            uc, c = self.unconditional_condition, self.condition
            if torch.is_tensor(c) and torch.is_tensor(uc):   # the reference's one batched call (:308-311)
                out_u, out_c = self.model(torch.cat([x] * 2), torch.cat([t_in] * 2), torch.cat([uc, c]), **kw).chunk(2)
                return out_c, out_u
            return self.model(x, t_in, c, **kw), self.model(x, t_in, uc, **kw)
        if self.guidance_type == "classifier-free":
            return self.model(x, t_in, self.condition, **kw), None
        return self.model(x, t_in, **kw), None

    def _cond_grad(self, x, t_in):
        """nabla_x log p_t(cond | x_t) of the user's classifier (:280-287)"""
        assert self.classifier_fn is not None
        with torch.enable_grad():
            x_in = x.detach().requires_grad_(True)
            log_prob = self.classifier_fn(x_in, t_in, self.condition, **self.classifier_kwargs)
            return torch.autograd.grad(log_prob.sum(), x_in)[0]

    def output(self, x, t, predict_x0=False, alpha_t=None, sigma_t=None):
        """noise (or with predict_x0 the data prediction (x - sigma_t noise) / alpha_t) at host times t [B]"""
        ns = self.ns
        t_in = ns.model_input_time(t)
        if bool((t_in == t_in[0]).all()):   # a device fill, not a pageable copy that would wait for the stream
            t_in = torch.full(t_in.shape, float(t_in[0]), device=x.device, dtype=torch.float32)
        else:
            t_in = t_in.to(x.device)
        out_c, out_u = self._evaluate(x, t_in)
        args = dict(model_type=self.model_type, predict_x0=predict_x0, scale=self.guidance_scale)
        if self.model_type != "noise":
            args.update(alpha_w=S._s(ns.marginal_alpha(t)), sigma_w=S._s(ns.marginal_std(t)))
        grad = None
        if self.guidance_type == "classifier":
            grad = _f32(self._cond_grad(x, t_in))
            args["grad_coef"] = S._s(self.guidance_scale * ns.marginal_std(t))
        if predict_x0:
            args.update(alpha_t=S._s(alpha_t), sigma_t=S._s(sigma_t))
        return ops.dpm_model_output(x, _f32(out_c), torch.empty_like(x), out_uncond=None if out_u is None else _f32(out_u),
                                    grad=grad, **args)

    def __call__(self, x, t_continuous):
        _check_cuda(x)
        x = _f32(x)
        return self.output(x, _host_t(t_continuous, x.shape[0]))


def model_wrapper(model, noise_schedule, model_type="noise", model_kwargs={}, guidance_type="uncond", condition=None,
                  unconditional_condition=None, guidance_scale=1., classifier_fn=None, classifier_kwargs={},
                  batched_cfg=True, use_cuda_graph=True):
    """The reference's model_wrapper (dpm_solver.py:161-316): a noise prediction function of (x, t_continuous) for
    the 'noise' / 'x_start' / 'v' model types and 'uncond' / 'classifier' / 'classifier-free' guidance.
    `batched_cfg` / `use_cuda_graph` choose the evaluation policy of the graph path (a ControlLDM's bound
    apply_model); other models ignore them."""
    assert model_type in ["noise", "x_start", "v"]
    assert guidance_type in ["uncond", "classifier", "classifier-free"]
    return _ModelFn(model, noise_schedule, model_type, model_kwargs, guidance_type, condition, unconditional_condition,
                    guidance_scale, classifier_fn, classifier_kwargs, batched_cfg, use_cuda_graph)


class DPM_Solver:
    def __init__(self, model_fn, noise_schedule, predict_x0=False, thresholding=False, max_val=1.):
        """DPM-Solver (predict_x0=False) or DPM-Solver++ (predict_x0=True, optionally with the dynamic thresholding
        of Imagen) for a noise prediction function `model_fn(x, t_continuous)`, best one from model_wrapper."""
        self.model = model_fn
        self.noise_schedule = noise_schedule
        self.predict_x0 = predict_x0
        self.thresholding = thresholding
        self.max_val = max_val

    # ---- model values
    def _value(self, x, t, predict_x0):
        _check_cuda(x)
        x = _f32(x)
        ns, th = self.noise_schedule, _host_t(t, x.shape[0])
        alpha_t = sigma_t = None
        if predict_x0:
            alpha_t, sigma_t = ns.marginal_alpha(th), ns.marginal_std(th)
        if isinstance(self.model, _ModelFn):
            m = self.model.output(x, th, predict_x0, alpha_t, sigma_t)
        else:
            noise = self.model(x, th.to(x.device))
            if not predict_x0:
                return noise
            m = ops.dpm_model_output(x, _f32(noise), torch.empty_like(x), predict_x0=True, sigma_t=S._s(sigma_t),
                                     alpha_t=S._s(alpha_t))
        if predict_x0 and self.thresholding:
            k_lo, k_hi, weight = S.quantile_rank(m[0].numel())
            ops.dpm_threshold_(m, k_lo, k_hi, weight, self.max_val)
        return m

    def noise_prediction_fn(self, x, t):
        return self._value(x, t, False)

    def data_prediction_fn(self, x, t):
        """the data prediction, with dynamic thresholding when enabled (dpm_solver.py:352-365)"""
        return self._value(x, t, True)

    def model_fn(self, x, t):
        return self._value(x, t, self.predict_x0)

    def get_time_steps(self, skip_type, t_T, t_0, N, device):
        return S.get_time_steps(self.noise_schedule, skip_type, t_T, t_0, N).to(device)

    def get_orders_and_timesteps_for_singlestep_solver(self, steps, order, skip_type, t_T, t_0, device):
        ts, orders = S.get_orders_and_timesteps_for_singlestep_solver(self.noise_schedule, steps, order, skip_type,
                                                                      t_T, t_0)
        return ts.to(device), orders

    def denoise_to_zero_fn(self, x, s):
        return self.data_prediction_fn(x, s)

    # ---- updates: host scalars from dpm_schedule, one kernel launch per state
    @staticmethod
    def _apply(u, x, m0, m1=None, m2=None):
        _check_cuda(x)
        return ops.dpm_solver_update(u.mode, _f32(x), m0, u.coef, m1, m2)

    def dpm_solver_first_update(self, x, s, t, model_s=None, return_intermediate=False):
        b = x.shape[0]
        s, t = _host_t(s, b), _host_t(t, b)
        u = S.first_update(self.noise_schedule, s, t, self.predict_x0)
        if model_s is None:
            model_s = self.model_fn(x, s)
        x_t = self._apply(u, x, model_s)
        return (x_t, {'model_s': model_s}) if return_intermediate else x_t

    def singlestep_dpm_solver_second_update(self, x, s, t, r1=0.5, model_s=None, return_intermediate=False,
                                            solver_type='dpm_solver'):
        b = x.shape[0]
        s, t = _host_t(s, b), _host_t(t, b)
        s1, mid, last = S.singlestep_second_update(self.noise_schedule, s, t, r1, self.predict_x0, solver_type)
        if model_s is None:
            model_s = self.model_fn(x, s)
        model_s1 = self.model_fn(self._apply(mid, x, model_s), s1)
        x_t = self._apply(last, x, model_s, model_s1)
        return (x_t, {'model_s': model_s, 'model_s1': model_s1}) if return_intermediate else x_t

    def singlestep_dpm_solver_third_update(self, x, s, t, r1=1. / 3., r2=2. / 3., model_s=None, model_s1=None,
                                           return_intermediate=False, solver_type='dpm_solver'):
        b = x.shape[0]
        s, t = _host_t(s, b), _host_t(t, b)
        s1, s2, mid1, mid2, last = S.singlestep_third_update(self.noise_schedule, s, t, r1, r2, self.predict_x0,
                                                             solver_type)
        if model_s is None:
            model_s = self.model_fn(x, s)
        if model_s1 is None:
            model_s1 = self.model_fn(self._apply(mid1, x, model_s), s1)
        model_s2 = self.model_fn(self._apply(mid2, x, model_s, model_s1), s2)
        if last.mode == "diff":
            x_t = self._apply(last, x, model_s, model_s2)
        else:
            x_t = self._apply(last, x, model_s, model_s1, model_s2)
        if return_intermediate:
            return x_t, {'model_s': model_s, 'model_s1': model_s1, 'model_s2': model_s2}
        return x_t

    def multistep_dpm_solver_second_update(self, x, model_prev_list, t_prev_list, t, solver_type="dpm_solver"):
        b = x.shape[0]
        u = S.multistep_second_update(self.noise_schedule, [_host_t(v, b) for v in t_prev_list], _host_t(t, b),
                                      self.predict_x0, solver_type)
        model_prev_1, model_prev_0 = model_prev_list
        return self._apply(u, x, model_prev_0, model_prev_1)

    def multistep_dpm_solver_third_update(self, x, model_prev_list, t_prev_list, t, solver_type='dpm_solver'):
        b = x.shape[0]
        u = S.multistep_third_update(self.noise_schedule, [_host_t(v, b) for v in t_prev_list], _host_t(t, b),
                                     self.predict_x0)
        model_prev_2, model_prev_1, model_prev_0 = model_prev_list
        return self._apply(u, x, model_prev_0, model_prev_1, model_prev_2)

    def singlestep_dpm_solver_update(self, x, s, t, order, return_intermediate=False, solver_type='dpm_solver', r1=None,
                                     r2=None):
        if order == 1:
            return self.dpm_solver_first_update(x, s, t, return_intermediate=return_intermediate)
        if order == 2:
            return self.singlestep_dpm_solver_second_update(x, s, t, return_intermediate=return_intermediate,
                                                            solver_type=solver_type, r1=r1)
        if order == 3:
            return self.singlestep_dpm_solver_third_update(x, s, t, return_intermediate=return_intermediate,
                                                           solver_type=solver_type, r1=r1, r2=r2)
        raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))

    def multistep_dpm_solver_update(self, x, model_prev_list, t_prev_list, t, order, solver_type='dpm_solver'):
        if order == 1:
            return self.dpm_solver_first_update(x, t_prev_list[-1], t, model_s=model_prev_list[-1])
        if order == 2:   # the newest two: order-3 runs drop to order 2 for their final steps
            return self.multistep_dpm_solver_second_update(x, model_prev_list[-2:], t_prev_list[-2:], t,
                                                           solver_type=solver_type)
        if order == 3:
            return self.multistep_dpm_solver_third_update(x, model_prev_list, t_prev_list, t, solver_type=solver_type)
        raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))

    def dpm_solver_adaptive(self, x, order, t_T, t_0, h_init=0.05, atol=0.0078, rtol=0.05, theta=0.9, t_err=1e-5,
                            solver_type='dpm_solver'):
        """DPM-Solver-12 / -23 (dpm_solver.py:878-937).  The step control runs on the host on [B] fp32 times as in
        the reference; each iteration reads the device error E once."""
        if order not in (2, 3):
            raise ValueError("For adaptive step size solver, order must be 2 or 3, got {}".format(order))
        _check_cuda(x)
        x = _f32(x)
        ns = self.noise_schedule
        s = t_T * torch.ones((x.shape[0],))
        lambda_s = ns.marginal_lambda(s)
        lambda_0 = ns.marginal_lambda(t_0 * torch.ones_like(s))
        h = h_init * torch.ones_like(s)
        x_prev = x
        nfe = 0
        if order == 2:
            r1 = 0.5
            lower_update = lambda x, s, t: self.dpm_solver_first_update(x, s, t, return_intermediate=True)
            higher_update = lambda x, s, t, **kw: self.singlestep_dpm_solver_second_update(
                x, s, t, r1=r1, solver_type=solver_type, **kw)
        else:
            r1, r2 = 1. / 3., 2. / 3.
            lower_update = lambda x, s, t: self.singlestep_dpm_solver_second_update(
                x, s, t, r1=r1, return_intermediate=True, solver_type=solver_type)
            higher_update = lambda x, s, t, **kw: self.singlestep_dpm_solver_third_update(
                x, s, t, r1=r1, r2=r2, solver_type=solver_type, **kw)
        err = torch.empty(1, device=x.device, dtype=torch.float32)
        while torch.abs((s - t_0)).mean() > t_err:
            t = ns.inverse_lambda(lambda_s + h)
            x_lower, lower_noise_kwargs = lower_update(x, s, t)
            x_higher = higher_update(x, s, t, **lower_noise_kwargs)
            E = ops.dpm_adaptive_error(x_lower, x_prev, x_higher, atol, rtol, err=err).cpu()[0]
            if torch.all(E <= 1.):
                x = x_higher
                s = t
                x_prev = x_lower
                lambda_s = ns.marginal_lambda(s)
            h = torch.min(theta * h * torch.float_power(E, -1. / order).float(), lambda_0 - lambda_s)
            nfe += order
        print('adaptive solver nfe', nfe)
        return x

    def sample(self, x, steps=20, t_start=None, t_end=None, order=3, skip_type='time_uniform', method='singlestep',
               lower_order_final=True, denoise_to_zero=False, solver_type='dpm_solver', atol=0.0078, rtol=0.05):
        """DPM_Solver.sample (dpm_solver.py:939-1097): x at t_end from x at t_start"""
        if method not in ('singlestep', 'multistep', 'singlestep_fixed', 'adaptive'):
            raise ValueError("Unsupported method {}, need to be 'singlestep', 'multistep', 'singlestep_fixed' or "
                             "'adaptive'".format(method))
        _check_cuda(x)
        x = _f32(x)
        ns = self.noise_schedule
        t_0 = 1. / ns.total_N if t_end is None else t_end
        t_T = ns.T if t_start is None else t_start
        b = x.shape[0]
        run = self.model.run() if isinstance(self.model, _ModelFn) else contextlib.nullcontext()
        with torch.no_grad(), run:
            if method == 'adaptive':
                x = self.dpm_solver_adaptive(x, order=order, t_T=t_T, t_0=t_0, atol=atol, rtol=rtol,
                                             solver_type=solver_type)
            elif method == 'multistep':
                assert steps >= order
                timesteps = S.get_time_steps(ns, skip_type, t_T, t_0, steps)
                assert timesteps.shape[0] - 1 == steps
                vec_t = timesteps[0].expand(b)
                model_prev_list, t_prev_list = [self.model_fn(x, vec_t)], [vec_t]
                for init_order in range(1, order):   # the first `order` values by lower-order multistep updates
                    vec_t = timesteps[init_order].expand(b)
                    x = self.multistep_dpm_solver_update(x, model_prev_list, t_prev_list, vec_t, init_order,
                                                         solver_type=solver_type)
                    model_prev_list.append(self.model_fn(x, vec_t))
                    t_prev_list.append(vec_t)
                for step in range(order, steps + 1):
                    vec_t = timesteps[step].expand(b)
                    step_order = min(order, steps + 1 - step) if lower_order_final and steps < 15 else order
                    x = self.multistep_dpm_solver_update(x, model_prev_list, t_prev_list, vec_t, step_order,
                                                         solver_type=solver_type)
                    model_prev_list, t_prev_list = model_prev_list[1:] + model_prev_list[-1:], t_prev_list[1:] + [vec_t]
                    if step < steps:   # no model value after the final update
                        model_prev_list[-1] = self.model_fn(x, vec_t)
            else:
                if method == 'singlestep':
                    timesteps_outer, orders = S.get_orders_and_timesteps_for_singlestep_solver(
                        ns, steps, order, skip_type, t_T, t_0)
                else:
                    orders = [order] * (steps // order)
                    timesteps_outer = S.get_time_steps(ns, skip_type, t_T, t_0, len(orders))
                for i, step_order in enumerate(orders):
                    t_T_inner, t_0_inner = timesteps_outer[i], timesteps_outer[i + 1]
                    timesteps_inner = S.get_time_steps(ns, skip_type, t_T_inner.item(), t_0_inner.item(), step_order)
                    lambda_inner = ns.marginal_lambda(timesteps_inner)
                    vec_s, vec_t = t_T_inner.tile(b), t_0_inner.tile(b)
                    h = lambda_inner[-1] - lambda_inner[0]
                    r1 = None if step_order <= 1 else (lambda_inner[1] - lambda_inner[0]) / h
                    r2 = None if step_order <= 2 else (lambda_inner[2] - lambda_inner[0]) / h
                    x = self.singlestep_dpm_solver_update(x, vec_s, vec_t, step_order, solver_type=solver_type,
                                                          r1=r1, r2=r2)
            if denoise_to_zero:
                x = self.denoise_to_zero_fn(x, torch.ones((b,)) * t_0)
        return x
