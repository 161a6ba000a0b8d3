"""Drop-in for the reference's `cldm/ddim_hacked.py`: `DDIMSampler` with the same methods, arguments and return
values.  Differences that do not change results:
  * `register_buffer` follows `model.device` (the reference hard-codes 'cuda', :17-21);
  * the per-step update (CFG combine, pred_x0, dir_xt, x_prev; reference :190-231, ~10 elementwise kernels plus four
    `torch.full`) is ONE kernel, `ctrlora_ddim_update`, with the same fp32 operation order (bit-identical outputs);
  * the two `apply_model` passes of classifier-free guidance run as one batch-2B pass (`batched_cfg=True`, the
    upstream ldm/models/diffusion/ddim.py:190-211 behaviour; set False for the reference's two sequential passes);
  * with fixed shapes the whole step is replayed from a CUDA graph (`use_cuda_graph=True`).
"""
import numpy as np
import torch
from tqdm import tqdm

from ctrlora_b200 import ops
from ctrlora_b200.graph import GraphedCallable
from ldm.modules.diffusionmodules.util import (extract_into_tensor, make_ddim_sampling_parameters,  # noqa: F401
                                               make_ddim_timesteps, noise_like)


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", batched_cfg=True, use_cuda_graph=True, **kwargs):
        super().__init__()
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.batched_cfg = batched_cfg
        self.use_cuda_graph = use_cuda_graph
        self._graph = None
        self._graph_key = None
        self._graphs = {}
        self._fp_params = None
        self._fp_ptr = None
        self._fp_calls = 0
        self._ctx_cache_mode = False   # True inside ddim_sampling / encode / decode: the conditioning is constant over the run
        self._cfg_buf = None
        self.last_stats = None

    def register_buffer(self, name, attr):
        if type(attr) == torch.Tensor and attr.device != self.model.device:
            attr = attr.to(self.model.device)
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        self.ddim_timesteps = make_ddim_timesteps(ddim_discr_method=ddim_discretize, num_ddim_timesteps=ddim_num_steps,
                                                  num_ddpm_timesteps=self.ddpm_num_timesteps, verbose=verbose)
        alphas_cumprod = self.model.alphas_cumprod
        assert alphas_cumprod.shape[0] == self.ddpm_num_timesteps, 'alphas have to be defined for each timestep'
        to_torch = lambda x: x.clone().detach().to(torch.float32).to(self.model.device)
        ac_cpu = alphas_cumprod.cpu()
        self.register_buffer('betas', to_torch(self.model.betas))
        self.register_buffer('alphas_cumprod', to_torch(alphas_cumprod))
        self.register_buffer('alphas_cumprod_prev', to_torch(self.model.alphas_cumprod_prev))
        self.register_buffer('sqrt_alphas_cumprod', to_torch(np.sqrt(ac_cpu)))
        self.register_buffer('sqrt_one_minus_alphas_cumprod', to_torch(np.sqrt(1. - ac_cpu)))
        self.register_buffer('log_one_minus_alphas_cumprod', to_torch(np.log(1. - ac_cpu)))
        self.register_buffer('sqrt_recip_alphas_cumprod', to_torch(np.sqrt(1. / ac_cpu)))
        self.register_buffer('sqrt_recipm1_alphas_cumprod', to_torch(np.sqrt(1. / ac_cpu - 1)))
        # per-index scalars stay on the host: they become kernel arguments, not device tensors
        sigmas, alphas, alphas_prev = make_ddim_sampling_parameters(alphacums=ac_cpu, ddim_timesteps=self.ddim_timesteps,
                                                                    eta=ddim_eta, verbose=verbose)
        self.ddim_sigmas = sigmas
        self.ddim_alphas = alphas
        self.ddim_alphas_prev = alphas_prev
        self.ddim_sqrt_one_minus_alphas = np.sqrt(1. - alphas)
        sigmas_orig = ddim_eta * torch.sqrt((1 - self.alphas_cumprod_prev) / (1 - self.alphas_cumprod) *
                                            (1 - self.alphas_cumprod / self.alphas_cumprod_prev))
        self.register_buffer('ddim_sigmas_for_original_num_steps', sigmas_orig)

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None, img_callback=None,
               quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None,
               corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, dynamic_threshold=None, ucg_schedule=None, **kwargs):
        if conditioning is not None and verbose:
            ctmp = conditioning
            if isinstance(ctmp, dict):
                ctmp = ctmp[list(ctmp.keys())[0]]
                while isinstance(ctmp, list):
                    ctmp = ctmp[0]
                if torch.is_tensor(ctmp) and ctmp.shape[0] != batch_size:
                    print(f"Warning: Got {ctmp.shape[0]} conditionings but batch-size is {batch_size}")
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta, verbose=verbose)
        C, H, W = shape
        size = (batch_size, C, H, W)
        if verbose:
            print(f'Data shape for DDIM sampling is {size}, eta {eta}')
        return self.ddim_sampling(conditioning, size, callback=callback, img_callback=img_callback,
                                  quantize_denoised=quantize_x0, mask=mask, x0=x0, ddim_use_original_steps=False,
                                  noise_dropout=noise_dropout, temperature=temperature, score_corrector=score_corrector,
                                  corrector_kwargs=corrector_kwargs, x_T=x_T, log_every_t=log_every_t,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning,
                                  dynamic_threshold=dynamic_threshold, ucg_schedule=ucg_schedule, verbose=verbose)

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, callback=None, timesteps=None,
                      quantize_denoised=False, mask=None, x0=None, img_callback=None, log_every_t=100, temperature=1.,
                      noise_dropout=0., score_corrector=None, corrector_kwargs=None, unconditional_guidance_scale=1.,
                      unconditional_conditioning=None, dynamic_threshold=None, ucg_schedule=None, verbose=True):
        device = self.model.betas.device
        b = shape[0]
        img = torch.randn(shape, device=device) if x_T is None else x_T
        if timesteps is None:
            timesteps = self.ddpm_num_timesteps if ddim_use_original_steps else self.ddim_timesteps
        elif not ddim_use_original_steps:
            subset_end = int(min(timesteps / self.ddim_timesteps.shape[0], 1) * self.ddim_timesteps.shape[0]) - 1
            timesteps = self.ddim_timesteps[:subset_end]
        intermediates = {'x_inter': [img], 'pred_x0': [img]}
        time_range = list(reversed(range(0, timesteps))) if ddim_use_original_steps else np.flip(timesteps)
        total_steps = timesteps if ddim_use_original_steps else timesteps.shape[0]
        if verbose:
            print(f"Running DDIM Sampling with {total_steps} timesteps")
        iterator = tqdm(time_range, desc='DDIM Sampler', total=total_steps, disable=not verbose)
        ts_all = self._step_tensors(time_range, b, device)  # every step's `ts` in one host->device copy
        with self._run_mode(self):  # constant conditioning over the run: K / V^T of the text context projected once
            for i, step in enumerate(iterator):
                index = total_steps - i - 1
                ts = ts_all[i]
                if mask is not None:
                    assert x0 is not None
                    img_orig = self.model.q_sample(x0, ts)
                    img = img_orig * mask + (1. - mask) * img
                if ucg_schedule is not None:
                    assert len(ucg_schedule) == len(time_range)
                    unconditional_guidance_scale = ucg_schedule[i]
                img, pred_x0 = self.p_sample_ddim(img, cond, ts, index=index, use_original_steps=ddim_use_original_steps,
                                                  quantize_denoised=quantize_denoised, temperature=temperature,
                                                  noise_dropout=noise_dropout, score_corrector=score_corrector,
                                                  corrector_kwargs=corrector_kwargs,
                                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                                  unconditional_conditioning=unconditional_conditioning,
                                                  dynamic_threshold=dynamic_threshold)
                if callback:
                    callback(i)
                if img_callback:
                    img_callback(pred_x0, i)
                if index % log_every_t == 0 or index == total_steps - 1:
                    intermediates['x_inter'].append(img)
                    intermediates['pred_x0'].append(pred_x0)
        return img, intermediates

    @staticmethod
    def _step_tensors(steps, batch, device):
        """int64 [len(steps), batch]: row i is the reference's `torch.full((b,), step)` of step i (ddim_hacked.py:152)"""
        steps = [int(v) for v in steps]
        host = torch.tensor(steps, dtype=torch.long)[:, None].expand(len(steps), batch).contiguous()
        return host.to(device, non_blocking=False)

    # ---------------------------------------------------------------------------------------------- eps prediction
    @staticmethod
    def _flat_cond(c):
        """(keys, tensors) of a {'c_crossattn': [T], 'c_concat': [T] | None, ...} dict, or None if not that shape."""
        if not isinstance(c, dict):
            return None
        keys, tensors = [], []
        for k in sorted(c):
            v = c[k]
            if v is None:
                keys.append((k, None))
            elif isinstance(v, list) and all(torch.is_tensor(t) for t in v):
                keys.append((k, len(v)))
                tensors += v
            else:
                return None
        return tuple(keys), tensors

    @staticmethod
    def _rebuild(keys, tensors):
        out, i = {}, 0
        for k, n in keys:
            if n is None:
                out[k] = None
            else:
                out[k] = list(tensors[i:i + n])
                i += n
        return out

    def _weights_fingerprint(self, full=False):
        """State of everything a captured apply_model graph bakes in besides shapes: the kernel-layout weight copies
        (ctrlora_b200.prepare) are built during warm-up, outside the capture, so a `load_state_dict` /
        `copy_weights_to_switchable` / optimizer step on the same model (the reference's gradio app re-uses one sampler
        across checkpoints, app/gradio_ctrlora.py) must invalidate the graph.  torch bumps `_version` on every in-place
        write (summed over the 1 174 parameters every call: ~60 us); storage swaps (`p.data = ...`) bump
        prepare.STRUCT_VERSION when this package does them, and the storage pointers themselves are re-verified at the start
        of every sampling run and every 64th call (`full`); the trainer's fused AdamW bumps prepare.TRAIN_VERSION."""
        from ctrlora_b200 import prepare
        if self._fp_params is None:
            # parameters and buffers (the IP-Adapter's `ip_scale` is a buffer the style app rewrites per request)
            self._fp_params = [t for m in (self.model.control_model, self.model.model.diffusion_model)
                               for t in list(m.parameters()) + list(m.buffers())]
        ver = sum([p._version for p in self._fp_params])
        self._fp_calls += 1
        if full or self._fp_ptr is None or self._fp_calls % 64 == 0:
            ptr = 0
            for p in self._fp_params:
                ptr ^= p.data_ptr()
            self._fp_ptr = ptr
        lw = getattr(self.model, "lora_weights", None)
        return (ver, self._fp_ptr, len(self._fp_params), prepare.TRAIN_VERSION, prepare.STRUCT_VERSION,
                None if lw is None else tuple(float(w) for w in lw))

    def _cfg_inputs(self, x, t, cond_tensors, uncond_tensors):
        """[cond | uncond] batch of one CFG step in persistent buffers: plain device-to-device copies (no ATen cat
        kernels per step); the conditioning halves are re-copied only when their tensors change."""
        b = x.shape[0]
        sig = (tuple(x.shape), x.dtype, t.dtype, tuple((tuple(a.shape), a.dtype) for a in cond_tensors))
        if self._cfg_buf is None or self._cfg_buf["sig"] != sig:
            mk = lambda a: torch.empty((2 * a.shape[0],) + tuple(a.shape[1:]), device=a.device, dtype=a.dtype)
            self._cfg_buf = {"sig": sig, "x": mk(x), "t": mk(t), "c": [mk(a) for a in cond_tensors], "src": None}
        buf = self._cfg_buf
        buf["x"][:b].copy_(x, non_blocking=True)
        buf["x"][b:].copy_(x, non_blocking=True)
        buf["t"][:b].copy_(t, non_blocking=True)
        buf["t"][b:].copy_(t, non_blocking=True)
        src = tuple((a.data_ptr(), a._version, u.data_ptr(), u._version) for a, u in zip(cond_tensors, uncond_tensors))
        if buf["src"] != src:
            for dst, a, u in zip(buf["c"], cond_tensors, uncond_tensors):
                dst[:b].copy_(a, non_blocking=True)
                dst[b:].copy_(u, non_blocking=True)
            buf["src"] = src
        return buf["x"], buf["t"], buf["c"]

    def _eps_pair(self, x, t, c, uc, use_cfg):
        """(e_cond, e_uncond | None) with the policy chosen at construction (batched CFG, CUDA graph)."""
        if not use_cfg:
            return self._apply(x, t, c), None
        fc, fu = self._flat_cond(c), self._flat_cond(uc)
        if self.batched_cfg and fc is not None and fu is not None and fc[0] == fu[0] and \
                all(a.shape == b_.shape for a, b_ in zip(fc[1], fu[1])):
            b = x.shape[0]
            x2, t2, both = self._cfg_inputs(x, t, fc[1], fu[1])
            e = self._apply(x2, t2, self._rebuild(fc[0], both), persistent=True)
            return e[:b], e[b:]
        e_c = self._apply(x, t, c)
        if self.use_cuda_graph:
            e_c = e_c.clone()  # the graph's static output buffer is overwritten by the second replay
        return e_c, self._apply(x, t, uc)

    def _apply(self, x, t, c, persistent=False):
        ctx_mode = False
        if self._ctx_cache_mode:
            cc = c.get("c_crossattn") if isinstance(c, dict) else None
            if isinstance(cc, list) and len(cc) == 1 and torch.is_tensor(cc[0]) and hasattr(self.model, "prepare_context"):
                # inside a sampling run the text conditioning is step-invariant: its K / V^T projections are computed once
                # (idempotent call) instead of 32 small GEMMs per step; graphs captured in this mode do not contain them
                self.model.prepare_context(cc[0])
                ctx_mode = True
        flat = self._flat_cond(c)
        if not self.use_cuda_graph or flat is None or not x.is_cuda:
            return self.model.apply_model(x, t, c)
        keys, tensors = flat
        # t's dtype is part of the key: a graph captured with int64 t would copy_ a float t (DPM-Solver's fractional
        # model times) into its int64 static input, truncating it
        key = (keys, tuple(x.shape), t.dtype, tuple(tuple(tt.shape) for tt in tensors), tuple(self.model.control_scales),
               self.model.only_mid_control, ctx_mode, self._weights_fingerprint())
        if self._graph is None or self._graph_key != key:
            cached = self._graphs.pop(key, None)  # a sampler alternates between at most a few keys (run mode on / off)
            if cached is None:
                # the callable must not refer to the sampler: the sampler holds the graph, and a cycle through it would
                # keep a dropped sampler's graph pools (and its model) on the device until a cyclic collection, which a
                # process that has called gc.freeze() never runs
                model, rebuild = self.model, self._rebuild
                fn = lambda xx, tt, *cs: model.apply_model(xx, tt, rebuild(keys, list(cs)))
                cached = GraphedCallable(fn, [x, t] + tensors, adopt_inputs=persistent)
            if self._graph is not None:
                self._graphs[self._graph_key] = self._graph
                while len(self._graphs) > 1:  # keep one spare graph (each owns its activation pool)
                    self._graphs.pop(next(iter(self._graphs)))
            self._graph, self._graph_key = cached, key
        return self._graph(x, t, *tensors)

    def run_mode(self):
        """`with sampler.run_mode(): ...` around a loop of p_sample_ddim calls whose conditioning does not change (what
        sample() / encode() / decode() do themselves): the text context's K / V^T projections are computed once."""
        return self._run_mode(self)

    class _run_mode:
        """context manager: marks a sampling run (constant conditioning; storage pointers re-verified once at its start)"""

        def __init__(self, sampler):
            self.s = sampler

        def __enter__(self):
            self.prev = self.s._ctx_cache_mode
            self.s._ctx_cache_mode = True
            self.s._fp_ptr = None  # full fingerprint on the run's first step
            return self.s

        def __exit__(self, *exc):
            self.s._ctx_cache_mode = self.prev
            return False

    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1., noise_dropout=0., score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1., unconditional_conditioning=None, dynamic_threshold=None):
        if score_corrector is not None or quantize_denoised or dynamic_threshold is not None or noise_dropout > 0.:
            raise NotImplementedError("score_corrector / quantize_denoised / dynamic_threshold / noise_dropout are not "
                                      "on the CtrLoRA path")
        if self.model.parameterization == "v":
            raise NotImplementedError("v-parameterisation is not on the CtrLoRA path")
        b, device = x.shape[0], x.device
        use_cfg = not (unconditional_conditioning is None or unconditional_guidance_scale == 1.)
        e_cond, e_uncond = self._eps_pair(x, t, c, unconditional_conditioning, use_cfg)
        if use_original_steps:
            a_t, a_prev = float(self.model.alphas_cumprod[index]), float(self.model.alphas_cumprod_prev[index])
            sqrt_1m = float(self.model.sqrt_one_minus_alphas_cumprod[index])
            sigma_t = float(self.ddim_sigmas_for_original_num_steps[index])
        else:
            a_t, a_prev = float(self.ddim_alphas[index]), float(self.ddim_alphas_prev[index])
            sqrt_1m, sigma_t = float(self.ddim_sqrt_one_minus_alphas[index]), float(self.ddim_sigmas[index])
        # the reference draws noise every step and multiplies it by sigma_t (= 0 at eta 0); drawing only when it is
        # used changes nothing but the global RNG position after sampling
        noise = noise_like(x.shape, device, repeat_noise) if sigma_t != 0. else None
        stats = torch.empty(b, device=device, dtype=torch.float32)
        x_prev, pred_x0 = ops.ddim_update(x.float().contiguous(), e_cond.float().contiguous(),
                                          None if e_uncond is None else e_uncond.float().contiguous(),
                                          unconditional_guidance_scale, a_t, a_prev, sigma_t, sqrt_1m, noise=noise,
                                          temperature=temperature, stats=stats)
        self.last_stats = stats  # sum(x_prev^2) per image: a cheap per-step health metric for callers
        return x_prev, pred_x0

    # ---------------------------------------------------------------------------------------------- encode / decode
    def _tables(self, use_original_steps, device):
        """(alpha table, sqrt(alpha), sqrt(1 - alpha)) as fp32 device tensors for either schedule."""
        if use_original_steps:
            return self.alphas_cumprod, self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod
        a = torch.as_tensor(self.ddim_alphas, dtype=torch.float32).to(device)
        return a, torch.sqrt(a), torch.as_tensor(self.ddim_sqrt_one_minus_alphas, dtype=torch.float32).to(device)

    @torch.no_grad()
    def stochastic_encode(self, x0, t, use_original_steps=False, noise=None):
        """x_t = sqrt(a_t) x0 + sqrt(1 - a_t) noise with t indexing the chosen schedule (reference :281-296): the same
        gather-and-blend kernel as q_sample."""
        _, sqrt_a, sqrt_1m = self._tables(use_original_steps, x0.device)
        if noise is None:
            noise = torch.randn_like(x0)
        return ops.q_sample(x0, noise, t, sqrt_a, sqrt_1m)

    @torch.no_grad()
    def decode(self, x_latent, cond, t_start, unconditional_guidance_scale=1.0, unconditional_conditioning=None,
               use_original_steps=False, callback=None):
        """Run the last `t_start` sampler steps from x_latent (reference :298-317)."""
        steps = (np.arange(self.ddpm_num_timesteps) if use_original_steps else self.ddim_timesteps)[:t_start]
        x_dec = x_latent
        ts_all = self._step_tensors(steps, x_latent.shape[0], x_latent.device)
        with self._run_mode(self):
            for i, index in enumerate(range(len(steps) - 1, -1, -1)):
                x_dec, _ = self.p_sample_ddim(x_dec, cond, ts_all[index], index=index, use_original_steps=use_original_steps,
                                              unconditional_guidance_scale=unconditional_guidance_scale,
                                              unconditional_conditioning=unconditional_conditioning)
                if callback:
                    callback(i)
        return x_dec

    @torch.no_grad()
    def encode(self, x0, c, t_enc, use_original_steps=False, return_intermediates=None,
               unconditional_guidance_scale=1.0, unconditional_conditioning=None, callback=None):
        """DDIM inversion x_0 -> x_{t_enc} (reference :233-279).  Each step is eps (graph-replayed apply_model, batched
        CFG like p_sample_ddim -- the reference's own CFG branch concatenates the cond dicts and cannot run with a
        ControlLDM) followed by ONE update kernel; the two per-step coefficients are evaluated on the host in fp32 with
        the reference's operation order, so scale-1 results are bit-identical given the same eps."""
        steps = np.arange(self.ddpm_num_timesteps) if use_original_steps else self.ddim_timesteps
        assert t_enc <= steps.shape[0]
        if use_original_steps:
            a_next_tab, a_tab = self.alphas_cumprod[:t_enc].cpu(), self.alphas_cumprod_prev[:t_enc].cpu()
        else:
            a_next_tab = torch.as_tensor(self.ddim_alphas[:t_enc], dtype=torch.float32).cpu()
            a_tab = torch.tensor(self.ddim_alphas_prev[:t_enc])  # numpy float64 holding fp32 values, like the reference:
            # the per-step coefficients below are then evaluated in float64 and rounded to fp32 once, as torch does when a
            # 0-dim float64 tensor multiplies an fp32 tensor
        use_cfg = not (unconditional_guidance_scale == 1. or unconditional_conditioning is None)
        x_next, kept, kept_steps = x0, [], []
        ts_all = self._step_tensors(steps[:t_enc], x0.shape[0], x0.device)
        every = (t_enc // return_intermediates) if return_intermediates else 0
        for i in range(t_enc):
            e_c, e_u = self._eps_pair(x_next, ts_all[i], c, unconditional_conditioning, use_cfg)
            an, a = a_next_tab[i], a_tab[i]
            c1 = (an / a).sqrt()
            c2 = an.sqrt() * ((1 / an - 1).sqrt() - (1 / a - 1).sqrt())
            x_next = ops.ddim_encode_update(x_next, e_c, e_u, unconditional_guidance_scale, float(c1), float(c2))
            if return_intermediates and ((i % every == 0 and i < t_enc - 1) or i >= t_enc - 2):
                kept.append(x_next)
                kept_steps.append(i)
            if callback:
                callback(i)
        out = {'x_encoded': x_next, 'intermediate_steps': kept_steps}
        if return_intermediates:
            out['intermediates'] = kept
        return x_next, out
