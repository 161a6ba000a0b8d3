"""Drop-in for the reference's `ldm/models/diffusion/plms.py`: `PLMSSampler` with the same constructor, `make_schedule`,
`sample()` / `plms_sampling()` arguments and `(samples, intermediates)` result.  It runs what the reference runs
(eta 0 only): step 0 is the pseudo improved Euler step, with a second model evaluation at `t_next` on a provisional
DDIM update, and later steps use the 2-, 3- and 4-term Adams-Bashforth combinations of the guided eps history, so S
steps cost S + 1 model evaluations.  Differences:
  * conditioning is anything `apply_model` accepts, with or without classifier-free guidance: the finetune /
    pretrain dict, the inference model's list of dicts, the style model's `c_ip`.  The reference cannot run on these
    (its `.shape` check, :84-91, and `torch.cat` over the cond dicts, :188-190, fail on ControlLDM conditioning);
  * the eps pair (batched CFG, CUDA-graph replay, weight-fingerprint re-capture, context cache for the run) is
    `DDIMSampler`'s, through a private `DDIMSampler` on the same model.  Step 0's two evaluations replay the same
    apply_model graph; the updates between them run outside it;
  * step 0's provisional update is `ctrlora_ddim_update`; every final update (CFG combine, e' of the step's order,
    pred_x0, x_prev; ~15 elementwise torch ops in the reference) is ONE kernel, `ctrlora_plms_update`, whose scalars
    come from ctrlora_b200.plms_schedule;
  * buffers follow `model.device` (the reference hard-codes 'cuda', :19-23).
"""
import torch
from tqdm import tqdm

from cldm.ddim_hacked import DDIMSampler
from ctrlora_b200 import ops, plms_schedule


class PLMSSampler(object):
    def __init__(self, model, schedule="linear", batched_cfg=True, use_cuda_graph=True, **kwargs):
        super().__init__()
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.eps_model = DDIMSampler(model, batched_cfg=batched_cfg, use_cuda_graph=use_cuda_graph)

    def register_buffer(self, name, attr):
        if type(attr) == torch.Tensor and attr.device != self.model.device:
            attr = attr.to(self.model.device)
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        """The reference's tables (:25-55), which are DDIM's: computed by the private DDIMSampler and shared with it."""
        if ddim_eta != 0:
            raise ValueError('ddim_eta must be 0 for PLMS')
        d = self.eps_model
        d.make_schedule(ddim_num_steps, ddim_discretize=ddim_discretize, ddim_eta=ddim_eta, verbose=verbose)
        for name in ("ddim_timesteps", "betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod",
                     "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod",
                     "sqrt_recipm1_alphas_cumprod", "ddim_sigmas", "ddim_alphas", "ddim_alphas_prev",
                     "ddim_sqrt_one_minus_alphas", "ddim_sigmas_for_original_num_steps"):
            setattr(self, name, getattr(d, name))

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None, img_callback=None,
               quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None,
               corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, dynamic_threshold=None, **kwargs):
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
            print(f'Data shape for PLMS sampling is {size}')
        return self.plms_sampling(conditioning, size, callback=callback, img_callback=img_callback,
                                  quantize_denoised=quantize_x0, mask=mask, x0=x0, ddim_use_original_steps=False,
                                  noise_dropout=noise_dropout, temperature=temperature, score_corrector=score_corrector,
                                  corrector_kwargs=corrector_kwargs, x_T=x_T, log_every_t=log_every_t,
                                  unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning,
                                  dynamic_threshold=dynamic_threshold, verbose=verbose)

    @torch.no_grad()
    def plms_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, callback=None, timesteps=None,
                      quantize_denoised=False, mask=None, x0=None, img_callback=None, log_every_t=100, temperature=1.,
                      noise_dropout=0., score_corrector=None, corrector_kwargs=None, unconditional_guidance_scale=1.,
                      unconditional_conditioning=None, dynamic_threshold=None, verbose=True):
        if score_corrector is not None or quantize_denoised or dynamic_threshold is not None or noise_dropout > 0.:
            raise NotImplementedError("score_corrector / quantize_denoised / dynamic_threshold / noise_dropout are not "
                                      "on the CtrLoRA path")
        if self.model.parameterization == "v":
            raise NotImplementedError("v-parameterisation is not on the CtrLoRA path")
        if ddim_use_original_steps:
            # the reference reads model.ddim_sigmas_for_original_num_steps there (:203), which no model defines
            raise NotImplementedError("ddim_use_original_steps is not on the CtrLoRA path")
        device = self.model.betas.device
        if device.type != "cuda":
            raise RuntimeError("ctrlora_b200: PLMSSampler needs the model on a CUDA device (no CPU path)")
        b = shape[0]
        img = torch.randn(shape, device=device) if x_T is None else x_T
        if timesteps is None:
            timesteps = self.ddim_timesteps
        else:
            subset_end = int(min(timesteps / self.ddim_timesteps.shape[0], 1) * self.ddim_timesteps.shape[0]) - 1
            timesteps = self.ddim_timesteps[:subset_end]
        intermediates = {'x_inter': [img], 'pred_x0': [img]}
        steps = plms_schedule.time_range(timesteps)
        total_steps = len(steps)
        plan = plms_schedule.plan(steps, self.ddim_alphas, self.ddim_alphas_prev, self.ddim_sqrt_one_minus_alphas,
                                  self.ddim_sigmas)
        if verbose:
            print(f"Running PLMS Sampling with {total_steps} timesteps")
        d = self.eps_model
        ts_all = d._step_tensors([st.t for st in plan] + [st.t_next for st in plan[:1]], b, device)
        use_cfg = not (unconditional_conditioning is None or unconditional_guidance_scale == 1.)
        scale = unconditional_guidance_scale
        # the reference draws noise_like in every update and multiplies it by sigma_t (= 0 here, :220); drawing none
        # changes the global RNG position after sampling and, with mask / x0, q_sample's noise from step 1 on
        hist = [torch.empty(shape, device=device, dtype=torch.float32) for _ in range(4)]  # e_t of the last 4 steps
        f32 = lambda e: None if e is None else e.float().contiguous()
        with d._run_mode(d):
            for i, st in enumerate(tqdm(plan, desc='PLMS Sampler', total=total_steps, disable=not verbose)):
                ts = ts_all[i]
                if mask is not None:
                    assert x0 is not None
                    img_orig = self.model.q_sample(x0, ts)
                    img = img_orig * mask + (1. - mask) * img
                x = img.float().contiguous()
                e_c, e_u = d._eps_pair(x, ts, cond, unconditional_conditioning, use_cfg)
                kw = {}
                if i == 0:
                    # pseudo improved Euler (:227-231): eps at t_next on DDIM's x_prev; the pair is copied out of the
                    # graph's output buffer, which the second evaluation overwrites.  ctrlora_ddim_update takes its
                    # square roots with sqrtf (correctly rounded), the final update torch CPU's: they can differ by an ulp
                    # (DESIGN §7)
                    e_c, e_u = e_c.float().clone(), None if e_u is None else e_u.float().clone()
                    x_prov, _ = ops.ddim_update(x, e_c, e_u, scale, st.a_t, st.a_prev, st.sigma_t,
                                                st.sqrt_one_minus_at)
                    en_c, en_u = d._eps_pair(x_prov, ts_all[total_steps], cond, unconditional_conditioning, use_cfg)
                    kw["e_next"] = (f32(en_c), f32(en_u))
                else:
                    kw["old"] = [hist[(i - k) % 4] for k in range(1, min(i, 3) + 1)]
                img, pred_x0 = ops.plms_update(x, f32(e_c), f32(e_u), hist[i % 4], scale, **st.kernel_args(), **kw)
                if callback:
                    callback(i)
                if img_callback:
                    img_callback(pred_x0, i)
                if st.index % log_every_t == 0 or st.index == total_steps - 1:
                    intermediates['x_inter'].append(img)
                    intermediates['pred_x0'].append(pred_x0)
        return img, intermediates
