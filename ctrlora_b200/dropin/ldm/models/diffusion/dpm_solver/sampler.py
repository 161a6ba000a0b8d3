"""Drop-in for the reference's `ldm/models/diffusion/dpm_solver/sampler.py`: `DPMSolverSampler` with the same
constructor, `sample()` signature and `(x, None)` result.  It runs what the reference's `sample()` runs
(:72-85): DPM-Solver++ (data prediction), multistep, order 2, `time_uniform` steps, `lower_order_final`, one model
evaluation per step and none after the final update.  Differences:
  * conditioning is anything `apply_model` accepts, with or without classifier-free guidance: the finetune /
    pretrain dict and the inference model's list of dicts.  The reference cannot run on these (its `.shape` check,
    :51-58, and `torch.cat` over the cond dicts, dpm_solver.py:308-310, fail on ControlLDM conditioning);
  * model times are the reference's fractional fp32 values (t_continuous - 1/N) * 1000, embedded at fp32;
  * the eps pair (batched CFG, CUDA-graph replay, context cache for the run) is `DDIMSampler`'s, through a private
    `DDIMSampler` on the same model;
  * the per-step update (CFG combine, data prediction, order-1 / order-2 step; ~10 elementwise torch ops in the
    reference) is ONE kernel, `ctrlora_dpm_multistep_update`, whose scalars come from ctrlora_b200.dpm_schedule;
  * buffers follow `model.device` (the reference hard-codes 'cuda', :20-24).
`callback`, `img_callback`, `mask` and `x0` are accepted and ignored, as in the reference.
"""
import torch

from cldm.ddim_hacked import DDIMSampler
from ctrlora_b200 import dpm_schedule, ops


class DPMSolverSampler(object):
    def __init__(self, model, batched_cfg=True, use_cuda_graph=True, **kwargs):
        super().__init__()
        self.model = model
        to_torch = lambda x: x.clone().detach().to(torch.float32).to(model.device)
        self.register_buffer('alphas_cumprod', to_torch(model.alphas_cumprod))
        self.eps_model = DDIMSampler(model, batched_cfg=batched_cfg, use_cuda_graph=use_cuda_graph)

    def register_buffer(self, name, attr):
        if type(attr) == torch.Tensor and attr.device != self.model.device:
            attr = attr.to(self.model.device)
        setattr(self, name, attr)

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None, img_callback=None,
               quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None,
               corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, **kwargs):
        if self.model.parameterization == "v":
            raise NotImplementedError("v-parameterisation is not on the CtrLoRA path")
        C, H, W = shape
        size = (batch_size, C, H, W)
        if verbose:
            print(f'Data shape for DPM-Solver sampling is {size}, sampling steps {S}')
        device = self.model.betas.device
        if device.type != "cuda":
            raise RuntimeError("ctrlora_b200: DPMSolverSampler needs the model on a CUDA device (no CPU path)")
        x = torch.randn(size, device=device) if x_T is None else x_T
        x = x.to(device=device, dtype=torch.float32).contiguous()
        plan = dpm_schedule.multistep_plan(self.alphas_cumprod, S)
        # every step's model time as the fp32 [B] vector the reference feeds apply_model, in one host->device copy
        times = torch.tensor([st.model_time for st in plan], dtype=torch.float32)
        times = times[:, None].expand(len(plan), x.shape[0]).contiguous().to(device)
        use_cfg = not (unconditional_guidance_scale == 1. or unconditional_conditioning is None)
        hist = [torch.empty_like(x), torch.empty_like(x)]  # data predictions of this step and the previous one
        sampler = self.eps_model
        with sampler._run_mode(sampler):
            for i, st in enumerate(plan):
                e_c, e_u = sampler._eps_pair(x, times[i], conditioning, unconditional_conditioning, use_cfg)
                x = ops.dpm_multistep_update(x, e_c.float().contiguous(),
                                             None if e_u is None else e_u.float().contiguous(),
                                             hist[(i - 1) % 2] if st.order == 2 else None, hist[i % 2],
                                             unconditional_guidance_scale, **st.kernel_args())
        return x.to(device), None
