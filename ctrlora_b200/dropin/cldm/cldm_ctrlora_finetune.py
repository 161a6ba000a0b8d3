"""Drop-in for the reference's `cldm/cldm_ctrlora_finetune.py`: the LoRA-finetune ControlNet (every nn.Linear of the
ControlNet becomes a LoRACompatibleLinear with a fresh LoRALinearLayer; the image-space hint block is deleted) and
its LatentDiffusion wrapper."""
import os

import torch

from cldm.cldm import ControlLDM, ControlNet
from cldm.ddim_hacked import DDIMSampler
from cldm.lora import LoRALinearLayer
from cldm._inject import plain_linears, set_child, to_lora_linear


class ControlNetFinetune(ControlNet):
    def __init__(self, ft_with_lora=True, lora_rank=128, norm_trainable=True, zero_trainable=True, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.ft_with_lora = ft_with_lora
        self.lora_rank = lora_rank
        self.norm_trainable = norm_trainable
        self.zero_trainable = zero_trainable
        del self.input_hint_block
        if ft_with_lora:
            for name, m in plain_linears(self):
                set_child(self, name, to_lora_linear(m, LoRALinearLayer(m.in_features, m.out_features, rank=lora_rank)))

    def forward(self, hint, timesteps, context, **kwargs):
        return self.forward_latent_hint(hint, timesteps, context)


def trainable_parameters(control_model, log_path=None):
    """The optimizer's parameter set, reference configure_optimizers :88-104: name-substring filter in its if/elif
    order; also written to ./tmp/*.txt like the reference when `log_path` is given."""
    picked = []
    for n, p in control_model.named_parameters():
        assert 'input_hint' not in n
        if getattr(control_model, "ft_with_lora", True):
            if 'lora_layer' in n:
                picked.append((n, p))
            elif ('zero_convs' in n or 'middle_block_out' in n) and control_model.zero_trainable:
                picked.append((n, p))
            elif 'norm' in n and control_model.norm_trainable:
                picked.append((n, p))
        else:
            assert 'lora_layer' not in n
            picked.append((n, p))
    if log_path:
        os.makedirs(os.path.dirname(log_path) or ".", exist_ok=True)
        with open(log_path, 'w') as f:
            f.write('\n'.join(n for n, _ in picked) + '\n')
    return picked


class ControlFinetuneLDM(ControlLDM):
    @torch.no_grad()
    def sample_log(self, cond, batch_size, ddim, ddim_steps, **kwargs):
        sampler = DDIMSampler(self)
        b, c, h, w = cond["c_concat"][0].shape
        shape = (self.channels, h // 8, w // 8) if c != self.channels else (self.channels, h, w)
        return sampler.sample(ddim_steps, batch_size, shape, cond, verbose=False, **kwargs)

    def apply_model(self, x_noisy, t, cond, *args, **kwargs):
        assert isinstance(cond, dict)
        diffusion_model = self.model.diffusion_model
        cond_txt = cond['c_crossattn'][0] if len(cond['c_crossattn']) == 1 else torch.cat(cond['c_crossattn'], 1)
        if cond['c_concat'] is None:
            return diffusion_model(x=x_noisy, timesteps=t, context=cond_txt, control=None,
                                   only_mid_control=self.only_mid_control)
        hint = self.hint_latent(cond['c_concat'])
        return self.control_and_unet(x_noisy, hint, t, cond_txt, self.scaled_control)

    def configure_optimizers(self):
        picked = trainable_parameters(self.control_model, './tmp/finetune_trainable_params.txt')
        params = [p for _, p in picked]
        print(f'Optimizable params: {sum(p.numel() for p in params) / 1e6:.1f}M')
        return torch.optim.AdamW(params, lr=self.learning_rate)
