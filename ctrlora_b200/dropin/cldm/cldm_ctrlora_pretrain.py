"""Drop-in for the reference's `cldm/cldm_ctrlora_pretrain.py`: base-ControlNet pretraining with one LoRA set per
task in `loras_dict`, re-pointed per mini-batch by `switch_lora(task)`."""
import torch
import torch.nn as nn

from cldm.cldm import ControlLDM, ControlNet
from cldm.ddim_hacked import DDIMSampler
from cldm.lora import LoRACompatibleLinear, LoRALinearLayer
from cldm._inject import plain_linears, set_child, to_lora_linear


class ControlNetPretrain(ControlNet):
    def __init__(self, lora_rank, tasks, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.lora_rank = lora_rank
        self.tasks = list(tasks)
        self.n_tasks = len(self.tasks)
        del self.input_hint_block
        linears = plain_linears(self)
        self.loras_dict = nn.ModuleDict({
            task: nn.ModuleList([LoRALinearLayer(m.in_features, m.out_features, rank=lora_rank) for _, m in linears])
            for task in self.tasks})
        for name, m in linears:
            set_child(self, name, to_lora_linear(m))
        self._lora_linears = None

    def forward(self, hint, timesteps, context, **kwargs):
        return self.forward_latent_hint(hint, timesteps, context)

    def lora_linears(self):
        """LoRACompatibleLinear modules in named_modules() order: index i pairs with loras_dict[task][i]."""
        if self._lora_linears is None:
            self.__dict__["_lora_linears"] = [m for _, m in self.named_modules() if isinstance(m, LoRACompatibleLinear)]
        return self._lora_linears

    def switch_lora(self, task: str):
        assert task in self.tasks
        for m, lora in zip(self.lora_linears(), self.loras_dict[task]):
            m.set_lora_layer(lora)


class ControlPretrainLDM(ControlLDM):
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
        self.control_model.switch_lora(cond['task'])
        hint = self.hint_latent(cond['c_concat'])
        return self.control_and_unet(x_noisy, hint, t, cond_txt, self.scaled_control)

    def configure_optimizers(self):
        params = list(self.control_model.parameters())
        print(f'Optimizable params: {sum(p.numel() for p in params) / 1e6:.1f}M')
        return torch.optim.AdamW(params, lr=self.learning_rate)
