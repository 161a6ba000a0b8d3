"""Multi-LoRA inference with an IP-Adapter image prompt (reference cldm/cldm_ctrlora_style_inference.py: identical to
cldm_ctrlora_inference.py except apply_model, :156-189): `conds[0]['c_ip']` holds the image-prompt tokens, every
cross-attention of the UNet (cldm.cldm_style.ControlledUnetModel) receives the pair [text, ip]; a condition without
hint (`c_concat == [None]`, guess mode of the style app) runs the UNet without control."""
import torch

from ctrlora_b200 import ops
from cldm.cldm_ctrlora_inference import ControlInferenceLDM as _ControlInferenceLDM
from cldm.cldm_ctrlora_inference import ControlNetInference  # noqa: F401
from ctrlora_b200.runtime import Scaled


class ControlInferenceLDM(_ControlInferenceLDM):
    def apply_model(self, x_noisy, t, conds, *args, **kwargs):
        if isinstance(conds, dict):
            conds = [conds]
        assert isinstance(conds, (list, tuple))
        assert len(conds) == self.control_model.lora_num
        assert len(self.lora_weights) == self.control_model.lora_num
        diffusion_model = self.model.diffusion_model
        cc = conds[0]['c_crossattn']
        cond_txt = cc[0] if len(cc) == 1 else torch.cat(cc, 1)
        c_ip = conds[0].get('c_ip')
        cond_ip = None if c_ip is None else (c_ip[0] if len(c_ip) == 1 else torch.cat(c_ip, 1))
        concat = conds[0].get('c_concat')
        if concat is not None and concat[0] is not None:
            if len(conds) > 1 and getattr(self, "grouped_multi_lora", True):
                hints = [self.hint_latent(cond['c_concat']) for cond in conds]
                stacks = self.control_model.forward_grouped(hints, t, cond_txt)
            else:
                stacks = []
                for i, cond in enumerate(conds):
                    self.control_model.switch_lora(i)
                    stacks.append(self.control_model(hint=self.hint_latent(cond['c_concat']), timesteps=t, context=cond_txt))
            if len(stacks) == 1:
                control = [Scaled(c, s * self.lora_weights[0]) for c, s in zip(stacks[0], self.control_scales)]
            else:
                control = [ops.weighted_sum([st[j] for st in stacks], [s * w for w in self.lora_weights])
                           for j, s in enumerate(self.control_scales)]
        else:
            control = None
        # one [text, ip] pair per transformer depth (reference :184-187)
        context_with_ip = [[txt, cond_ip] for txt in cond_txt] if isinstance(cond_txt, list) else [[cond_txt, cond_ip]]
        return diffusion_model(x=x_noisy, timesteps=t, context=context_with_ip, control=control,
                               only_mid_control=self.only_mid_control)
