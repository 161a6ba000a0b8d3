"""Drop-in for the reference's `cldm/model.py`: `create_model(config_path)` and `load_state_dict(path)`.
OmegaConf is optional (PyYAML is enough for these configs)."""
import os

import torch
import yaml

from ldm.util import instantiate_from_config


def get_state_dict(d):
    return d.get('state_dict', d)


def load_state_dict(ckpt_path, location='cpu'):
    _, extension = os.path.splitext(ckpt_path)
    if extension.lower() == ".safetensors":
        import safetensors.torch
        state_dict = safetensors.torch.load_file(ckpt_path, device=location)
    else:
        state_dict = get_state_dict(torch.load(ckpt_path, map_location=torch.device(location)))
    state_dict = get_state_dict(state_dict)
    print(f'Loaded state_dict from [{ckpt_path}]')
    return state_dict


def load_config(config_path):
    try:
        from omegaconf import OmegaConf
        return OmegaConf.load(config_path)
    except ImportError:
        with open(config_path) as f:
            return yaml.safe_load(f)


class skip_param_init:
    """Context manager: construct modules without running their (slow, CPU) default initialisers — for models whose
    weights are about to be overwritten by a checkpoint or a synthetic state dict.  Zero-initialised modules
    (zero_module) and LoRA inits still run."""
    _names = ("kaiming_uniform_", "uniform_", "normal_", "trunc_normal_")

    def __enter__(self):
        self._saved = {n: getattr(torch.nn.init, n) for n in self._names}
        for n in self._names:
            setattr(torch.nn.init, n, lambda t, *a, **k: t)
        return self

    def __exit__(self, *exc):
        for n, f in self._saved.items():
            setattr(torch.nn.init, n, f)


TEXT_ENCODER_TARGET = "ctrlora_b200.text_encoder.FrozenCLIPEmbedder"


def create_model(config_path, init_weights=True, text_encoder=False):
    """Build the model of `config_path` on the CPU.  text_encoder=True builds this package's CLIP text encoder
    (ctrlora_b200.text_encoder.FrozenCLIPEmbedder) as `cond_stage_model`, from the config's cond_stage_config params;
    a dict also overrides those params (e.g. {"version": local_dir, "layer": "hidden", "layer_idx": -2}).  Without it
    cond_stage_model is whatever the config's target resolves to (None when it is not importable)."""
    config = load_config(config_path)
    model_cfg = config["model"] if isinstance(config, dict) else config.model
    if text_encoder:
        cond = model_cfg["params"].get("cond_stage_config")
        params = dict(cond.get("params") or {}) if cond is not None and not isinstance(cond, str) else {}
        if isinstance(text_encoder, dict):
            params.update(text_encoder)
        model_cfg["params"]["cond_stage_config"] = {"target": TEXT_ENCODER_TARGET, "params": params}
    if init_weights:
        model = instantiate_from_config(model_cfg).cpu()
    else:
        with skip_param_init():
            model = instantiate_from_config(model_cfg).cpu()
    if text_encoder and getattr(model, "cond_stage_model", None) is None:
        raise RuntimeError(f"{config_path}: the text encoder ({TEXT_ENCODER_TARGET}) could not be built")
    print(f'Loaded model config from [{config_path}]')
    return model
