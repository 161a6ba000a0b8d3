"""Import the UNMODIFIED reference (/root/reference) in this container by injecting small stand-ins for the
third-party packages that are not installed (omegaconf, pytorch_lightning, open_clip) and for the CLIP text encoder
(needs the HF hub).  Used only by tools/make_golden.py to generate tests/golden/*; never by the product or the
GPU-side tests (the reference tree does not exist on the GPU box).
"""
import os
import sys
import types

import torch
import torch.nn as nn
import yaml

REFERENCE_ROOT = os.environ.get("CTRLORA_REFERENCE", "/root/reference")


class _AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    __setattr__ = dict.__setitem__


class ListConfig(list):
    pass


def _wrap(o):
    if isinstance(o, dict):
        return _AttrDict({k: _wrap(v) for k, v in o.items()})
    if isinstance(o, list):
        return ListConfig(_wrap(v) for v in o)
    return o


def install():
    if "omegaconf" not in sys.modules:
        m = types.ModuleType("omegaconf")

        class OmegaConf:
            @staticmethod
            def load(path):
                with open(path) as f:
                    return _wrap(yaml.safe_load(f))

            @staticmethod
            def create(obj):
                return _wrap(obj)

        m.OmegaConf, m.ListConfig = OmegaConf, ListConfig
        m.__path__ = []
        lc = types.ModuleType("omegaconf.listconfig")
        lc.ListConfig = ListConfig
        m.listconfig = lc
        sys.modules["omegaconf"] = m
        sys.modules["omegaconf.listconfig"] = lc
    if "pytorch_lightning" not in sys.modules:
        pl = types.ModuleType("pytorch_lightning")

        class LightningModule(nn.Module):
            @property
            def device(self):
                try:
                    return next(self.parameters()).device
                except StopIteration:
                    return torch.device("cpu")

            def log(self, *a, **k):
                pass

            def log_dict(self, *a, **k):
                pass

        pl.LightningModule = LightningModule
        util = types.ModuleType("pytorch_lightning.utilities")
        dist = types.ModuleType("pytorch_lightning.utilities.distributed")
        dist.rank_zero_only = lambda f: f
        util.distributed = dist
        cb = types.ModuleType("pytorch_lightning.callbacks")

        class Callback:
            pass

        cb.Callback = Callback
        pl.utilities, pl.callbacks = util, cb
        sys.modules.update({"pytorch_lightning": pl, "pytorch_lightning.utilities": util,
                            "pytorch_lightning.utilities.distributed": dist, "pytorch_lightning.callbacks": cb})
    if "open_clip" not in sys.modules:
        sys.modules["open_clip"] = types.ModuleType("open_clip")
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    # CLIP text encoder stub (context is synthetic everywhere in this repo)
    import ldm.modules.encoders.modules as enc

    class _NoClip(nn.Module):
        def __init__(self, *a, **k):
            super().__init__()

        def forward(self, text):
            raise RuntimeError("CLIP is stubbed: pass the [B,77,768] context directly")

        encode = forward

    enc.FrozenCLIPEmbedder = _NoClip


def reference_module(name):
    install()
    import importlib
    return importlib.import_module(name)


def install_openpose_shims():
    """Import-only stand-ins for matplotlib and skimage, which the reference's annotator.openpose imports but whose body
    path (Body, OpenposeDetector without hands and faces) never calls; touching them raises"""
    def stub(name):
        m = types.ModuleType(name)
        m.__path__ = []

        def missing(attr):
            if attr.startswith("__"):
                raise AttributeError(attr)
            raise RuntimeError(f"{name}.{attr} is an import-only stand-in: the body path must not use it")
        m.__getattr__ = missing
        return m
    for name in ("matplotlib", "matplotlib.pyplot", "skimage", "skimage.measure"):
        sys.modules.setdefault(name, stub(name))
    sys.modules["matplotlib"].__dict__["pyplot"] = sys.modules["matplotlib.pyplot"]
    sys.modules["skimage"].__dict__["measure"] = sys.modules["skimage.measure"]
    sys.modules["skimage.measure"].__dict__["label"] = None
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
