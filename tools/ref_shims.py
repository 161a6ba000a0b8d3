"""Import the UNMODIFIED reference (/root/reference) in this container by injecting small stand-ins for the
third-party packages that are not installed (omegaconf, pytorch_lightning, open_clip) and for the CLIP text encoder
(needs the HF hub).  Used only by tools/make_golden.py to generate tests/golden/*; never by the product or the
GPU-side tests (the reference tree does not exist on the GPU box).
"""
import contextlib
import os
import sys
import tempfile
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


def install_timm_shim():
    """A stand-in for timm, which the reference's annotator.midas imports (midas/vit.py) and which is not installed:
    `timm.create_model("vit_large_patch16_384")` returns a VisionTransformer with timm's module names and forward
    (patch_embed.proj, cls_token, pos_embed, pos_drop, blocks[i].{norm1, attn.qkv, attn.proj, norm2, mlp.fc1, mlp.fc2},
    norm, head; pre-norm blocks, LayerNorm eps 1e-6, exact GELU, softmax attention scaled by d_head^-1/2).  The weights
    are left at torch's default init: the caller loads its own."""
    if "timm" in sys.modules:
        return

    class PatchEmbed(nn.Module):
        def __init__(self, dim, patch):
            super().__init__()
            self.proj = nn.Conv2d(3, dim, kernel_size=patch, stride=patch)

        def forward(self, x):
            return self.proj(x).flatten(2).transpose(1, 2)

    class Attention(nn.Module):
        def __init__(self, dim, heads):
            super().__init__()
            self.num_heads, self.scale = heads, (dim // heads) ** -0.5
            self.qkv = nn.Linear(dim, dim * 3)
            self.attn_drop = nn.Dropout(0.0)
            self.proj = nn.Linear(dim, dim)
            self.proj_drop = nn.Dropout(0.0)

        def forward(self, x):
            b, n, c = x.shape
            qkv = self.qkv(x).reshape(b, n, 3, self.num_heads, c // self.num_heads).permute(2, 0, 3, 1, 4)
            q, k, v = qkv[0], qkv[1], qkv[2]
            attn = (q @ k.transpose(-2, -1)) * self.scale
            attn = self.attn_drop(attn.softmax(dim=-1))
            x = (attn @ v).transpose(1, 2).reshape(b, n, c)
            return self.proj_drop(self.proj(x))

    class Mlp(nn.Module):
        def __init__(self, dim, hidden):
            super().__init__()
            self.fc1, self.act, self.fc2 = nn.Linear(dim, hidden), nn.GELU(), nn.Linear(hidden, dim)
            self.drop = nn.Dropout(0.0)

        def forward(self, x):
            return self.drop(self.fc2(self.drop(self.act(self.fc1(x)))))

    class Block(nn.Module):
        def __init__(self, dim, heads, mlp_ratio):
            super().__init__()
            self.norm1 = nn.LayerNorm(dim, eps=1e-6)
            self.attn = Attention(dim, heads)
            self.norm2 = nn.LayerNorm(dim, eps=1e-6)
            self.mlp = Mlp(dim, int(dim * mlp_ratio))

        def forward(self, x):
            x = x + self.attn(self.norm1(x))
            return x + self.mlp(self.norm2(x))

    class VisionTransformer(nn.Module):
        def __init__(self, img_size=384, patch_size=16, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4.0,
                     num_classes=1000):
            super().__init__()
            self.patch_embed = PatchEmbed(embed_dim, patch_size)
            self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
            self.pos_embed = nn.Parameter(torch.zeros(1, (img_size // patch_size) ** 2 + 1, embed_dim))
            self.pos_drop = nn.Dropout(0.0)
            self.blocks = nn.Sequential(*[Block(embed_dim, num_heads, mlp_ratio) for _ in range(depth)])
            self.norm = nn.LayerNorm(embed_dim, eps=1e-6)
            self.head = nn.Linear(embed_dim, num_classes)

        def forward_features(self, x):
            x = self.patch_embed(x)
            x = torch.cat((self.cls_token.expand(x.shape[0], -1, -1), x), dim=1)
            x = self.pos_drop(x + self.pos_embed)
            return self.norm(self.blocks(x))

        def forward(self, x):
            return self.head(self.forward_features(x)[:, 0])

    configs = {"vit_large_patch16_384": dict(img_size=384, patch_size=16, embed_dim=1024, depth=24, num_heads=16)}

    def create_model(name, pretrained=False, **kwargs):
        if pretrained:
            raise RuntimeError("the timm stand-in has no pretrained weights")
        if name not in configs:
            raise NotImplementedError(f"the timm stand-in builds {sorted(configs)} only, not {name!r}")
        return VisionTransformer(**configs[name], **kwargs)

    m = types.ModuleType("timm")
    m.create_model, m.VisionTransformer = create_model, VisionTransformer
    sys.modules["timm"] = m


def install_uniformer_shims():
    """Stand-ins for what the reference's annotator.uniformer (its vendored mmcv and mmseg) imports and is not
    installed: addict.Dict (mmcv.Config's attribute dict), yapf's FormatCode (Config.pretty_text only), prettytable
    (mmseg's evaluation tables, never printed here), timm.models.layers' DropPath, to_2tuple and trunc_normal_ (the
    UniFormer backbone; DropPath is the identity in eval mode) and an import-only matplotlib"""
    install_openpose_shims()
    if "addict" not in sys.modules:
        m = types.ModuleType("addict")

        class Dict(dict):
            """addict.Dict's behaviour as mmcv.Config uses it: attribute access, nested dicts converted on
            construction, a missing key raises (mmcv's ConfigDict overrides __missing__ to raise as well)"""

            def __init__(self, *args, **kwargs):
                super().__init__()
                for arg in args:
                    if isinstance(arg, dict):
                        for k, v in arg.items():
                            self[k] = self._hook(v)
                    elif isinstance(arg, tuple) and not isinstance(arg[0], tuple):
                        self[arg[0]] = self._hook(arg[1])
                    elif arg is not None:
                        for k, v in iter(arg):
                            self[k] = self._hook(v)
                for k, v in kwargs.items():
                    self[k] = self._hook(v)

            @classmethod
            def _hook(cls, item):
                if isinstance(item, dict):
                    return cls(item)
                if isinstance(item, (list, tuple)):
                    return type(item)(cls._hook(e) for e in item)
                return item

            def __getattr__(self, k):
                return self.__getitem__(k)

            def __setattr__(self, k, v):
                self[k] = v

            def __missing__(self, k):
                raise KeyError(k)

            def to_dict(self):
                return {k: v.to_dict() if isinstance(v, Dict) else v for k, v in self.items()}

            def __deepcopy__(self, memo):
                import copy
                other = self.__class__()
                memo[id(self)] = other
                for k, v in self.items():
                    other[copy.deepcopy(k, memo)] = copy.deepcopy(v, memo)
                return other

        m.Dict = Dict
        sys.modules["addict"] = m
    if "yapf" not in sys.modules:
        names = ("yapf", "yapf.yapflib", "yapf.yapflib.yapf_api")
        mods = {n: types.ModuleType(n) for n in names}
        for n in names[:2]:
            mods[n].__path__ = []
        mods["yapf.yapflib.yapf_api"].FormatCode = lambda text, **k: (text, False)
        sys.modules.update(mods)
    if "prettytable" not in sys.modules:
        m = types.ModuleType("prettytable")

        class PrettyTable:
            def __init__(self, *a, **k):
                raise RuntimeError("prettytable is an import-only stand-in")

        m.PrettyTable = PrettyTable
        sys.modules["prettytable"] = m
    if "timm.models.layers" not in sys.modules:
        timm = sys.modules.get("timm") or types.ModuleType("timm")
        timm.__path__ = []
        models = types.ModuleType("timm.models")
        models.__path__ = []
        layers = types.ModuleType("timm.models.layers")

        class DropPath(nn.Module):
            def __init__(self, drop_prob=0.0):
                super().__init__()
                self.drop_prob = drop_prob

            def forward(self, x):
                if self.drop_prob == 0.0 or not self.training:
                    return x
                keep = 1 - self.drop_prob
                mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
                return x * mask / keep

        layers.DropPath = DropPath
        layers.to_2tuple = lambda x: tuple(x) if isinstance(x, (list, tuple)) else (x, x)
        layers.trunc_normal_ = lambda t, mean=0.0, std=1.0, a=-2.0, b=2.0: nn.init.trunc_normal_(t, mean, std, a, b)
        timm.models, models.layers = models, layers
        sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers})


@contextlib.contextmanager
def mlsd_on_cpu(state_dict):
    """The unmodified reference annotator.mlsd, importable and runnable on the CPU for the duration of the block: yields
    the module.  Tensor.cuda and Module.cuda are no-ops inside (its MLSDdetector and pred_lines call them), and its
    annotator_ckpts_path points at a temporary directory holding `state_dict` as mlsd_large_512_fp32.pth, so the
    detector loads it instead of downloading."""
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import importlib
    mod = importlib.import_module("annotator.mlsd")
    saved = (torch.Tensor.cuda, nn.Module.cuda, mod.annotator_ckpts_path)
    with tempfile.TemporaryDirectory() as d:
        torch.save(state_dict, os.path.join(d, "mlsd_large_512_fp32.pth"))
        torch.Tensor.cuda = lambda self, *a, **k: self
        nn.Module.cuda = lambda self, *a, **k: self
        mod.annotator_ckpts_path = d
        try:
            yield mod
        finally:
            torch.Tensor.cuda, nn.Module.cuda, mod.annotator_ckpts_path = saved
