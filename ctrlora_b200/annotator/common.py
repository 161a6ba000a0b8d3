"""What every annotator shares: the checkpoint lookup, the frozen-network setup and device check, a bounded cache of
size-keyed tables, the 3x3 tap list, the sub-pixel split of a stride-2 ConvTranspose2d and cv2's linear resize rule."""
import collections
import os

import numpy as np
import torch

from .. import prepare

TAPS3 = [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]


def default_ckpt_dir():
    """the reference's annotator_ckpts_path when its `annotator` package is importable, else None"""
    try:
        from annotator.util import annotator_ckpts_path
    except ImportError:
        return None
    return annotator_ckpts_path


def checkpoint_path(ckpt_dir, name):
    """the path of checkpoint `name` in `ckpt_dir` (None: default_ckpt_dir()).  Nothing is downloaded: a missing
    directory or file raises FileNotFoundError with the path the file was expected at."""
    ckpt_dir = ckpt_dir if ckpt_dir is not None else default_ckpt_dir()
    if ckpt_dir is None:
        raise FileNotFoundError("no checkpoint directory: the reference's annotator package is not importable, so "
                                f"pass ckpt_dir (the directory holding {name})")
    path = os.path.join(ckpt_dir, name)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{name} not found at {path}: ctrlora_b200 never downloads checkpoints; fetch "
                                f"lllyasviel/Annotators' {name} into {ckpt_dir}")
    return path


def freeze(net):
    """The end of a network's __init__: split_k = 0 (passed to every GEMM: 0 lets the tile model choose; 1 pins one plan
    per row, so a batch of B equals B batches of 1 bit for bit), eval mode, no gradients, and the PrepCache of its
    kernel-layout weights (rebuilt whenever a parameter changes, e.g. after load_state_dict)"""
    net.split_k = 0
    net.eval()
    for p in net.parameters():
        p.requires_grad = False
    net.__dict__["_prep"] = prepare.PrepCache()


def device_input(net, x, param):
    """x as contiguous fp32 on `param`'s device, which must be a CUDA device"""
    dev = param.device
    if dev.type != "cuda":
        raise RuntimeError(f"{type(net).__name__} runs on the sm_90a kernels only: move the model to a CUDA device")
    return x.to(dev, torch.float32).contiguous()


class SizeCache(collections.OrderedDict):
    """Tables keyed by an input size: the `capacity` most recently used are kept (the least recently used goes first),
    so a caller that runs many sizes holds a bounded set.  An entry built from `params` is rebuilt once one of them
    changes, by the rule of prepare.PrepCache."""

    def __init__(self, capacity):
        super().__init__()
        self.capacity = capacity
        self._vers = {}

    def fetch(self, key, build, params=()):
        ver = prepare._ver(*params)
        if key not in self or self._vers[key] != ver:
            with torch.no_grad():
                self[key] = build()
            self._vers[key] = ver
            while len(self) > self.capacity:
                del self._vers[self.popitem(last=False)[0]]
        self.move_to_end(key)
        return self[key]


def phase_taps(rows, py, px):
    """[(dy, dx, ky, kx)] of the sub-pixel phase (py, px) of a stride-2 ConvTranspose2d: output row 2m + py reads input
    row m + dy through kernel row ky for each (dy, ky) of rows[py]; the same for columns.  The order of `rows` is the
    order of the phase GEMM's K."""
    return [(dy, dx, ky, kx) for dy, ky in rows[py] for dx, kx in rows[px]]


def phase_weights(convt, rows, split=False):
    """ConvTranspose2d weight [Cin, Cout, k, k] -> per phase 2 py + px: (gather taps [(dy, dx)], fp16 [Cout, 1,
    taps * Cin]) or, with split, (taps, fp16 [Cout, 1, taps * Cin / 2] over the first half of the input channels, fp16
    [Cout, taps * Cin / 2] over the second)"""
    wt = convt.weight.detach().float().permute(1, 2, 3, 0)  # [Cout, ky, kx, Cin]
    cin = wt.shape[-1]
    res = []
    for py in (0, 1):
        for px in (0, 1):
            taps = phase_taps(rows, py, px)
            sel = torch.stack([wt[:, ky, kx] for _, _, ky, kx in taps], 1)  # [Cout, taps, Cin]
            halves = (sel[..., :cin // 2], sel[..., cin // 2:]) if split else (sel,)
            ws = [prepare.linear_weight(h.reshape(h.shape[0], -1).contiguous()) for h in halves]
            if split:
                ws[1] = ws[1].view(ws[1].shape[0], -1)
            res.append(([(dy, dx) for dy, dx, _, _ in taps], *ws))
    return res


def linear_src_coord(src, dst):
    """cv2.resize(INTER_LINEAR)'s source coordinates along one axis of length src -> dst, before any clamping: (int64
    [dst] sx, float32 [dst] fx).  OpenCV's resizeGeneric rule: scale = 1 / (dst / src) in float64,
    f = (float)((i + 0.5) * scale - 0.5), sx = floor(f), fx = f - sx in float32."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(f).astype(np.int64)
    return sx, (f - sx.astype(np.float32)).astype(np.float32)
