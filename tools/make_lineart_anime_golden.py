"""Generate tests/golden/lineart_anime_golden.pt: what the reference's anime line-art annotator computes, in fp32 on the
CPU.

    python tools/make_lineart_anime_golden.py

The unmodified reference `annotator.lineart_anime.UnetGenerator(3, 1, 8, 64, InstanceNorm2d partial)` is imported from
the reference tree and loaded with the synthetic weights of tests/lineart_anime_golden.py.  LineartAnimeDetector.
__call__ (:134-149) is replayed with one substitution: the reference moves the image and the model to the GPU
(`.cuda()`), here they stay on the CPU, so the fixture is torch's fp32 CPU result.  The steps are the same: the cubic
resize to multiples of 256, `torch.from_numpy(img).float() / 127.5 - 1.0`, 'h w c -> 1 c h w', `model(x)[0, 0] *
127.5 + 127.5`, the cubic resize back and `.clip(0, 255).astype(np.uint8)`.  The fixture stores, per network size, the
network output model(x)[0, 0] (in row bands, each small enough for one part file), the uint8 map, every block's output
at tests/lineart_anime_golden.py's sample positions (cloned in the forward hook: the parent's in-place ReLU overwrites
it afterwards), and the input checksum; for the detector size, the uint8 map and the checksum; and the state-dict keys
and shapes.  Running it twice writes identical bytes.
"""
import functools
import os
import sys

import cv2
import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import save_golden  # noqa: E402
import lineart_anime_golden as lg  # noqa: E402


def reference_generator():
    sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.lineart_anime import UnetGenerator, UnetSkipConnectionBlock
    norm_layer = functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)
    model = UnetGenerator(3, 1, lg.NUM_DOWNS, 64, norm_layer=norm_layer, use_dropout=False).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(lg.weights(shapes), strict=True)
    blocks = [m for m in model.modules() if isinstance(m, UnetSkipConnectionBlock)]  # outermost first
    return model, blocks


def detect(model, input_image, stages=None):
    """LineartAnimeDetector.__call__ on the CPU -> (network output [Hn, Wn], uint8 map [H, W])"""
    H, W, C = input_image.shape
    Hn = 256 * int(np.ceil(float(H) / 256.0))
    Wn = 256 * int(np.ceil(float(W) / 256.0))
    img = cv2.resize(input_image, (Wn, Hn), interpolation=cv2.INTER_CUBIC)
    with torch.no_grad():
        image_feed = torch.from_numpy(img).float()       # reference: .cuda()
        image_feed = image_feed / 127.5 - 1.0
        image_feed = image_feed.permute(2, 0, 1).unsqueeze(0)  # rearrange 'h w c -> 1 c h w'
        y = model(image_feed)[0, 0]
        line = y * 127.5 + 127.5
        line = line.cpu().numpy()
        line = cv2.resize(line, (W, H), interpolation=cv2.INTER_CUBIC)
        line = line.clip(0, 255).astype(np.uint8)
    return y.clone(), line


def run(model, blocks, size):
    img = lg.image(size)
    stages = {}

    def hook(i):
        return lambda m, inp, out: stages.__setitem__(i, out.detach().clone())
    hooks = [b.register_forward_hook(hook(i)) for i, b in enumerate(blocks) if i > 0]
    y, u8 = detect(model, img)
    for h in hooks:
        h.remove()
    res = {"input_sum": int(img.astype("int64").sum()), "u8": torch.from_numpy(u8)}
    for i in sorted(stages):
        s = stages[i]
        _, c, h, w = s.shape
        res[f"block{i}"] = lg.sample_stage(s, lg.stage_positions(h, w, c))
    print(f"{size}: net out mean {y.mean():.4f} min {y.min():.4f} max {y.max():.4f}, uint8 levels "
          f"{int(u8.min())}..{int(u8.max())}, blocks {[tuple(stages[i].shape) for i in sorted(stages)]}")
    return res, lg.map_bands(y)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, blocks = reference_generator()
    g = {"seed": lg.SEED, "keys": [(k, tuple(v.shape)) for k, v in model.state_dict().items()],
         "torch": torch.__version__, "cv2": cv2.__version__}
    for size in lg.SIZES:
        g[size], g[f"{size}.map"] = run(model, blocks, size)
    img = lg.image(lg.DETECTOR_SIZE)
    _, u8 = detect(model, img)
    g["detector"] = {"input_sum": int(img.astype("int64").sum()), "u8": torch.from_numpy(u8)}
    print(f"detector {lg.DETECTOR_SIZE}: uint8 levels {int(u8.min())}..{int(u8.max())}")
    path = os.path.join(ROOT, "tests", "golden", "lineart_anime_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
