"""Generate tests/golden/hed_golden.pt: what the reference's HED and HED-sketch annotators compute, in fp32 on the CPU.

    python tools/make_hed_golden.py

The unmodified reference `annotator.hed.ControlNetHED_Apache2` (annotator/hed/__init__.py) is imported from the
reference tree and loaded with the synthetic weights of tests/hed_golden.py.  For each size, HEDdetector.__call__'s
arithmetic (:65-79) is replayed with one substitution: the reference moves the image and the model to the GPU
(`.cuda()`), here they stay on the CPU, so the fixture is torch's fp32 CPU result followed by the reference's own numpy /
cv2 post-process: `torch.from_numpy(input_image.copy()).float()`, 'h w c -> 1 c h w', the five projections as float32,
`cv2.resize(e, (W, H), interpolation=cv2.INTER_LINEAR)`, the float32 `np.mean` over the stack, the float64 sigmoid,
`safe_step` for safe=True, and `(edge * 255.0).clip(0, 255).astype(np.uint8)`.

The fixture stores, per size: the uint8 maps for safe=False and safe=True, the fp32 mean map and the first side map (in
row bands), the other four side maps whole, the five blocks' outputs at tests/hed_golden.py's sample positions, and
input checksums.  For HED-sketch it calls the reference's own HEDSketchDetector.__call__ on an instance made with
__new__ whose `.hed` returns the 200 x 328 uint8 map (or its darkened copy, hed_golden.dark, which makes the retry loop
run) and stores the sketch and numpy's global RNG state afterwards, for each seed of hed_golden.SKETCH_SEEDS.  Running it
twice writes identical bytes.
"""
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import save_golden  # noqa: E402
import hed_golden as hg  # noqa: E402


def reference_modules():
    sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.hed import ControlNetHED_Apache2
    from annotator.hedsketch import HEDSketchDetector
    from annotator.util import safe_step
    model = ControlNetHED_Apache2().float().eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(hg.weights(shapes), strict=True)
    return model, HEDSketchDetector, safe_step


def run(model, safe_step, size):
    img = hg.image(size)
    H, W, _ = img.shape
    stages, peaks = [], [0.0] * 5
    hooks = []
    for i, blk in enumerate([model.block1, model.block2, model.block3, model.block4, model.block5]):
        # the block returns (h, projection): h is the block's output
        hooks.append(blk.projection.register_forward_hook(lambda m, inp, o: stages.append(inp[0].detach().clone())))
        for conv in blk.convs:  # the largest |pre-ReLU activation|, which bounds what the fp16 activations must hold
            hooks.append(conv.register_forward_hook(
                lambda m, inp, o, i=i: peaks.__setitem__(i, max(peaks[i], float(o.abs().max())))))
    with torch.no_grad():
        image_hed = torch.from_numpy(img.copy()).float()          # reference: .cuda()
        image_hed = image_hed.permute(2, 0, 1).unsqueeze(0)       # rearrange 'h w c -> 1 c h w'
        edges = model(image_hed)
        edges = [e.detach().cpu().numpy().astype(np.float32)[0, 0] for e in edges]
    for h in hooks:
        h.remove()
    sides = [torch.from_numpy(e.copy()) for e in edges]
    edges = [cv2.resize(e, (W, H), interpolation=cv2.INTER_LINEAR) for e in edges]
    edges = np.stack(edges, axis=2)
    mean = np.mean(edges, axis=2)
    edge = 1 / (1 + np.exp(-mean.astype(np.float64)))
    u8 = (edge * 255.0).clip(0, 255).astype(np.uint8)
    u8_safe = (safe_step(edge) * 255.0).clip(0, 255).astype(np.uint8)
    res = {"input_sum": int(img.astype("int64").sum()), "u8": torch.from_numpy(u8), "u8_safe": torch.from_numpy(u8_safe),
           "peaks": peaks}
    for i, e in enumerate(sides[1:], 2):
        res[f"e{i}"] = e
    for i, s in enumerate(stages):
        _, c, h, w = s.shape
        res[f"stage{i}"] = hg.sample_stage(s, hg.stage_positions(h, w, c))
    bins = np.bincount((edge.astype(np.float32) * 3.0).astype(np.int32).ravel(), minlength=4) / edge.size
    print(f"{size}: mean map mean {mean.mean():.3f} std {mean.std():.3f}, uint8 levels {int(u8.min())}..{int(u8.max())}, "
          f"safe_step bins 0/1/2/3: " + " / ".join(f"{b:.2%}" for b in bins) +
          f"; max |pre-ReLU activation| per block: " + ", ".join(f"{p:.0f}" for p in peaks) +
          f"; side maps {[tuple(s.shape) for s in sides]}")
    return res, hg.map_bands(torch.from_numpy(mean.copy())), hg.map_bands(sides[0])


def sketch_cases(HEDSketchDetector, edge):
    """the reference's HEDSketchDetector.__call__ on a stub HED that returns `edge` (and its darkened copy)"""
    class StubHED:
        def __init__(self, m):
            self.m = m

        def __call__(self, input_image, safe=False):
            return self.m.copy()

    cases = {}
    for src, m in (("hed", edge), ("dark", hg.dark(edge))):
        det = HEDSketchDetector.__new__(HEDSketchDetector)
        det.hed = StubHED(m)
        for seed in hg.SKETCH_SEEDS[src]:
            np.random.seed(seed)
            out = det(np.zeros((m.shape[0], m.shape[1], 3), np.uint8))
            st = np.random.get_state()
            cases[f"{src}.{seed}"] = {"out": torch.from_numpy(out.copy()),
                                      "state_keys": torch.from_numpy(st[1].astype(np.int64)),
                                      "state_pos": int(st[2]), "state_gauss": (int(st[3]), float(st[4]))}
            print(f"hedsketch {src} seed {seed}: RNG position {st[2]} of 624, pixels < 5: {float((out < 5).mean()):.3%}")
    return cases


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, HEDSketchDetector, safe_step = reference_modules()
    g = {"seed": hg.SEED, "keys": [(k, tuple(v.shape)) for k, v in model.state_dict().items()],
         "torch": torch.__version__, "cv2": cv2.__version__, "numpy": np.__version__}
    for size in hg.SIZES:
        g[size], g[f"{size}.mean"], g[f"{size}.e1"] = run(model, safe_step, size)
    g["sketch"] = sketch_cases(HEDSketchDetector, g["200x328"]["u8"].numpy())
    path = os.path.join(ROOT, "tests", "golden", "hed_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
