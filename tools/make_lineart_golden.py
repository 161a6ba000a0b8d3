"""Generate tests/golden/lineart_golden.pt: what the reference's line-art annotator computes, in fp32 on the CPU.

    python tools/make_lineart_golden.py

The unmodified reference `annotator.lineart.Generator(3, 1, 3)` (annotator/lineart/__init__.py) is imported from the
reference tree and loaded with the synthetic weights of tests/lineart_golden.py.  For each size, LineartDetector.
__call__'s arithmetic (:111-122) is replayed with one substitution: the reference moves the image and the model to the
GPU (`.cuda()`), here they stay on the CPU, so the fixture is torch's fp32 CPU result.  The steps are the same:
`torch.from_numpy(image).float() / 255.0`, 'h w c -> 1 c h w', `model(image)[0][0]`, and
`(line * 255.0).clip(0, 255).astype(np.uint8)`.  The fixture stores the fp32 map (in row bands, each small enough for
one part file), the uint8 map, the outputs of model0 ... model3 at tests/lineart_golden.py's sample positions, the
state-dict keys and shapes, and input checksums.  Running it twice writes identical bytes.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import save_golden  # noqa: E402
import lineart_golden as lg  # noqa: E402


def reference_generator():
    sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.lineart import Generator
    model = Generator(3, 1, lg.N_RESIDUAL).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(lg.weights(shapes), strict=True)
    return model


def run(model, size):
    img = lg.image(size)
    stages = []
    hooks = [getattr(model, f"model{i}").register_forward_hook(lambda m, i, o: stages.append(o.detach().clone()))
             for i in range(4)]
    with torch.no_grad():
        image = torch.from_numpy(img).float()          # reference: .cuda()
        image = image / 255.0
        image = image.permute(2, 0, 1).unsqueeze(0)    # rearrange 'h w c -> 1 c h w'
        line = model(image)[0][0]
        line = line.cpu().numpy()
    for h in hooks:
        h.remove()
    res = {"input_sum": int(img.astype("int64").sum()), "u8": torch.from_numpy(lg.quantise(line))}
    for i, s in enumerate(stages):
        _, c, h, w = s.shape
        res[f"stage{i}"] = lg.sample_stage(s, lg.stage_positions(h, w, c))
    u8 = res["u8"]
    print(f"{size}: map mean {line.mean():.4f} min {line.min():.4f} max {line.max():.4f}, uint8 levels "
          f"{int(u8.min())}..{int(u8.max())}, stages {[tuple(s.shape) for s in stages]}")
    return res, lg.map_bands(torch.from_numpy(line.copy()))


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model = reference_generator()
    g = {"seed": lg.SEED, "keys": [(k, tuple(v.shape)) for k, v in model.state_dict().items()],
         "torch": torch.__version__}
    for size in lg.SIZES:
        g[size], g[f"{size}.map"] = run(model, size)
    path = os.path.join(ROOT, "tests", "golden", "lineart_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
