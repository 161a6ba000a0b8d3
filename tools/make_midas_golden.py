"""Generate tests/golden/midas_golden.pt: what the reference's MiDaS annotator computes, in fp32 on the CPU.

    python tools/make_midas_golden.py

The unmodified reference `annotator.midas` is imported from the reference tree with tools/ref_shims.py's timm stand-in.
`MidasDetector.__call__` runs as written, with two substitutions made inside this tool only: `api.load_model` returns a
`DPTDepthModel(path=None, backbone="vitl16_384", non_negative=True)` loaded (strict) with tests/midas_golden.py's
synthetic weights instead of reading dpt_large_384.pt, and `.cuda()` of modules and tensors is a no-op, so the fixture is
torch's fp32 CPU result.  Per size the fixture stores the raw depth, the uint8 depth and normal maps (each in row bands)
and the input checksum, as entries "<size>.depth" etc.; at midas_golden.STAGE_SIZE (entries "stage.*") also every block-level intermediate, fp32 without the batch dim
("stage.stages"): the four hooked ViT streams, the
reassembled layer_1..4, layer1_rn..layer4_rn, refinenet4..1, the head's 32-channel activation and the depth.  And the
state-dict keys and shapes.  Running it twice writes identical bytes.
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
import midas_golden as mg  # noqa: E402


def reference_detector():
    """(MidasDetector, its MiDaSInference) with the fixture's weights, on the CPU"""
    ref_shims.install_timm_shim()
    if ref_shims.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    import annotator.midas as M
    from annotator.midas import api
    from annotator.midas.midas.dpt_depth import DPTDepthModel

    def load_model(model_type):
        assert model_type == "dpt_large"
        return DPTDepthModel(path=None, backbone="vitl16_384", non_negative=True).eval(), None

    api.load_model = load_model
    M.MiDaSInference.__init__.__globals__["load_model"] = load_model
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.Tensor.cuda = lambda self, *a, **k: self
    det = M.MidasDetector()
    inf = det.model
    shapes = {k: tuple(v.shape) for k, v in inf.state_dict().items()}
    inf.load_state_dict(mg.weights(shapes), strict=True)
    return det, inf


def run(det, inf, size, stages=False):
    img = mg.image(size)
    got = {}
    hooks = [inf.register_forward_hook(lambda m, i, o: got.__setitem__("depth", o.detach().clone()))]
    st = {}
    if stages:
        dpt = inf.model
        pre, sc = dpt.pretrained, dpt.scratch
        mods = {f"layer{k}": getattr(pre, f"act_postprocess{k}")[3 if k == 3 else 4] for k in (1, 2, 3, 4)}
        mods.update({f"layer{k}_rn": getattr(sc, f"layer{k}_rn") for k in (1, 2, 3, 4)})
        mods.update({f"refinenet{k}": getattr(sc, f"refinenet{k}") for k in (1, 2, 3, 4)})
        mods["head"] = sc.output_conv[3]
        for i, blk in zip((1, 2, 3, 4), (5, 11, 17, 23)):
            mods[f"hook{i}"] = pre.model.blocks[blk]
        for name, m in mods.items():
            hooks.append(m.register_forward_hook(
                lambda m, i, o, name=name: st.__setitem__(name, o.detach().clone()[0])))
    depth_image, normal_image = det(img)
    for h in hooks:
        h.remove()
    depth = got["depth"][0]
    res = {"input_sum": int(img.astype("int64").sum()), "depth": mg.bands(depth),
           "depth_u8": mg.bands(torch.from_numpy(depth_image)), "normal_u8": mg.bands(torch.from_numpy(normal_image))}
    st["depth"] = depth
    print(f"{size}: depth {tuple(depth.shape)} min {depth.min():.4f} max {depth.max():.4f} mean {depth.mean():.4f} "
          f"positive {(depth > 0).float().mean():.3f}; depth_u8 levels {len(np.unique(depth_image))}, normal_u8 "
          f"x levels {len(np.unique(normal_image[..., 0]))}")
    if stages:
        res["stages"] = st
    return res


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    det, inf = reference_detector()
    g = {"seed": mg.SEED, "keys": [(k, tuple(v.shape)) for k, v in inf.state_dict().items()],
         "torch": torch.__version__, "cv2": cv2.__version__, "numpy": np.__version__}
    with torch.no_grad():
        for size in list(mg.SIZES) + ["stage"]:
            res = run(det, inf, mg.STAGE_SIZE if size == "stage" else size, stages=size == "stage")
            # one entry per map, each a dict of row bands (or of stages): the part splitter moves sub-entries
            for key, val in res.items():
                g[f"{size}.{key}"] = val
    path = os.path.join(ROOT, "tests", "golden", "midas_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
