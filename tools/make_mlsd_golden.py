"""Generate tests/golden/mlsd_golden.pt: what the reference's M-LSD line annotator computes, in fp32 on the CPU.

    python tools/make_mlsd_golden.py

The unmodified reference `annotator.mlsd` is imported from the reference tree; tools/ref_shims.py's mlsd_on_cpu makes
its .cuda() calls no-ops and points its checkpoint directory at tests/mlsd_golden.py's synthetic weights, so
`MLSDdetector()` loads them (strict) and `MLSDdetector.__call__(img, thr_v, thr_d)` runs as written.  Per size the
fixture stores, from hooks on that call: the backbone's c1 .. c5 and the network output at sampled positions, the
decode's 200 candidates (flat index, score, the fp32 segment length and the four displacements, in the layout of
ops.mlsd_decode) and the 201st score, and for every (thr_v, thr_d) of THRESHOLDS the segments pred_lines returned and
the non-zero pixels of the map __call__ returned.  For one size it also stores the full centre and displacement maps.
The sizes the reference turns into zeros store only that.  Also the state-dict keys and shapes.  Running it twice writes
identical bytes.
"""
import os
import sys

import cv2
import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import bands, save_golden  # noqa: E402
import mlsd_golden as mg  # noqa: E402

REL_GAP = 1e-6  # no score or length may lie this close (relative) to a tested threshold: float32 vs float64 compares


def run(mod, det, size):
    img = mg.image(size)
    h, w = img.shape[:2]
    res = {"input_sum": int(img.astype("int64").sum())}
    got = {}
    net = det.model
    hooks = [net.backbone.register_forward_hook(lambda m, i, o: got.__setitem__("features", [t.clone() for t in o])),
             net.register_forward_hook(lambda m, i, o: got.__setitem__("out", o.clone()))]
    utils = sys.modules["annotator.mlsd.utils"]
    real_decode, real_pred = utils.deccode_output_score_and_ptss, mod.pred_lines

    def decode(*a, **k):
        r = real_decode(*a, **k)
        got["decode"] = r
        return r

    def pred(*a, **k):
        r = real_pred(*a, **k)
        got.setdefault("lines", []).append(np.array(r, dtype=np.float64))
        return r

    utils.deccode_output_score_and_ptss, mod.pred_lines = decode, pred
    try:
        maps = []
        for thr_v, thr_d in mg.THRESHOLDS:
            got.pop("lines", None)
            m = det(img, thr_v, thr_d)
            assert m.shape == (h, w) and m.dtype == np.uint8
            maps.append((thr_v, thr_d, m, got.get("lines", [None])[0]))
    finally:
        utils.deccode_output_score_and_ptss, mod.pred_lines = real_decode, real_pred
        for hk in hooks:
            hk.remove()
    if size in mg.ZERO_SIZES:
        assert all(not m.any() for _, _, m, _ in maps), f"{size}: the reference drew lines"
        res["zero"] = True
        print(f"{size}: all-zero maps")
        return res
    out = got["out"]
    for i, f in enumerate(got["features"] + [out]):
        _, c, fh, fw = f.shape
        res[f"stage{i}"] = mg.sample_stage(f, mg.stage_positions(fh, fw, c))
        res[f"stage{i}.shape"] = (c, fh, fw)
    pts, scores, vmap = got["decode"]
    h2, w2 = out.shape[2:]
    start, end = vmap[:, :, :2], vmap[:, :, 2:]
    dist_map = np.sqrt(np.sum((start - end) ** 2, axis=-1))
    ys, xs = pts[:, 0], pts[:, 1]
    val = np.concatenate([scores[:, None], dist_map[ys, xs][:, None], vmap[ys, xs]], axis=1).astype(np.float32)
    res["cand_idx"] = torch.from_numpy((ys * w2 + xs).astype(np.int64))
    res["cand_val"] = torch.from_numpy(np.ascontiguousarray(val))
    # the 201st score, from the reference's decode recomputed with topk(201)
    heat = torch.sigmoid(out[:, 0])
    keep = (F.max_pool2d(heat, 3, stride=1, padding=1) == heat).float()
    top = (heat * keep).reshape(-1).topk(201).values
    assert torch.equal(top[:200], torch.from_numpy(scores)), "recomputed scores differ from the reference's"
    res["score201"] = float(top[200])
    for thr_v, thr_d, m, lines in maps:
        for v, name, thr in ((val[:, 0], "score", thr_v), (val[:, 1], "length", thr_d)):
            near = np.abs(v.astype(np.float64) - thr) <= REL_GAP * thr
            assert not near.any(), f"{size}: a {name} lies within {REL_GAP} of {thr}"
        key = f"thr{thr_v}_{thr_d}"
        res[f"{key}.nonzero"] = torch.from_numpy(np.stack(np.nonzero(m), 1).astype(np.int32))
        res[f"{key}.lines"] = None if lines is None else torch.from_numpy(lines)
    if size == mg.FULL_SIZE:
        res["maps"] = bands(out[0, :5].permute(1, 2, 0).contiguous(), rows=32)
    gap = float(top[199] - top[200])
    print(f"{size}: out {tuple(out.shape)}, scores {scores.min():.3f} .. {scores.max():.3f}, 200th - 201st {gap:.3g}, "
          f"lengths {val[:, 1].min():.3f} .. {val[:, 1].max():.3f}; lines per pair "
          f"{[0 if l is None else len(l) for _, _, _, l in maps]}")
    return res


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    if ref_shims.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.mlsd.models.mbv2_mlsd_large import MobileV2_MLSD_Large
    ref = MobileV2_MLSD_Large()
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    bn = [n for n, m in ref.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    sd = mg.weights(shapes, bn)
    g = {"seed": mg.SEED, "keys": [(k, tuple(v.shape)) for k, v in ref.state_dict().items()],
         "torch": torch.__version__, "cv2": cv2.__version__, "numpy": np.__version__}
    with ref_shims.mlsd_on_cpu(sd) as mod, torch.no_grad():
        det = mod.MLSDdetector()
        for size in mg.SIZES:
            for key, val in run(mod, det, size).items():
                g[f"{size}.{key}"] = val
    path = os.path.join(ROOT, "tests", "golden", "mlsd_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
