"""Generate tests/golden/openpose_golden.pt: what the reference's OpenPose body estimator computes, on the CPU.

    python tools/make_openpose_golden.py

The unmodified reference `annotator.openpose` is imported from the reference tree, with import-only stand-ins for
matplotlib and skimage (tools/ref_shims.py), which its body path never calls.

Network cases: `bodypose_model` loaded with tests/openpose_golden.py's synthetic weights runs in fp32 on the CPU at the
network inputs of four image sizes.  The input is made by the reference's own util.smart_resize_k and
util.padRightDownCorner with the arithmetic of Body.__call__ (body.py:40-43); the reference moves it to the GPU when
one exists, here it stays on the CPU.  Stored: the padded uint8 input, the pad, and the two stride-8 outputs.

Post-process cases: the reference's own Body.__call__ and OpenposeDetector.__call__ on an instance made with __new__
whose network returns tests/openpose_golden.py's planted maps.  body.py's module-level `gaussian_filter` and `sorted`
are wrapped to record what the reference smooths and the scored limb candidates it sorts (i, j, score, ...), without
changing either result.  Stored: candidate, subset, the sorted candidates per limb, the pose dict and the canvas.

Every discrete decision is checked for a margin, which is stored: each peak against its neighbours and the 0.1
threshold (on the reference's smoothed maps), each PAF sample of every candidate pair against 0.05 and each pair score
against 0 (from tests/openpose_golden.py's float64 restatement of body.py:107-131 on the reference's resampled PAFs, which
must pick the recorded candidates and reproduce their scores within 1e-12), the gaps between the scores in each limb's sort order, and each person's mean score
against 0.4.  Running it twice writes identical bytes.
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
import openpose_golden as og  # noqa: E402
from ctrlora_b200.annotator import openpose as op  # noqa: E402  (geometry and limb tables; no device code)

MIN_MARGIN = 2e-5  # 20 x the resampling error of the device tables against cv2 (about 1e-6 on O(1) maps)


def reference_modules():
    ref_shims.install_openpose_shims()
    import annotator.openpose as R
    from annotator.openpose import body as RB, model as RM, util as RU
    return R, RB, RM, RU


def network_case(RM, RU, size):
    model = RM.bodypose_model().float().eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(og.weights(shapes), strict=True)
    img = og.image(size)
    scale = 0.5 * 368 / img.shape[0]                                     # body.py:34 (scale_search [0.5], boxsize 368)
    resized = RU.smart_resize_k(img, fx=scale, fy=scale)
    padded, pad = RU.padRightDownCorner(resized, 8, 128)
    im = np.ascontiguousarray(np.transpose(np.float32(padded[:, :, :, np.newaxis]), (3, 2, 0, 1)) / 256 - 0.5)
    with torch.no_grad():
        paf, heat = model(torch.from_numpy(im).float())                  # reference: .cuda() when available
    print(f"network {size}: input {tuple(im.shape)}, pad {pad}, heatmap std {float(heat.std()):.4f} "
          f"(> 0: {float((heat > 0).float().mean()):.1%}), PAF std {float(paf.std()):.4f}")
    assert float(heat.abs().max()) > 0 and float(heat.std()) > 1e-3, "vacuous heatmaps"
    return {"padded": torch.from_numpy(padded.copy()), "pad": list(pad), "paf": paf.clone(), "heat": heat.clone()}


def peaks(s):
    """body.py:86-95's peak mask of one smoothed map"""
    p = np.pad(s, 1)
    return (s >= p[:-2, 1:-1]) & (s >= p[2:, 1:-1]) & (s >= p[1:-1, :-2]) & (s >= p[1:-1, 2:]) & (s > op.THRE_PEAK)


def peak_margin(smoothed):
    """the smallest distance of any pixel's peak decision from flipping: a peak's smallest (value - neighbour) and
    (value - 0.1); a non-peak's largest failing difference"""
    worst = np.inf
    for s in smoothed:
        pad = np.pad(s, 1)
        diffs = np.stack([s - pad[:-2, 1:-1], s - pad[2:, 1:-1], s - pad[1:-1, :-2], s - pad[1:-1, 2:], s - 0.1])
        peak = (diffs[:4] >= 0).all(axis=0) & (diffs[4] > 0)
        worst = min(worst, float(np.abs(diffs[:, peak]).min(initial=np.inf)))
        failing = np.where(np.concatenate([diffs[:4] < 0, diffs[4:] <= 0]), np.abs(diffs), 0.0).max(axis=0)
        worst = min(worst, float(failing[~peak].min(initial=np.inf)))
    return worst


def postprocess_case(R, RB, RU, case):
    h, w = og.PP_CASES[case]["size"]
    paf8, heat8 = og.planted_maps(case)
    _, _, ph, pw = op.geometry(h, w)

    class StubNet:
        def __call__(self, data):
            assert tuple(data.shape) == (1, 3, ph, pw), data.shape
            return paf8.clone(), heat8.clone()

    smoothed, sorted_lists = [], []
    gf, builtin_sorted = RB.gaussian_filter, sorted

    def recording_gf(m, sigma):
        r = gf(m, sigma=sigma)
        smoothed.append(r.copy())
        return r

    def recording_sorted(lst, key, reverse):
        sorted_lists.append([list(c) for c in lst])
        return builtin_sorted(lst, key=key, reverse=reverse)

    RB.gaussian_filter, RB.sorted = recording_gf, recording_sorted
    try:
        body = RB.Body.__new__(RB.Body)
        body.model = StubNet()
        rgb = og.dummy_image(case)
        candidate, subset = body(rgb[:, :, ::-1].copy())
        smooth_maps, limb_lists = list(smoothed), list(sorted_lists)
        det = R.OpenposeDetector.__new__(R.OpenposeDetector)
        det.body_estimation = body
        pose = det(rgb, return_is_index=True)
        canvas = det(rgb)
    finally:
        RB.gaussian_filter = gf
        del RB.sorted

    # the full-size PAFs as Body computes them (body.py:61-64), for the restated pair scores
    _, pad = RU.padRightDownCorner(np.zeros((op.geometry(h, w)[0], op.geometry(h, w)[1], 3), np.uint8), 8, 128)
    paf = RU.smart_resize_k(np.transpose(np.squeeze(paf8.numpy()), (1, 2, 0)), fx=8, fy=8)
    paf = RU.smart_resize(paf[:ph - pad[2], :pw - pad[3], :], (h, w))
    counts = np.array([int(peaks(s).sum()) for s in smooth_maps])
    assert counts.sum() == (len(candidate) if candidate.ndim == 2 else 0)
    scores = og.pair_scores(paf.astype(np.float64), candidate, counts, h)
    recorded = dict(zip(sorted(scores), limb_lists))
    assert len(recorded) == len(limb_lists) == len(scores)
    sample_margin, score_margin, gap_margin = np.inf, np.inf, np.inf
    limb_cands = {}
    for k, rows in scores.items():
        passed = [[i, j, s] for i, j, s, smp in rows if (smp > op.THRE_PAF).sum() > 0.8 * len(smp) and s > 0]
        got = [c[:3] for c in recorded[k]]
        assert [c[:2] for c in got] == [c[:2] for c in passed], (k, got, passed)
        assert np.allclose([c[2] for c in got], [c[2] for c in passed], rtol=1e-12, atol=0), k
        limb_cands[k] = torch.tensor(got, dtype=torch.float64).reshape(-1, 3)
        for _, _, s, smp in rows:
            sample_margin = min(sample_margin, float(np.abs(smp - op.THRE_PAF).min()))
            if (smp > op.THRE_PAF).sum() > 0.8 * len(smp):
                score_margin = min(score_margin, abs(s))
        ss = sorted(c[2] for c in got)
        if len(ss) > 1:
            gap_margin = min(gap_margin, float(np.diff(ss).min()))
    person_margin = min([abs(p[-2] / p[-1] - 0.4) for p in subset], default=np.inf)
    margins = {"peak": peak_margin(smooth_maps), "paf_sample": sample_margin, "pair_score": score_margin,
               "score_gap": gap_margin, "person_mean": person_margin}
    print(f"post-process {case}: {int(counts.sum())} peaks {counts.tolist()}, {len(subset)} people, margins " +
          ", ".join(f"{k} {v:.3g}" for k, v in margins.items()))
    for k, v in margins.items():
        assert v > MIN_MARGIN, (case, k, v)
    return {"candidate": torch.from_numpy(np.asarray(candidate, np.float64).copy()),
            "subset": torch.from_numpy(subset.copy()), "counts": torch.from_numpy(counts.astype(np.int64)),
            "limb_candidates": limb_cands, "pose": pose, "canvas": torch.from_numpy(canvas.copy()),
            "margins": margins}


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    R, RB, RM, RU = reference_modules()
    keys = [(k, tuple(v.shape)) for k, v in RM.bodypose_model().state_dict().items()]
    g = {"seed": og.SEED, "keys": keys, "torch": torch.__version__, "cv2": cv2.__version__, "numpy": np.__version__}
    for size in og.NET_SIZES:
        g[f"net.{size}"] = network_case(RM, RU, size)
    for case in og.PP_CASES:
        g[f"pp.{case}"] = postprocess_case(R, RB, RU, case)
    path = os.path.join(ROOT, "tests", "golden", "openpose_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
