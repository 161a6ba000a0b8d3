"""The OpenPose body annotator on an H100: 7x7 implicit GEMMs against fp32 conv2d, the pool-only side-pool launch, the
post-process kernels against cv2 / scipy / numpy, bodypose_model against the reference's fp32 CPU result
(tests/golden/openpose_golden.pt), batching, the device post-process on the reference's planted maps, and the detector
end to end.  Run with -s to print the measured figures."""
import os

import cv2
import numpy as np
import pytest
import scipy.ndimage
import torch
import torch.nn.functional as F

from golden_io import load_golden
import openpose_golden as og
from tolerances import close, norm_rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "openpose_golden.pt")
SCORE_RTOL = 1e-5
# bodypose_model's PAFs and heatmaps against the reference's fp32 network (synthetic weights, four input sizes), norm-
# relative: 26 convs of fp16 activations, 10 of them 7x7.  Measured on an H100 80GB HBM3 at 700 W: at most 1.79e-3
# (the PAFs at 384x640), heatmaps at most 1.16e-3
NET_BOUND = 2.2e-3
# resampled heatmaps and their float64 Gaussian against cv2 + scipy on the same stride-8 maps, relative to the map's
# largest value (float64 tables against cv2's float32 two-step resize)
MAP_BOUND = 1e-5


@pytest.fixture(autouse=True, scope="module")
def no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def _model(golden):
    from ctrlora_b200.annotator.openpose import bodypose_model
    model = bodypose_model()
    model.load_state_dict(og.weights({k: s for k, s in golden["keys"]}), strict=True)
    return model.cuda()


@pytest.fixture(scope="module")
def model(golden):
    return _model(golden)


# ------------------------------------------------------------------------------------------------ 7x7 GEMM
@pytest.mark.parametrize("hw", [(23, 23), (23, 39), (13, 17)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("c,n,seg", [(128, 128, 0), (192, 40, 0), (192, 256, 0), (192, 256, 128), (128, 24, 0)])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("split_k", [0, 1, 4])
@pytest.mark.parametrize("simt", [False, True])
def test_gemm_7x7_against_conv2d(hw, c, n, seg, relu, split_k, simt):
    from ctrlora_b200 import ops
    if simt and split_k:
        pytest.skip("the CUDA-core twin has no split-K plan")
    h, w = hw
    g = torch.Generator(device="cuda").manual_seed(h * 1000 + w * 10 + n)
    b = 2
    x = torch.randn((b, h, w, c), device="cuda", generator=g).half()
    if c == 192:  # the stage input buffer: 185 live channels, zero padding columns
        x[..., 166:168] = 0
        x[..., 187:] = 0
    wt = (torch.randn((n, 49, c), device="cuda", generator=g) * (49 * c) ** -0.5).half()
    bias = torch.randn(n, device="cuda", generator=g) * 0.1
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), wt.view(n, 7, 7, c).permute(0, 3, 1, 2).double(), bias.double(),
                   padding=3).permute(0, 2, 3, 1)
    if relu:
        ref = ref.clamp_min(0)
    run = ops.gemm_relu if relu else ops.gemm
    kw = dict(ksize=7, bias=bias, split_k=split_k, simt=simt)
    if seg:
        outs = [torch.empty((b, h, w, seg), device="cuda", dtype=torch.float16) for _ in range(n // seg)]
        run(x, wt, seg_outs=outs, seg_width=seg, **kw)
        got = torch.cat(outs, dim=-1)
    else:
        got = run(x, wt, **kw)
    close(got, ref, what=f"7x7 {hw} c{c} n{n} seg{seg} relu{relu} split{split_k} simt{simt}")


def test_gemm_7x7_writes_a_column_slice():
    """a producer of the stage buffer: N = 40 into columns 128..167 of a 192-wide buffer, its neighbours untouched"""
    from ctrlora_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((1, 23, 23, 128), device="cuda", generator=g).half()
    wt = (torch.randn((40, 1, 128), device="cuda", generator=g) * 128 ** -0.5).half()
    buf = torch.full((1, 23, 23, 192), 7.0, device="cuda", dtype=torch.float16)
    ops.gemm(x, wt, out=buf[..., 128:168])
    ref = (x.double().reshape(-1, 128) @ wt.double().reshape(40, 128).T).reshape(1, 23, 23, 40)
    close(buf[..., 128:168], ref)
    assert (buf[..., :128] == 7).all() and (buf[..., 168:] == 7).all()


@pytest.mark.parametrize("hwc", [(184, 312, 64), (46, 78, 128), (23, 39, 256), (9, 7, 512)])
def test_max_pool_only(hwc):
    from ctrlora_b200 import ops
    h, w, c = hwc
    x = torch.randn((2, h, w, c), device="cuda").half()
    got = ops.max_pool2x2(x)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(got.float(), ref)


# ------------------------------------------------------------------------------------------------ post-process kernels
def _pixel_major(t):
    """[1, C, h8, w8] -> fp32 pixel-major [h8, w8, C] on the GPU"""
    return t[0].permute(1, 2, 0).contiguous().float().cuda()


def _host_maps(maps8, h, w):
    """Body's two cv2 resizes of the stride-8 maps [C, h8, w8] (numpy float32) -> float32 [C, h, w]"""
    from ctrlora_b200.annotator import openpose as op
    rh, rw, ph, pw = op.geometry(h, w)
    interp = op.resize_interp(rh, rw, h, w)
    return np.stack([cv2.resize(cv2.resize(m, (pw, ph), interpolation=cv2.INTER_LANCZOS4)[:rh, :rw], (w, h),
                                interpolation=interp) for m in maps8])


@pytest.mark.parametrize("case", list(og.PP_CASES))
def test_resample_smooth_peaks_kernels(case):
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator import openpose as op
    h, w = og.PP_CASES[case]["size"]
    _, heat8 = og.planted_maps(case)
    post = op.PostProcess()
    tabs = post.tables(h, w, "cuda")
    heat = ops.openpose_resample(_pixel_major(heat8), tabs, 18)
    ref = _host_maps(heat8[0, :18].numpy(), h, w)
    err = (heat.cpu().numpy() - ref).__abs__().max() / np.abs(ref).max()
    print(f"{case}: resample max err {err:.2e}")
    assert err < MAP_BOUND
    smooth = ops.openpose_smooth(heat, op.gaussian_weights())
    ref_s = np.stack([scipy.ndimage.gaussian_filter(m.astype(np.float64), sigma=3) for m in heat.cpu().numpy()])
    assert np.abs(smooth.cpu().numpy() - ref_s).max() <= 1e-14 * np.abs(ref_s).max()
    px, py, part, score = ops.openpose_peaks(smooth, heat, op.THRE_PEAK, capacity=4)  # forces the second pass
    s = smooth.cpu().numpy()
    p = np.pad(s, ((0, 0), (1, 1), (1, 1)))
    mask = ((s >= p[:, :-2, 1:-1]) & (s >= p[:, 2:, 1:-1]) & (s >= p[:, 1:-1, :-2]) & (s >= p[:, 1:-1, 2:]) &
            (s > op.THRE_PEAK))
    parts, ys, xs = np.nonzero(mask)
    assert np.array_equal(part.cpu().numpy(), parts) and np.array_equal(py.cpu().numpy(), ys)
    assert np.array_equal(px.cpu().numpy(), xs)
    assert np.array_equal(score.cpu().numpy(), heat.cpu().numpy()[parts, ys, xs])


def test_smooth_reflects_short_lines():
    """maps shorter than the 12-tap radius reflect more than once, as scipy does"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator import openpose as op
    x = torch.rand((2, 9, 5), device="cuda")
    got = ops.openpose_smooth(x, op.gaussian_weights()).cpu().numpy()
    ref = np.stack([scipy.ndimage.gaussian_filter(m.astype(np.float64), sigma=3) for m in x.cpu().numpy()])
    assert np.abs(got - ref).max() <= 1e-14


@pytest.mark.parametrize("case", list(og.PP_CASES))
def test_device_postprocess_matches_reference(golden, case):
    """planted maps -> exactly the reference's peaks, ids, limbs and people; scores within 1e-5; the same canvas"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator import openpose as op
    g = golden[f"pp.{case}"]
    h, w = og.PP_CASES[case]["size"]
    paf8, heat8 = og.planted_maps(case)
    paf_px, heat_px = _pixel_major(paf8), _pixel_major(heat8)
    post = op.PostProcess()
    candidate, subset = post(paf_px, heat_px, h, w)
    ref_c, ref_s = g["candidate"].numpy(), g["subset"].numpy()
    assert candidate.shape == ref_c.shape
    assert np.array_equal(candidate[:, [0, 1, 3]], ref_c[:, [0, 1, 3]])
    np.testing.assert_allclose(candidate[:, 2], ref_c[:, 2], rtol=SCORE_RTOL, atol=0)
    assert subset.shape == ref_s.shape
    assert np.array_equal(subset[:, :18], ref_s[:, :18]) and np.array_equal(subset[:, 19], ref_s[:, 19])
    np.testing.assert_allclose(subset[:, 18], ref_s[:, 18], rtol=SCORE_RTOL, atol=0)
    pose = op.pose_dict(candidate, subset, h, w)
    assert np.array_equal(op.draw_body(pose, h, w), g["canvas"].numpy())
    # the pair scores themselves: every passing pair of every limb, through the wrapper the detector uses
    _, _, (px, py, part, _) = post.peaks(heat_px, h, w)
    counts = g["counts"].numpy()
    first = np.concatenate([[0], np.cumsum(counts)])
    limbs, pairs, order = [], 0, []
    for k, ((a, b), (cx, cy)) in enumerate(zip(op.LIMB_PARTS, op.LIMB_PAF)):
        if counts[a - 1] and counts[b - 1]:
            limbs.append((pairs, int(first[a - 1]), int(counts[a - 1]), int(first[b - 1]), int(counts[b - 1]),
                          cx - 19, cy - 19))
            order.append((k, pairs, int(counts[a - 1] * counts[b - 1]), int(counts[b - 1])))
            pairs += counts[a - 1] * counts[b - 1]
    sc, ok = ops.openpose_limbs(paf_px, post.tables(h, w, "cuda"), px, py, limbs, h, op.THRE_PAF)
    sc, ok = sc.cpu().numpy(), ok.cpu().numpy()
    for k, base, n, n_b in order:
        ref = g["limb_candidates"][k].numpy()
        sel = np.nonzero(ok[base:base + n])[0]
        assert np.array_equal(np.stack([sel // n_b, sel % n_b], 1), ref[:, :2].astype(int).reshape(-1, 2)), k
        np.testing.assert_allclose(sc[base + sel], ref[:, 2], rtol=SCORE_RTOL, atol=0)


# ------------------------------------------------------------------------------------------------ network
@pytest.mark.parametrize("size", list(og.NET_SIZES))
def test_network_matches_reference(model, golden, size):
    from ctrlora_b200.annotator import openpose as op
    g = golden[f"net.{size}"]
    x = torch.from_numpy(op.network_input(og.image(size))).cuda()
    paf, heat = model(x)
    r_paf, r_heat = norm_rel(paf.cpu(), g["paf"]), norm_rel(heat.cpu(), g["heat"])
    print(f"{size}: PAF norm-rel {r_paf:.2e}, heatmaps {r_heat:.2e}")
    assert paf.shape == g["paf"].shape and heat.shape == g["heat"].shape
    assert r_paf < NET_BOUND and r_heat < NET_BOUND


def test_batch_equals_single_images(golden):
    from ctrlora_b200.annotator import openpose as op
    model = _model(golden)
    model.split_k = 1
    xs = [torch.from_numpy(op.network_input(og.image(s))) for s in ("384x640", "120x200")]
    xs.append(-xs[0].flip(-1))
    batch = model(torch.cat(xs).cuda())
    for i, x in enumerate(xs):
        single = model(x.cuda())
        assert torch.equal(batch[0][i:i + 1], single[0]) and torch.equal(batch[1][i:i + 1], single[1])


def test_detector_end_to_end(golden, tmp_path):
    """the whole detector on synthetic weights: its resampled and smoothed heatmaps against cv2 + scipy run on its own
    network output, and the pose dict and canvas it returns"""
    from ctrlora_b200.annotator import openpose as op
    model = op.bodypose_model()
    sd = og.weights({k: s for k, s in golden["keys"]})
    torch.save({k.split(".", 1)[1]: v for k, v in sd.items()}, tmp_path / "body_pose_model.pth")
    det = op.OpenposeDetector(ckpt_dir=str(tmp_path))
    img = og.image("384x640")
    h, w = img.shape[:2]
    body = det.body_estimation
    paf, heat_px = body.model.run_maps(torch.from_numpy(op.network_input(img[:, :, ::-1].copy())).cuda())
    heat, smooth, _ = body.post.peaks(heat_px[0], h, w)
    ref = _host_maps(heat_px[0].permute(2, 0, 1)[:18].cpu().numpy(), h, w)
    err = np.abs(heat.cpu().numpy() - ref).max() / np.abs(ref).max()
    ref_s = np.stack([scipy.ndimage.gaussian_filter(m.astype(np.float64), sigma=3) for m in ref])
    err_s = np.abs(smooth.cpu().numpy() - ref_s).max() / np.abs(ref_s).max()
    print(f"detector 384x640: resampled heatmaps max err {err:.2e}, smoothed {err_s:.2e}")
    assert err < MAP_BOUND and err_s < MAP_BOUND
    pose = det(img, return_is_index=True)
    canvas = det(img)
    assert set(pose) == {"bodies", "hands", "faces"} and pose["hands"] == [] and pose["faces"] == []
    assert canvas.shape == (h, w, 3) and canvas.dtype == np.uint8
    assert np.array_equal(canvas, op.draw_body(pose, h, w))
    with pytest.raises(NotImplementedError):
        det(img, hand_and_face=True)
