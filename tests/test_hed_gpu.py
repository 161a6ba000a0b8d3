"""The HED annotators on an H100: the GEMM's ReLU epilogue on every store path, the side / pool and fuse kernels against
torch and cv2, ControlNetHED_Apache2 against the reference's fp32 CPU result (tests/golden/hed_golden.pt),
determinism, batching, and HEDdetector / HEDSketchDetector end to end.

Bounds are norm-relative errors ||ours - ref|| / ||ref|| unless stated, each set above the figure measured on an H100
80GB HBM3 at 700 W (noted beside it) with some headroom.  Run with -s to print the measured figures."""
import os

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_io import load_golden
import hed_golden as hg

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hed_golden.pt")

# the network against the fixture (synthetic weights, fp16 activations, fp32 accumulation); measured at 512^2 /
# 384x640 / 200x328: side maps e1 ... e5 at most 8.1e-4, 1.5e-3, 3.1e-3, 2.8e-3, 2.4e-3; block outputs at most 4.9e-4,
# 6.1e-4, 7.3e-4, 8.6e-4, 9.8e-4; mean map max |diff| 1.66e-2 / 1.50e-2 / 1.32e-2 (its std is about 2); uint8 (safe=False)
# at most 1 level off, 9.9-10.6 % of the pixels off at all; safe=True 289 / 236 / 64 pixels in another bin, all where
# allowed
SIDE_BOUND = 6e-3
STAGE_BOUND = 2e-3
MEAN_ABS_BOUND = 0.03
# side projection: fp32 sums of C fp16 x fp32 products in another order than float64 torch; measured 6.0e-8 ... 1.1e-7
SIDE_KERNEL_BOUND = 1e-6
# fuse: the resize against cv2 (restated coordinates; see test_resize_tables_reproduce_cv2) and the fp32 mean; measured
# max |diff| 1.4e-6 ... 2.8e-6, and at most 2 uint8 pixels off by one, each next to a quantisation step
FUSE_ABS_BOUND = 1e-5


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(autouse=True, scope="module")
def no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


@pytest.fixture(scope="module")
def hed(golden):
    from ctrlora_b200.annotator.hed import ControlNetHED_Apache2
    model = ControlNetHED_Apache2()
    model.load_state_dict(hg.weights({k: s for k, s in golden["keys"]}), strict=True)
    return model.cuda()


def image_tensor(img):
    return torch.from_numpy(img.copy()).float().permute(2, 0, 1).unsqueeze(0).contiguous().cuda()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ GEMM ReLU epilogue
# (ksize, B, H, W, C, N, block_n, split_k, extra): block_n 64 / 128 / 160 with a short K loop run ping-pong, with a long
# one (3x3 at C = 320: 45 k-steps) cooperative; 256 and 320 are cooperative; split_k = 3 splits every tile (the
# row-per-thread epilogue after the split-K sum); "f32" and "residual" take the other store paths
RELU_CASES = [
    (1, 1, 32, 64, 256, 320, 64, 0, None),
    (1, 1, 32, 64, 256, 320, 128, 0, None),
    (1, 1, 32, 64, 256, 320, 160, 0, "residual"),
    (3, 1, 32, 32, 320, 320, 64, 0, None),
    (3, 1, 32, 32, 320, 320, 128, 0, None),
    (3, 1, 32, 32, 320, 320, 160, 0, None),
    (3, 1, 32, 32, 320, 320, 256, 0, None),
    (3, 1, 32, 32, 320, 320, 320, 0, "residual"),
    (3, 2, 48, 40, 64, 64, 0, 0, None),       # ksize 3 at C = 64 (HED's block1), tile model's choice
    (3, 1, 100, 164, 64, 128, 0, 0, None),    # block2's first conv at 200 x 328
    (3, 1, 24, 40, 128, 128, 128, 3, None),
    (3, 1, 24, 40, 128, 128, 0, 0, "f32"),
    (1, 1, 16, 16, 256, 64, 64, 3, "residual"),
]


@pytest.mark.parametrize("ksize,b,h,w,c,n,block_n,split_k,extra", RELU_CASES)
@pytest.mark.parametrize("simt", [False, True])
def test_gemm_relu_equals_clamped_gemm(ksize, b, h, w, c, n, block_n, split_k, extra, simt):
    from ctrlora_b200 import ops
    if simt and (block_n or split_k):
        pytest.skip("the CUDA-core twin has no tiles")
    g = torch.Generator(device="cuda").manual_seed(ksize * 1000 + c + n + block_n)
    a = torch.randn(b, h, w, c, device="cuda", generator=g).half()
    wt = (torch.randn(n, ksize * ksize, c, device="cuda", generator=g) * (ksize * ksize * c) ** -0.5).half()
    bias = torch.randn(n, device="cuda", generator=g) * 0.5
    kw = dict(ksize=ksize, bias=bias, block_n=block_n, split_k=split_k, simt=simt, out_f32=extra == "f32")
    if extra == "residual":
        kw["residual"] = torch.randn(b, h, w, n, device="cuda", generator=g).half()
    plain = ops.gemm(a, wt, **kw)
    got = ops.gemm_relu(a, wt, **kw)
    assert (plain < 0).any() and (plain > 0).any()
    assert torch.equal(got, plain.clamp_min(0))


# ------------------------------------------------------------------------------------------------ side / pool
@pytest.mark.parametrize("b,h,w,c", [(1, 512, 512, 64), (1, 100, 164, 128), (2, 50, 82, 256), (1, 25, 41, 512),
                                     (3, 12, 20, 512), (1, 7, 9, 64)])
@pytest.mark.parametrize("pool", [True, False])
def test_side_pool_against_torch(b, h, w, c, pool):
    from ctrlora_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(b * 100003 + h * 1009 + w * 31 + c + int(pool))
    x = torch.relu(torch.randn(b, c, h, w, device="cuda", generator=g) * 50).half()
    weight = torch.randn(1, c, 1, 1, device="cuda", generator=g) * c ** -0.5
    bias = torch.randn(1, device="cuda", generator=g)
    side, pooled = ops.hed_side_pool(nhwc(x), weight.reshape(-1).contiguous(), bias, pool)
    ref = F.conv2d(x.double(), weight.double(), bias.double())
    e = rel(side, ref)
    print(f"side {(b, h, w, c)}: rel {e:.2e}")
    assert e < SIDE_KERNEL_BOUND
    if pool:
        assert torch.equal(pooled, nhwc(F.max_pool2d(x, 2, 2)))
    else:
        assert pooled is None


# ------------------------------------------------------------------------------------------------ fuse
@pytest.mark.parametrize("size", list(hg.SIZES))
@pytest.mark.parametrize("safe", [False, True])
def test_fuse_against_cv2_numpy(hed, size, safe):
    """on the kernel's own side maps: the mean within FUSE_ABS_BOUND, and the uint8 map equal wherever the
    reference's sigmoid does not sit within that error of a quantisation step"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.hed import level_sizes
    sides = hed(image_tensor(hg.image(size)))
    h, w = sides[0].shape[2:]
    assert [tuple(s.shape[2:]) for s in sides] == level_sizes(h, w)
    mean, u8 = ops.hed_fuse(list(sides), hed._resize_tables(h, w, sides[0].device), safe)
    ref_mean, ref_u8 = hg.host_post([s[0, 0].cpu().numpy() for s in sides], safe)
    err = float(np.abs(mean[0].cpu().numpy() - ref_mean).max())
    d = np.abs(u8[0].cpu().numpy().astype(int) - ref_u8.astype(int))
    sig = 1 / (1 + np.exp(-ref_mean.astype(np.float64)))
    q = sig * (3.0 if safe else 255.0)
    near = np.abs(q - np.round(q)) < 0.25 * (3.0 if safe else 255.0) * 2 * FUSE_ABS_BOUND + 1e-9
    print(f"fuse {size} safe={safe}: mean max |diff| {err:.2e}, uint8 differing {int((d > 0).sum())} "
          f"(near a step: {int(near.sum())})")
    assert err < FUSE_ABS_BOUND
    assert not (d[~near] > 0).any()
    assert int(d.max()) <= (128 if safe else 1)


# ------------------------------------------------------------------------------------------------ the network
@pytest.mark.parametrize("size", list(hg.SIZES))
def test_hed_matches_reference(hed, golden, size):
    g = golden[size]
    img = hg.image(size)
    assert int(img.astype(np.int64).sum()) == g["input_sum"]
    x = image_tensor(img)
    sides, stages = hed.forward_stages(x)
    e_side = [rel(sides[0][0, 0].cpu(), hg.golden_map(golden, size, "e1"))]
    e_side += [rel(sides[i][0, 0].cpu(), g[f"e{i + 1}"]) for i in range(1, 5)]
    e_stage = []
    for i, s in enumerate(stages):
        _, c, h, w = s.shape
        e_stage.append(rel(hg.sample_stage(s, hg.stage_positions(h, w, c)), g[f"stage{i}"]))
    ref_mean = hg.golden_map(golden, size, "mean")
    mean, u8 = hed.detect(x, safe=False)
    _, u8s = hed.detect(x, safe=True)
    mean_err = float((mean[0].cpu() - ref_mean).abs().max())
    d = (u8[0].cpu().int() - g["u8"].int()).abs()
    # safe=True: a pixel may change bins only where the reference's 3 sigmoid lies within the measured error of an
    # integer (sigmoid' <= 1/4)
    q = 3.0 / (1 + np.exp(-ref_mean.double().numpy()))
    near = torch.from_numpy(np.abs(q - np.round(q)) <= 0.75 * mean_err + 1e-6)
    ds = (u8s[0].cpu().int() - g["u8_safe"].int()).abs()
    print(f"{size}: sides " + ", ".join(f"{e:.2e}" for e in e_side) + "; stages " +
          ", ".join(f"{e:.2e}" for e in e_stage) + f"; mean max |diff| {mean_err:.2e}; uint8 max |diff| {int(d.max())}, "
          f"differing {float((d > 0).float().mean()):.4%}; safe differing {int((ds > 0).sum())} (allowed {int(near.sum())}); "
          f"reference peak |activation| per block {[round(p) for p in g['peaks']]}")
    assert max(e_side) < SIDE_BOUND
    assert max(e_stage) < STAGE_BOUND
    assert mean_err < MEAN_ABS_BOUND
    assert int(d.max()) <= 1
    assert not (ds[~near] > 0).any()


def test_hed_is_deterministic(hed):
    x = image_tensor(hg.image("384x640"))
    a, b = hed.detect(x), hed.detect(x)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    sa, sb = hed(x), hed(x)
    assert all(torch.equal(p, q) for p, q in zip(sa, sb))


def test_batch_equals_single_images(hed):
    xs = [image_tensor(hg.image((72, 104), tag=f".{i}")) for i in range(4)]
    batch = torch.cat(xs)
    old = hed.split_k
    try:
        hed.split_k = 1
        one = [hed(x) for x in xs]
        got = hed(batch)
        for lvl in range(5):
            assert torch.equal(got[lvl], torch.cat([o[lvl] for o in one]))
        m1 = torch.cat([hed.detect(x)[1] for x in xs])
        assert torch.equal(hed.detect(batch)[1], m1)
    finally:
        hed.split_k = old


def test_odd_and_minimum_sizes(hed):
    for h, w in ((16, 16), (17, 31), (33, 16)):
        sides = hed(image_tensor(hg.image((h, w))))
        assert [tuple(s.shape[2:]) for s in sides] == [(h >> i, w >> i) for i in range(5)]
        assert all(torch.isfinite(s).all() for s in sides)


# ------------------------------------------------------------------------------------------------ the detectors
def test_hed_detectors_end_to_end(golden, tmp_path):
    from ctrlora_b200.annotator.hed import HEDdetector
    from ctrlora_b200.annotator.hedsketch import HEDSketchDetector
    torch.save(hg.weights({k: s for k, s in golden["keys"]}), tmp_path / "ControlNetHED.pth")
    det = HEDdetector(ckpt_dir=str(tmp_path))
    img = hg.image("200x328")
    edge = det(img)
    assert edge.dtype == np.uint8 and edge.shape == img.shape[:2]
    assert np.abs(edge.astype(int) - golden["200x328"]["u8"].numpy().astype(int)).max() <= 1
    edge_safe = det(img, safe=True)
    assert set(np.unique(edge_safe).tolist()) <= {0, 127, 255}

    sk = HEDSketchDetector(ckpt_dir=str(tmp_path))
    old = np.random.get_state()
    try:
        np.random.seed(0)
        out = sk(img)
        thr = np.random.RandomState(0).randint(110, 160)
    finally:
        np.random.set_state(old)
    ref = golden["sketch"]["hed.0"]["out"].numpy()
    assert out.dtype == np.uint8 and out.shape == img.shape
    # the same first threshold on a map within one level of the reference's: the sketches differ only where a pixel
    # of the map sits at the threshold (and the blur spreads that)
    diff = (out != ref).any(axis=2)
    at_thr = np.abs(golden["200x328"]["u8"].numpy().astype(int) - thr) <= 1
    near = cv2.dilate(at_thr.astype(np.uint8), np.ones((3, 3), np.uint8)).astype(bool)
    print(f"hedsketch: {int(diff.sum())} pixels differ from the reference's sketch, all within 1 pixel of a map value "
          f"at the threshold {thr}")
    assert not (diff & ~near).any()
