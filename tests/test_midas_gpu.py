"""The MiDaS depth annotator on an H100: each new kernel against fp32 torch, the rectangular patch gather against the
square one, ctrlora_attention_f16 at d_head 64 and DPT-Large's token counts, every DPT stage and the depth against the
reference's fp32 CPU result (tests/golden/midas_golden.pt), MidasDetector's uint8 maps, determinism and batches.

Bounds are norm-relative errors ||ours - ref|| / ||ref|| unless stated, each set above the figure measured on an H100
80GB HBM3 (noted beside it) with headroom.  Run with -s to print the measured figures."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_io import load_golden  # noqa: E402
import midas_golden as mg  # noqa: E402
import midas_launches as ML  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "midas_golden.pt")

# DPTDepthModel.forward against the fixture (synthetic weights, fp16 activations, fp32 accumulation, fp32 ViT stream);
# measured: depth 2.49e-4 ... 3.03e-4 at the four sizes; stages 4.60e-4 (hook1) ... 9.68e-4 (head)
DEPTH_BOUND = 6e-4
STAGE_BOUND = 2e-3
# the detector's uint8 maps against the fixture's.  The depth map: every pixel within one level, 4.8 % ... 10.4 % of
# them off by one.  The normal map comes from finite differences of the depth, which amplify its error (the image's
# fine noise makes the gradients small against the depth): up to 3 levels off, 24 % ... 26 % of the pixels off, 0.38 %
# ... 0.50 % by more than one level
DEPTH_U8_MAX_DIFF, DEPTH_U8_SHARE = 1, 0.15
NORMAL_U8_MAX_DIFF, NORMAL_U8_SHARE, NORMAL_U8_SHARE_2 = 4, 0.35, 0.01
# the ConvTranspose2d as GEMM + depth-to-space: measured 2.05e-4
KERNEL_BOUND = 5e-4


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(autouse=True, scope="module")
def no_tf32():
    """fp32 torch references in full fp32"""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def synth_weights(golden):
    return mg.weights({k: s for k, s in golden["keys"]})


@pytest.fixture(scope="module")
def inference(golden):
    from ctrlora_b200.annotator.midas import DPTDepthModel
    model = DPTDepthModel()
    sd = {k[len("model."):]: v for k, v in synth_weights(golden).items()}
    model.load_state_dict(sd, strict=True)
    return model.cuda()


@pytest.fixture(scope="module")
def ckpt_dir(golden, tmp_path_factory):
    d = tmp_path_factory.mktemp("midas_ckpt")
    sd = {k[len("model."):]: v for k, v in synth_weights(golden).items()}
    torch.save(sd, d / "dpt_large_384.pt")
    return str(d)


def nchw(t):
    return t.float().permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("b,h,w,c,s", [(1, 24, 24, 256, 4), (2, 24, 40, 512, 2), (1, 3, 5, 12, 3), (1, 2, 2, 4, 1)])
def test_depth_to_space_bias(b, h, w, c, s):
    """a kernel = stride ConvTranspose2d as GEMM columns (ky * s + kx) * C + c, then depth-to-space + bias: the bias
    added in fp32 before the one fp16 rounding"""
    from ctrlora_b200 import ops
    src = torch.randn(b, h, w, s * s * c, device="cuda")
    bias = torch.randn(c, device="cuda")
    got = ops.depth_to_space_bias(src, bias, s)
    ref = src.view(b, h, w, s, s, c).permute(0, 1, 3, 2, 4, 5).reshape(b, h * s, w * s, c) + bias
    assert torch.equal(got, ref.half())


def test_conv_transpose_as_gemm():
    """act_postprocess1's ConvTranspose2d(256, 256, 4, stride 4) as the model runs it against F.conv_transpose2d"""
    from ctrlora_b200 import ops, prepare
    x = torch.randn(1, 24, 40, 256, device="cuda").half()
    wt = torch.randn(256, 256, 4, 4, device="cuda") / 64
    bias = torch.randn(256, device="cuda")
    w16 = prepare.linear_weight(wt.permute(2, 3, 1, 0).reshape(16 * 256, 256).contiguous())
    got = ops.depth_to_space_bias(ops.gemm(x, w16, out_f32=True), bias, 4)
    ref = F.conv_transpose2d(nchw(x), wt.half().float(), bias, stride=4)
    err = rel(nchw(got), ref)
    print(f"conv transpose as GEMM: {err:.2e}")
    assert err < KERNEL_BOUND


@pytest.mark.parametrize("shape", [(1, 24, 40, 256), (2, 7, 9, 8), (1, 3, 5, 24)])
def test_add_relu(shape):
    """s = fp16(a + b) and relu(s) in one pass; b omitted: relu(a) only"""
    from ctrlora_b200 import ops
    a = (torch.randn(*shape, device="cuda") * 4).half()
    b = (torch.randn(*shape, device="cuda") * 4).half()
    s, r = ops.add_relu(a, b)
    ref = (a.float() + b.float()).half()
    assert torch.equal(s, ref) and torch.equal(r, ref.clamp_min(0))
    assert torch.equal(ops.add_relu(a), a.clamp_min(0))


@pytest.mark.parametrize("b,h,w,c", [(1, 12, 20, 256), (2, 1, 2, 256), (1, 2, 3, 8), (1, 192, 320, 128), (1, 5, 7, 24)])
def test_upsample_bilinear2x(b, h, w, c):
    """F.interpolate(x2, bilinear, align_corners=True) on fp16 NHWC: within one fp16 unit of torch's own fp16 CUDA kernel,
    whose fp32 weights and sums it restates (FMA contraction may differ).  Measured on an H100: bit-equal.  (An fp32
    interpolation is no yardstick per element: where neighbours cancel, its own weight rounding moves a small result by
    more than one unit of it.)"""
    from ctrlora_b200 import ops
    x = torch.randn(b, h, w, c, device="cuda").half()
    got = ops.upsample_bilinear2x(x)
    ref16 = ML.upsample_bilinear2x(x)
    u16 = ML.one_ulp_f16(got, ref16)
    same = (got == ref16).float().mean().item()
    print(f"upsample {b}x{h}x{w}x{c}: {same:.4f} equal to torch fp16, max {u16:.2f} units from it")
    assert u16 <= 1.0


@pytest.mark.parametrize("b,h,w,c", [(1, 384, 640, 32), (2, 5, 7, 16)])
def test_midas_head_out(b, h, w, c):
    """Conv2d(C -> 1, 1) + bias + ReLU into fp32"""
    from ctrlora_b200 import ops
    x = torch.randn(b, h, w, c, device="cuda").half()
    wt, bias = torch.randn(c, device="cuda"), torch.randn(1, device="cuda")
    got = ops.midas_head_out(x, wt, bias)
    ref = F.relu((x.float() * wt).sum(-1) + bias)
    assert (got - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())


def _maps_reference(depth, a, bg_th):
    """MidasDetector.__call__'s post-process in numpy / cv2 on one fp32 [H, W] depth"""
    import cv2
    depth_pt = depth.copy()
    depth_pt -= np.min(depth_pt)
    depth_pt /= np.max(depth_pt)
    depth_image = (depth_pt * 255.0).clip(0, 255).astype(np.uint8)
    x = cv2.Sobel(depth, cv2.CV_32F, 1, 0, ksize=3)
    y = cv2.Sobel(depth, cv2.CV_32F, 0, 1, ksize=3)
    z = np.ones_like(x) * a
    x[depth_pt < bg_th] = 0
    y[depth_pt < bg_th] = 0
    normal = np.stack([x, y, z], axis=2)
    normal /= np.sum(normal ** 2.0, axis=2, keepdims=True) ** 0.5
    return depth_image, (normal * 127.5 + 127.5).clip(0, 255).astype(np.uint8)


@pytest.mark.parametrize("h,w", [(384, 384), (192, 320), (37, 53)])
def test_midas_maps_against_numpy_and_cv2(h, w):
    """the device post-process against the reference's numpy / cv2 code on the same fp32 depth: the uint8 depth map is
    exact; the normal map within one level (cv2's Sobel sums in another order in the last bit)"""
    from ctrlora_b200 import ops
    g = torch.Generator().manual_seed(h * w)
    depth = (torch.rand(2, h, w, generator=g) * 5).cumsum(1) / h
    depth[1, : h // 3] = 0.0  # a background band below bg_th
    d8, n8 = ops.midas_maps(depth.cuda(), np.pi * 0.2, 0.02)
    for i in range(2):
        rd, rn = _maps_reference(depth[i].numpy(), np.pi * 0.2, 0.02)
        assert np.array_equal(d8[i].cpu().numpy(), rd)
        diff = np.abs(n8[i].cpu().numpy().astype(int) - rn.astype(int))
        print(f"normal map {h}x{w}: max diff {diff.max()}, off by one {(diff > 0).mean():.2e}")
        assert diff.max() <= 1 and (diff > 0).mean() < 1e-3


def test_patch_gather_hw_square_is_the_clip_gather():
    """ctrlora_patch_gather_hw on a square image writes what ctrlora_clip_patch_gather writes, bit for bit"""
    from ctrlora_b200 import ops
    for dtype, patch, s, k_pad in ((torch.float32, 16, 384, 768), (torch.float16, 14, 224, 592)):
        x = torch.randn(2, 3, s, s, device="cuda").to(dtype)
        assert torch.equal(ops.patch_gather_hw(x, patch, k_pad), ops.clip_patch_gather(x, patch, k_pad))


@pytest.mark.parametrize("h,w", [(384, 640), (200, 328)])
def test_patch_gather_hw_rectangular(h, w):
    """the 16 x 16 patch conv as gather + GEMM rows: F.unfold of the cropped image"""
    from ctrlora_b200 import ops
    x = torch.randn(1, 3, h, w, device="cuda")
    got = ops.patch_gather_hw(x, 16, 768)
    gh, gw = h // 16, w // 16
    ref = F.unfold(x[:, :, :16 * gh, :16 * gw], 16, stride=16)[0].T
    assert torch.equal(got.float(), ref.half().float())


@pytest.mark.parametrize("n", [577, 1025, 1537, 25])
def test_attention_d64_at_dpt_token_counts(n):
    """ctrlora_attention_f16 at d_head 64 (its 80-wide instantiation) with DPT-Large's key counts, partial key tiles
    included, against fp32 softmax attention"""
    from ctrlora_b200 import ops
    b, heads, d = 1, 16, 64
    g = torch.Generator(device="cuda").manual_seed(n)
    q, k, v = (torch.randn(b * n, heads * d, device="cuda", generator=g).half() for _ in range(3))
    n_pad = (n + 7) // 8 * 8
    vt = torch.zeros(b, heads, d, n_pad, device="cuda", dtype=torch.float16)
    vt[..., :n] = v.view(b, n, heads, d).permute(0, 2, 3, 1)
    out = ops.attention(q, k, vt, b, heads, n, n, d)
    qv, kv, vv = (t.float().view(n, heads, d).transpose(0, 1) for t in (q, k, v))
    ref = ((qv @ kv.transpose(1, 2)) * d ** -0.5).softmax(-1) @ vv
    err = rel(out.float(), ref.transpose(0, 1).reshape(n, heads * d))
    print(f"attention d64 n={n}: {err:.2e}")
    assert err < 6e-4  # measured 2.50e-4 ... 2.79e-4


# ------------------------------------------------------------------------------------------------ the model
def test_stages_against_the_reference(golden, inference):
    """every hooked ViT stream, reassembled layer, layerN_rn, refinenet and the head against the reference's fp32 CPU
    intermediates at midas_golden.STAGE_SIZE"""
    img = mg.image(mg.STAGE_SIZE)
    assert int(img.astype("int64").sum()) == golden["stage.input_sum"]
    want = golden["stage.stages"]
    depth, st = inference.forward_stages(mg.image_tensor(img).cuda())
    got = {f"hook{i}": h.view(-1, h.shape[-1]) for i, h in enumerate(st["hooks"], 1)}
    got.update({f"layer{i}": nchw(t)[0] for i, t in enumerate(st["layers"], 1)})
    got.update({f"layer{i}_rn": nchw(t)[0] for i, t in enumerate(st["rn"], 1)})
    got.update({f"refinenet{i}": nchw(t)[0] for i, t in zip((4, 3, 2, 1), st["paths"])})
    got["head"] = nchw(st["head"])[0]
    got["depth"] = depth[0]
    worst = 0.0
    for name, ref in want.items():
        err = rel(got[name].cpu(), ref)
        print(f"stage {name}: {err:.2e}")
        worst = max(worst, err)
    assert worst < STAGE_BOUND


@pytest.mark.parametrize("size", list(mg.SIZES))
def test_depth_against_the_reference(golden, inference, size):
    img = mg.image(size)
    assert int(img.astype("int64").sum()) == golden[f"{size}.input_sum"]
    depth = inference(mg.image_tensor(img).cuda())[0].cpu()
    ref = mg.unband(golden[f"{size}.depth"])
    assert depth.shape == ref.shape
    err = rel(depth, ref)
    print(f"depth {size}: {err:.2e}")
    assert err < DEPTH_BOUND


@pytest.mark.parametrize("size", list(mg.SIZES))
def test_detector_maps(golden, ckpt_dir, size):
    from ctrlora_b200.annotator.midas import MidasDetector
    det = MidasDetector(ckpt_dir=ckpt_dir)
    d8, n8 = det(mg.image(size))
    for name, got, max_diff, share in (("depth_u8", d8, DEPTH_U8_MAX_DIFF, DEPTH_U8_SHARE),
                                       ("normal_u8", n8, NORMAL_U8_MAX_DIFF, NORMAL_U8_SHARE)):
        ref = mg.unband(golden[f"{size}.{name}"]).numpy()
        assert got.shape == ref.shape and got.dtype == np.uint8
        diff = np.abs(got.astype(int) - ref.astype(int))
        print(f"detector {size} {name}: max diff {diff.max()}, share off {(diff > 0).mean():.3f}, more than one level off "
              f"{(diff > 1).mean():.4f}")
        assert diff.max() <= max_diff and (diff > 0).mean() < share
        if name == "normal_u8":
            assert (diff > 1).mean() < NORMAL_U8_SHARE_2


def test_two_calls_bit_identical(inference):
    x = mg.image_tensor(mg.image("384x640")).cuda()
    assert torch.equal(inference(x), inference(x))


def test_batch_of_two_equals_two_batches_of_one(inference):
    """with split_k = 1 every GEMM keeps one plan per row, so a batch of 2 equals two batches of 1 bit for bit; under the
    tile model's own plans (split_k = 0) a batch of 2 may split K differently, within a tolerance"""
    xs = [mg.image_tensor(mg.image("384", tag=t)).cuda() for t in ("a", "b")]
    for sk in (1, 0):
        inference.split_k = sk
        try:
            both = inference(torch.cat(xs))
            ones = [inference(x)[0] for x in xs]
        finally:
            inference.split_k = 0
        for i, one in enumerate(ones):
            err = rel(both[i], one)
            print(f"batch 2 image {i}, split_k {sk}: {err:.2e}")
            if sk == 1:
                assert torch.equal(both[i], one)
            assert err < 6e-4  # measured 2.05e-4 with split_k = 0


def test_detector_launches(ckpt_dir, monkeypatch):
    """every kernel launch of one MidasDetector call at 384 x 640 against its fp32 launch reference (tests/launch_refs.py
    and tests/midas_launches.py)"""
    from ctrlora_b200.annotator.midas import MidasDetector
    det = MidasDetector(ckpt_dir=ckpt_dir)
    img = mg.image("384x640")
    det(img)  # builds the kernel-layout weights outside the shadow
    sh = ML.shadow(monkeypatch)
    d8, n8 = det(img)
    sh.check("MidasDetector at 384x640")
    assert d8.shape == (384, 640) and n8.shape == (384, 640, 3)
    recs = [(op, shape) for op, shape, _ in sh.records]
    ops_seen = {op for op, _ in recs}
    assert set(ML.NEW) <= ops_seen, sorted(set(ML.NEW) - ops_seen)
    assert {"gemm", "gemm_relu", "attention", "im2col_s2"} <= ops_seen
    assert any(op == "attention" and "nq=961 nk=961 d=64" in s for op, s in recs)
    assert any(op == "small_linear" and f"ld={961 * 1024}" in s for op, s in recs)
    assert any(op == "cast_rows" and f"ld={961 * 1024}" in s for op, s in recs)
    assert any(op == "gemm" and "rowbias" in s.rsplit(" ", 1)[-1].split(",") for op, s in recs)
    assert any(op == "gemm" and "K=9x256" in s and "res" in s.rsplit(" ", 1)[-1].split(",") for op, s in recs)
    assert any(op == "gemm_relu" and "K=9x256" in s for op, s in recs)


def test_weights_follow_load_state_dict(golden, inference):
    """the kernel copies come from a PrepCache: loading new weights changes the depth, loading the old ones restores it"""
    x = mg.image_tensor(mg.image(mg.STAGE_SIZE)).cuda()
    before = inference(x)
    sd = {k: v.clone() for k, v in inference.state_dict().items()}
    mod = dict(sd)
    mod["scratch.output_conv.4.bias"] = sd["scratch.output_conv.4.bias"] + 1.0
    inference.load_state_dict(mod, strict=True)
    assert not torch.equal(inference(x), before)
    inference.load_state_dict(sd, strict=True)
    assert torch.equal(inference(x), before)
