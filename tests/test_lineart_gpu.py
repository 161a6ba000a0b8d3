"""The line-art annotator on an H100: each new kernel against fp32 torch at the detector's shapes, Generator.forward
against the reference's fp32 CPU result (tests/golden/lineart_golden.pt), determinism, and LineartDetector end to end.

Bounds are norm-relative errors ||ours - ref|| / ||ref|| unless stated, each set above the figure measured on an H100
80GB HBM3 (noted beside it) with some headroom.  Run with -s to print the measured figures."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_io import load_golden
import lineart_golden as lg

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lineart_golden.pt")

# Generator.forward against the fixture (synthetic weights, fp16 activations, fp32 accumulation and statistics); measured
# at 512^2 / 384x640 / 64^2: map 6.75e-4 / 6.75e-4 / 7.19e-4; model0 6.63e-4, model1 1.27e-3, model2 2.29e-3, model3 2.53e-3
# (worst of the three sizes); uint8 at most 1 level off, 7.7-7.8 % of the pixels off at all
MAP_BOUND = 1.5e-3
STAGE_BOUND = {0: 1.5e-3, 1: 2.5e-3, 2: 4.5e-3, 3: 5e-3}
# the transposed-conv phases: an fp16 GEMM against fp32 torch over K = 128 ... 1024; measured 2.81e-4 ... 3.05e-4
PHASE_BOUND = 6e-4
# instance norm: the fp16 rounding of the output dominates; measured 2.06e-4 ... 2.12e-4
NORM_BOUND = 4e-4
# the output conv: fp32 accumulation of 3136 fp16 x fp32 products in another order than cuDNN's; measured 1.31e-7
OUT_BOUND = 1e-6


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(autouse=True, scope="module")
def no_tf32():
    """fp32 torch references in full fp32 (cuDNN convs default to TF32)"""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


@pytest.fixture(scope="module")
def generator(golden):
    from ctrlora_b200.annotator.lineart import Generator
    model = Generator(3, 1, lg.N_RESIDUAL)
    model.load_state_dict(lg.weights({k: s for k, s in golden["keys"]}), strict=True)
    return model.cuda()


def image_tensor(img):
    return (torch.from_numpy(img).float() / 255.0).permute(2, 0, 1).unsqueeze(0).contiguous().cuda()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("b,h,w,c", [(1, 128, 128, 256), (2, 24, 40, 256), (1, 8, 8, 256)])
def test_tap_gather_reflect_3x3(b, h, w, c):
    """the residual blocks' ReflectionPad2d(1) + 3x3 taps: a copy, exact"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart import TAPS3
    x = torch.randn(b, c, h, w, device="cuda").half()
    got = ops.tap_gather(nhwc(x), TAPS3, reflect=True, k_pad=9 * c)
    xp = F.pad(x.float(), (1, 1, 1, 1), mode="reflect")
    ref = torch.cat([xp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w] for dy, dx in TAPS3], 1)
    assert torch.equal(got.float(), nhwc(ref))


@pytest.mark.parametrize("h,w", [(512, 512), (384, 640), (64, 64)])
def test_tap_gather_reflect_7x7_from_fp32_nchw(h, w):
    """model0's ReflectionPad2d(3) + 7x7 taps from the fp32 input, K = 147 zero-padded to 160: exact up to the fp16 cast"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart import TAPS7
    x = torch.rand(1, 3, h, w, device="cuda")
    got = ops.tap_gather(x, TAPS7, reflect=True, k_pad=160)
    xp = F.pad(x, (3, 3, 3, 3), mode="reflect")
    ref = torch.cat([xp[:, :, 3 + dy:3 + dy + h, 3 + dx:3 + dx + w] for dy, dx in TAPS7], 1)
    assert torch.equal(got[..., :147].float(), nhwc(ref).half().float())
    assert not got[..., 147:].any()


@pytest.mark.parametrize("cin,cout,h", [(256, 128, 128), (128, 64, 256), (256, 128, 24)])
def test_transposed_conv_phases(cin, cout, h):
    """each sub-pixel phase (zero-masked tap gather + GEMM with the kernel slice) against F.conv_transpose2d"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart import Generator
    convt = torch.nn.ConvTranspose2d(cin, cout, 3, stride=2, padding=1, output_padding=1, bias=False).cuda()
    x = torch.randn(1, cin, h, h, device="cuda").half()
    ref = F.conv_transpose2d(x.float(), convt.weight.float(), stride=2, padding=1, output_padding=1)
    phases = Generator(3, 1, 0)._phase_weights("t", convt)
    for p, (taps, wp) in enumerate(phases):
        got = ops.gemm(ops.tap_gather(nhwc(x), taps, reflect=False, k_pad=len(taps) * cin), wp)
        e = rel(got.float(), nhwc(ref[:, :, p >> 1::2, p & 1::2]))
        print(f"convT {cin}->{cout} at {h}x{h}, phase {p} ({len(taps)} taps): rel {e:.2e}")
        assert e < PHASE_BOUND, (p, e)


NORM_SHAPES = [(1, 512, 512, 64), (1, 256, 256, 128), (1, 128, 128, 256), (2, 96, 160, 256), (3, 16, 16, 256)]


@pytest.mark.parametrize("b,h,w,c", NORM_SHAPES)
@pytest.mark.parametrize("mode", ["relu", "residual"])
def test_instance_norm(b, h, w, c, mode):
    from ctrlora_b200 import ops
    x = (torch.randn(b, c, h, w, device="cuda") * 3 + 40 * torch.randn(1, c, 1, 1, device="cuda")).half()
    res = torch.randn(b, c, h, w, device="cuda").half() if mode == "residual" else None
    ref = F.instance_norm(x.float(), eps=1e-5)
    ref = ref + res.float() if res is not None else F.relu(ref)
    got = ops.instance_norm(nhwc(x), relu=mode == "relu", residual=None if res is None else nhwc(res))
    e = rel(got.float(), nhwc(ref))
    print(f"instance norm {mode} {(b, h, w, c)}: rel {e:.2e}")
    assert e < NORM_BOUND


@pytest.mark.parametrize("b,h,w,c", [(1, 128, 128, 128), (1, 256, 256, 64), (2, 12, 20, 64)])
def test_instance_norm_phases(b, h, w, c):
    """phases=True: statistics over the four phase outputs, written interleaved to [B, 2H, 2W, C]"""
    from ctrlora_b200 import ops
    full = (torch.randn(b, c, 2 * h, 2 * w, device="cuda") * 2 + 5).half()
    ph = torch.stack([nhwc(full[:, :, p >> 1::2, p & 1::2]) for p in range(4)])
    got = ops.instance_norm(ph.contiguous(), relu=True, phases=True)
    e = rel(got.float(), nhwc(F.relu(F.instance_norm(full.float(), eps=1e-5))))
    print(f"instance norm phases {(b, h, w, c)}: rel {e:.2e}")
    assert e < NORM_BOUND


@pytest.mark.parametrize("b,h,w", [(1, 512, 512), (1, 384, 640), (2, 36, 20)])
def test_output_conv_sigmoid_u8(b, h, w):
    from ctrlora_b200 import ops
    x = torch.relu(torch.randn(b, 64, h, w, device="cuda")).half()
    conv = torch.nn.Conv2d(64, 1, 7).cuda()
    wk = conv.weight.detach()[0].permute(1, 2, 0).reshape(49, 64).contiguous()
    y, u8 = ops.lineart_out(nhwc(x), wk, conv.bias.detach().float(), want_u8=True)
    with torch.no_grad():
        ref = torch.sigmoid(F.conv2d(F.pad(x.float(), (3, 3, 3, 3), mode="reflect"), conv.weight, conv.bias))
    e = rel(y, ref)
    print(f"output conv {(b, h, w)}: rel {e:.2e}")
    assert e < OUT_BOUND
    assert torch.equal(u8.cpu(), torch.from_numpy(lg.quantise(y[:, 0].cpu().numpy())))
    assert (u8.int() - torch.from_numpy(lg.quantise(ref[:, 0].cpu().numpy())).cuda().int()).abs().max() <= 1


def test_output_u8_clip_bounds():
    """sigmoid saturating to exactly 1.0 gives 255 and tiny values give 0, as the reference's clip + truncation"""
    from ctrlora_b200 import ops
    x = torch.ones(1, 16, 16, 64, device="cuda").half()
    wk = torch.zeros(49, 64, device="cuda")
    for bias, level in ((40.0, 255), (-40.0, 0), (0.0, 127)):
        y, u8 = ops.lineart_out(x, wk, torch.tensor([bias], device="cuda"), want_u8=True)
        assert (u8 == level).all(), (bias, u8.unique())
        assert torch.equal(u8.cpu(), torch.from_numpy(lg.quantise(y[:, 0].cpu().numpy())))


# ------------------------------------------------------------------------------------------------ the network
@pytest.mark.parametrize("size", list(lg.SIZES))
def test_generator_matches_reference(generator, golden, size):
    g = golden[size]
    img = lg.image(size)
    assert int(img.astype(np.int64).sum()) == g["input_sum"]
    y, stages = generator.forward_stages(image_tensor(img))
    e_map = rel(y[0, 0].cpu(), lg.golden_map(golden, size))
    errs = {}
    for i, s in enumerate(stages):
        _, c, h, w = s.shape
        errs[i] = rel(lg.sample_stage(s, lg.stage_positions(h, w, c)), g[f"stage{i}"])
    _, u8 = generator.detect(image_tensor(img))
    d = (u8[0].cpu().int() - g["u8"].int()).abs()
    print(f"{size}: map rel {e_map:.2e}, stages " + ", ".join(f"model{i} {e:.2e}" for i, e in errs.items()) +
          f"; uint8 max |diff| {int(d.max())}, differing {float((d > 0).float().mean()):.4%}")
    assert e_map < MAP_BOUND
    for i, e in errs.items():
        assert e < STAGE_BOUND[i], (i, e)
    assert int(d.max()) <= 1


def test_generator_is_deterministic(generator):
    x = image_tensor(lg.image("384x640"))
    a, b = generator(x), generator(x)
    assert torch.equal(a, b)


def test_batch_equals_single_images(generator):
    xs = [image_tensor(lg.image((64, 96), tag=f".{i}")) for i in range(4)]
    batch = torch.cat(xs)
    old = generator.split_k
    try:
        generator.split_k = 1
        one = torch.cat([generator(x) for x in xs])
        assert torch.equal(generator(batch), one)
    finally:
        generator.split_k = old
    e = rel(generator(batch), torch.cat([generator(x) for x in xs]))
    print(f"batch 4 vs 4 x batch 1 with the tile model's plans: rel {e:.2e}")
    assert e < MAP_BOUND


# ------------------------------------------------------------------------------------------------ the detector
def test_lineart_detector_end_to_end(golden, tmp_path):
    from ctrlora_b200.annotator.lineart import Generator, LineartDetector
    shapes = {k: s for k, s in golden["keys"]}
    fine = lg.weights(shapes)
    coarse = {k: v * 0.9 for k, v in fine.items()}
    torch.save(fine, tmp_path / "sk_model.pth")
    torch.save(coarse, tmp_path / "sk_model2.pth")
    det = LineartDetector(ckpt_dir=str(tmp_path))
    img = lg.image("64")
    line = det(img, coarse=False)
    assert line.dtype == np.uint8 and line.shape == img.shape[:2]
    assert np.abs(line.astype(int) - golden["64"]["u8"].numpy().astype(int)).max() <= 1
    ref_coarse = Generator(3, 1, 3)
    ref_coarse.load_state_dict(coarse)
    _, u8 = ref_coarse.cuda().detect(image_tensor(img))
    line_c = det(img, coarse=True)
    assert np.array_equal(line_c, u8[0].cpu().numpy())
    assert not np.array_equal(line_c, line)
