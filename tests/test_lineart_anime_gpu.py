"""The anime line-art annotator on an H100: each new or extended kernel against fp32 torch at the detector's shapes,
the existing line-art kernel calls against what the library recorded before they were extended, UnetGenerator.forward
and every block against the reference's fp32 CPU result (tests/golden/lineart_anime_golden.pt), determinism, batches,
LineartAnimeDetector end to end, and every kernel launch of one detector call against its fp32 launch reference
(tests/launch_refs.py, and tests/lineart_anime_launches.py for the two wrappers of this path).

Bounds are norm-relative errors ||ours - ref|| / ||ref|| unless stated, each set above the figure measured on an H100
80GB HBM3 (noted beside it) with some headroom.  Run with -s to print the measured figures."""
import functools
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_io import load_golden  # noqa: E402
import lineart_anime_launches as AL  # noqa: E402
import lineart_anime_golden as lg  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lineart_anime_golden.pt")
PARITY = os.path.join(ROOT, "tests", "golden", lg.PARITY_GOLDEN)
NORM = functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)

# UnetGenerator.forward against the fixture (synthetic weights, fp16 activations, fp32 accumulation and statistics);
# measured at 256^2 / 512^2 / 512 x 768: map 7.73e-4 / 6.97e-4 / 6.95e-4; blocks 1 ... 7 from 1.01e-3 (block 1) to
# 2.55e-3 (block 7 at 256^2, whose 2 x 2 norms see 4 and 16 pixels)
MAP_BOUND = 1.5e-3
BLOCK_BOUND = 4e-3
# the detector's uint8 maps against the fixture's: every pixel within one level, 2.65 % (500 x 740) and 3.04 %
# (512 x 768) of them off by one
U8_MAX_DIFF = 1
U8_SHARE = 0.045
# instance norm: the fp16 rounding of the output dominates; measured 1.98e-4 ... 2.10e-4
NORM_BOUND = 4e-4
# a transposed-conv phase over the two halves of a concatenation (two operand pairs in one GEMM); measured 2.89e-4 ...
# 3.06e-4
PHASE_BOUND = 6e-4
# the fused output conv: fp32 accumulation of 512 fp16 x fp32 products in another order than cuDNN's, then tanh;
# measured 2.13e-7 ... 2.75e-7
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


def synth_weights(golden):
    return lg.weights({k: s for k, s in golden["keys"]})


@pytest.fixture(scope="module")
def generator(golden):
    from ctrlora_b200.annotator.lineart_anime import UnetGenerator
    model = UnetGenerator(3, 1, lg.NUM_DOWNS, 64, norm_layer=NORM)
    model.load_state_dict(synth_weights(golden), strict=True)
    return model.cuda()


@pytest.fixture(scope="module")
def ckpt_dir(golden, tmp_path_factory):
    d = tmp_path_factory.mktemp("lineart_anime_ckpt")
    torch.save({"module." + k: v for k, v in synth_weights(golden).items()}, d / "netG.pth")
    return str(d)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("b,h,w,c,act", [(1, 256, 256, 64, "leaky"), (2, 64, 96, 256, "leaky"), (1, 4, 4, 512, "leaky"),
                                         (1, 2, 2, 512, "leaky"), (1, 128, 128, 128, "relu"), (1, 32, 48, 64, None)])
def test_tap_gather_stride2_activation(b, h, w, c, act):
    """the down convs' stride-2 16-tap gathers with LeakyReLU on load (and the other activations): exact copies of the
    fp32 activation rounded to fp16"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart_anime import TAPS4
    x = torch.randn(b, h, w, c, device="cuda").half()
    got = ops.tap_gather_act(x, TAPS4, reflect=False, k_pad=16 * c, stride=2, act=act)
    f = x.float() if act is None else (F.relu(x.float()) if act == "relu" else F.leaky_relu(x.float(), 0.2))
    cols = F.unfold(f.half().float().permute(0, 3, 1, 2), 4, padding=1, stride=2)       # [B, C * 16, L]
    ref = cols.view(b, c, 16, h // 2, w // 2).permute(0, 3, 4, 2, 1).reshape(b, h // 2, w // 2, 16 * c)
    assert torch.equal(got.float(), ref)
    assert torch.equal(got, AL.tap_gather_act(x, TAPS4, reflect=False, k_pad=16 * c, stride=2, act=act))


@pytest.mark.parametrize("h,w", [(512, 768), (256, 256)])
def test_tap_gather_stride2_from_fp32_nchw(h, w):
    """block 0's conv: 16 taps from the fp32 input, K = 48 zero-padded to 64, exact up to the fp16 cast"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart_anime import TAPS4
    x = torch.rand(1, 3, h, w, device="cuda") * 2 - 1
    got = ops.tap_gather_act(x, TAPS4, reflect=False, k_pad=64, stride=2)
    cols = F.unfold(x, 4, padding=1, stride=2).view(1, 3, 16, h // 2, w // 2).permute(0, 3, 4, 2, 1)
    assert torch.equal(got[..., :48].float(), cols.reshape(1, h // 2, w // 2, 48).half().float())
    assert not got[..., 48:].any()


def test_tap_gather_act_entry_point_without_stride_or_activation_is_the_old_gather():
    """ctrlora_tap_gather_act_f16 with stride 1 and no activation writes what ctrlora_tap_gather_f16 writes"""
    import ctypes as C
    from ctrlora_b200 import _lib, ops
    from ctrlora_b200.annotator.lineart import TAPS3
    x = torch.randn(2, 24, 40, 256, device="cuda").half()
    old = ops.tap_gather(x, TAPS3, reflect=True, k_pad=9 * 256)
    new = torch.empty_like(old)
    flat = (C.c_int * 18)(*[v for t in TAPS3 for v in t])
    _lib.check(_lib.load().ctrlora_tap_gather_act_f16(x.data_ptr(), 0, 256, new.data_ptr(), 2, 24, 40, 256,
                                                      C.cast(flat, C.c_void_p), 9, 1, 9 * 256, 1, 0, ops._sp()), "gather")
    assert torch.equal(old, new)


def test_existing_line_art_calls_are_unchanged():
    """the 64 / 128 / 256-channel instance norms (plain and phase-interleaved) and the stride-1 gathers give what the
    library returned before the 512-channel norm and the strided gathers were added, bit for bit
    (tools/make_lineart_anime_parity.py)"""
    from ctrlora_b200 import ops
    want = load_golden(PARITY)
    got = lg.parity_calls(ops, torch.device("cuda"))
    assert sorted(got) == sorted(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k


NORM_SHAPES = [(1, 4, 4, 512), (1, 2, 2, 512), (1, 1, 1, 512), (3, 16, 24, 512), (1, 64, 64, 512), (2, 2, 2, 256)]


@pytest.mark.parametrize("b,h,w,c", NORM_SHAPES)
def test_instance_norm_512_and_tiny_images(b, h, w, c):
    from ctrlora_b200 import ops
    x = (torch.randn(b, c, h, w, device="cuda") * 3 + 40 * torch.randn(1, c, 1, 1, device="cuda")).half()
    got = ops.instance_norm(nhwc(x), relu=False)
    ref = nhwc(F.instance_norm(x.float(), eps=1e-5)) if h * w > 1 else torch.zeros_like(got, dtype=torch.float32)
    if h * w == 1:  # a single pixel normalises to exactly 0 (the reference's F.instance_norm refuses 1 x 1 inputs)
        assert not got.any()
        return
    e = rel(got.float(), ref)
    print(f"instance norm {(b, h, w, c)}: rel {e:.2e}")
    assert e < NORM_BOUND


@pytest.mark.parametrize("b,h,w,c", [(1, 1, 1, 512), (1, 2, 2, 512), (2, 4, 6, 512), (1, 32, 32, 256)])
def test_instance_norm_phases_512(b, h, w, c):
    """phases=True over the transposed convs' phase outputs, down to the 1 x 1 phases of the 2 x 2 norm at 256^2"""
    from ctrlora_b200 import ops
    full = (torch.randn(b, c, 2 * h, 2 * w, device="cuda") * 2 + 5).half()
    ph = torch.stack([nhwc(full[:, :, p >> 1::2, p & 1::2]) for p in range(4)])
    got = ops.instance_norm(ph.contiguous(), relu=False, phases=True)
    e = rel(got.float(), nhwc(F.instance_norm(full.float(), eps=1e-5)))
    print(f"instance norm phases {(b, h, w, c)}: rel {e:.2e}")
    assert e < NORM_BOUND


@pytest.mark.parametrize("i,h", [(1, 128), (3, 32), (6, 4), (7, 1)])
def test_transposed_conv_phases_over_the_concatenation(generator, i, h):
    """block i's ConvTranspose2d over relu([x | up]) as four phases, each one GEMM with two operand pairs (the
    innermost block, 7: one operand) against F.conv_transpose2d on the materialised concatenation"""
    from ctrlora_b200 import ops
    blk = generator.blocks()[i]
    convt = blk.convs()[1]
    cin = convt.in_channels
    inner = i == lg.NUM_DOWNS - 1
    skip = torch.randn(1, h, h, cin if inner else cin // 2, device="cuda").half()
    up = None if inner else torch.randn(1, h, h, cin // 2, device="cuda").half()
    cat = F.relu(skip.float()) if inner else F.relu(torch.cat([skip.float(), up.float()], -1))
    ref = F.conv_transpose2d(cat.permute(0, 3, 1, 2), convt.weight.float(), stride=2, padding=1)
    if inner:
        skip = F.relu(skip)  # the innermost block's operand is the conv's ReLU'd output
    for p, (taps, *ws) in enumerate(generator._phase_weights(i, convt, split=not inner)):
        a = ops.tap_gather_act(skip, taps, reflect=False, k_pad=4 * skip.shape[-1], act=None if inner else "relu")
        if inner:
            got = ops.gemm(a, ws[0])
        else:
            got = ops.gemm(a, ws[0], a2=ops.tap_gather_act(up, taps, reflect=False, k_pad=4 * up.shape[-1], act="relu"),
                           w2=ws[1])
        e = rel(got.float(), nhwc(ref[:, :, p >> 1::2, p & 1::2]))
        print(f"block {i} convT {cin}->{convt.out_channels} at {h}x{h}, phase {p}: rel {e:.2e}")
        assert e < PHASE_BOUND, (p, e)


@pytest.mark.parametrize("b,h,w", [(1, 256, 384), (1, 128, 128), (2, 20, 36), (1, 3, 5)])
@pytest.mark.parametrize("scale,shift", [(1.0, 0.0), (127.5, 127.5)])
def test_output_conv_tanh(b, h, w, scale, shift):
    from ctrlora_b200 import ops
    skip = torch.randn(b, h, w, 64, device="cuda").half()
    up = torch.randn(b, h, w, 64, device="cuda").half()
    convt = torch.nn.ConvTranspose2d(128, 1, 4, stride=2, padding=1).cuda()
    with torch.no_grad():
        convt.weight.mul_(0.25)
    wk = convt.weight.detach().reshape(128, 16).contiguous()
    y = ops.lineart_anime_out(skip, up, wk, convt.bias.detach().float(), scale=scale, shift=shift)
    with torch.no_grad():
        x = F.relu(torch.cat([skip.float(), up.float()], -1)).permute(0, 3, 1, 2)
        ref = torch.tanh(F.conv_transpose2d(x, convt.weight, convt.bias, stride=2, padding=1)) * scale + shift
    e = rel(y, ref) if shift == 0.0 else rel(y - shift, ref - shift)
    print(f"output conv {(b, h, w)} scale {scale}: rel {e:.2e}")
    assert y.shape == (b, 1, 2 * h, 2 * w)
    assert e < OUT_BOUND


# ------------------------------------------------------------------------------------------------ the network
@pytest.mark.parametrize("size", list(lg.SIZES))
def test_generator_matches_reference(generator, golden, size):
    g = golden[size]
    img = lg.image(size)
    assert int(img.astype(np.int64).sum()) == g["input_sum"]
    y, blocks = generator.forward_stages(lg.image_tensor(img).cuda())
    e_map = rel(y[0, 0].cpu(), lg.golden_map(golden, size))
    errs = {}
    for i, s in enumerate(blocks, start=1):
        _, c, h, w = s.shape
        errs[i] = rel(lg.sample_stage(s, lg.stage_positions(h, w, c)), g[f"block{i}"])
    print(f"{size}: map rel {e_map:.2e}, blocks " + ", ".join(f"{i} {e:.2e}" for i, e in errs.items()))
    assert len(blocks) == lg.NUM_DOWNS - 1
    assert e_map < MAP_BOUND
    for i, e in errs.items():
        assert e < BLOCK_BOUND, (i, e)


def test_generator_is_deterministic(generator):
    x = lg.image_tensor(lg.image("512x768")).cuda()
    a, b = generator(x), generator(x)
    assert torch.equal(a, b)


def test_batch_equals_single_images(generator):
    xs = [lg.image_tensor(lg.image((256, 512), tag=f".{i}")).cuda() for i in range(3)]
    batch = torch.cat(xs)
    old = generator.split_k
    try:
        generator.split_k = 1
        one = torch.cat([generator(x) for x in xs])
        assert torch.equal(generator(batch), one)
    finally:
        generator.split_k = old
    e = rel(generator(batch), torch.cat([generator(x) for x in xs]))
    print(f"batch 3 vs 3 x batch 1 with the tile model's plans: rel {e:.2e}")
    assert e < MAP_BOUND


# ------------------------------------------------------------------------------------------------ the detector
@pytest.mark.parametrize("case", ["detector", "512x768"])
def test_detector_end_to_end(golden, ckpt_dir, case):
    from ctrlora_b200.annotator.lineart_anime import LineartAnimeDetector
    det = LineartAnimeDetector(ckpt_dir=ckpt_dir)
    img = lg.image(lg.DETECTOR_SIZE if case == "detector" else case)
    assert int(img.astype(np.int64).sum()) == golden[case]["input_sum"]
    line = det(img)
    assert line.dtype == np.uint8 and line.shape == img.shape[:2]
    d = np.abs(line.astype(int) - golden[case]["u8"].numpy().astype(int))
    share = float((d > 0).mean())
    print(f"detector {img.shape[:2]}: uint8 max |diff| {int(d.max())}, differing {share:.4%}")
    assert int(d.max()) <= U8_MAX_DIFF
    assert share < U8_SHARE


def test_detector_launches(ckpt_dir, monkeypatch):
    """every kernel launch of one detector call at 512 x 768 against its fp32 launch reference"""
    from ctrlora_b200.annotator.lineart_anime import LineartAnimeDetector
    det = LineartAnimeDetector(ckpt_dir=ckpt_dir)
    img = lg.image("512x768")
    sh = AL.shadow(monkeypatch)
    line = det(img)
    sh.check("LineartAnimeDetector at 512x768")
    assert line.shape == img.shape[:2]
    recs = [(op, shape) for op, shape, _ in sh.records]
    assert any(op == "tap_gather_act" and "f32nchw" in s and "taps=16 zero k_pad=64 stride=2" in s for op, s in recs)
    assert any(op == "tap_gather_act" and "1x4x6x512" in s and "taps=16" in s and "act=leaky" in s for op, s in recs)
    assert any(op == "tap_gather_act" and "taps=4" in s and "act=relu" in s for op, s in recs)
    assert any(op == "gemm" and "a2" in s.rsplit(" ", 1)[-1].split(",") for op, s in recs)
    assert any(op == "instance_norm" and "512" in s and ",phases" in s for op, s in recs)
    assert any(op == "lineart_anime_out" and "scale=127.5" in s for op, s in recs)
