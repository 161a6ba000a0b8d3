"""The UniFormer segmentation annotator on an H100: each new kernel against fp32 torch, every backbone stage and the
logits against the reference's fp32 CPU result (tests/golden/uniformer_golden.pt), the labels and the RGB map of
UniformerDetector, determinism, weight reloads, batches, and every launch of one detector call.

Bounds are norm-relative errors ||ours - ref|| / ||ref|| unless stated, the end-to-end ones set 20 % above the figure
measured on an H100 80GB HBM3 (noted beside each).
Run with -s to print the measured figures."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_io import load_golden  # noqa: E402
from tolerances import close, norm_rel  # noqa: E402
import uniformer_golden as ug  # noqa: E402
import uniformer_launches as UL  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "uniformer_golden.pt")

# UniFormer-S's four features at sampled positions, worst of five sizes: 18 blocks with an fp16 residual stream,
# measured 2.16e-3 (the 1/32 level; 8.1e-4 at the 1/4 level)
STAGE_BOUND = 2.6e-3
# UPerHead's 1/4-level logits: measured 9.31e-4
LOGITS_BOUND = 1.12e-3
# absolute: labels must match where the reference's top-two logit margin exceeds this, twice the largest logit error
# measured (1.31e-2) + 20 %; the largest margin at which a label differed was 0.010
LABEL_MARGIN = 0.032
# share of the pixels whose label differs: measured 0.087 % ... 0.107 %
LABEL_SHARE = 1.3e-3


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
    from ctrlora_b200.annotator.uniformer import UniformerSegmentor
    net = UniformerSegmentor()
    bn = [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    return ug.weights({k: s for k, s in golden["keys"]}, bn)


@pytest.fixture(scope="module")
def ckpt_dir(golden, tmp_path_factory):
    """the synthetic weights in mmcv's layout, with the ADE palette as the checkpoint's meta"""
    d = tmp_path_factory.mktemp("uniformer_ckpt")
    meta = {"CLASSES": tuple(f"class{i}" for i in range(150)), "PALETTE": golden["palette"].tolist()}
    torch.save({"state_dict": synth_weights(golden), "meta": meta}, d / "upernet_global_small.pth")
    return str(d)


@pytest.fixture(scope="module")
def net(ckpt_dir):
    from ctrlora_b200.annotator.uniformer import UniformerSegmentor
    m = UniformerSegmentor().cuda()
    m.load(os.path.join(ckpt_dir, "upernet_global_small.pth"))
    return m


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def h16(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).half()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("b,h,w,c", [(1, 128, 213, 64), (2, 13, 27, 320), (1, 7, 5, 512), (1, 1, 3, 128)])
@pytest.mark.parametrize("res", [False, True])
def test_dwconv(k, b, h, w, c, res):
    from ctrlora_b200 import ops
    x = h16(b, h, w, c)
    wt = torch.randn(k * k, c, device="cuda") / k
    bias = torch.randn(c, device="cuda") * 0.1
    got = ops.dwconv(x, wt, bias, k, residual=x if res else None)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.t().reshape(c, 1, k, k), bias, padding=k // 2, groups=c)
    ref = nhwc(ref) + (x.float() if res else 0)
    close(got, ref, what=f"dwconv k{k}")


@pytest.mark.parametrize("src,dst", [((16, 26), (128, 213)), ((1, 1), (16, 27)), ((2, 2), (16, 26)), ((3, 3), (13, 64)),
                                     ((6, 6), (26, 53)), ((26, 53), (53, 106)), ((53, 106), (7, 11)), ((5, 5), (5, 5))])
def test_resize_bilinear(src, dst):
    from ctrlora_b200 import ops
    x = h16(2, *src, 64)
    got = ops.resize_bilinear(x, dst)
    ref = nhwc(F.interpolate(x.float().permute(0, 3, 1, 2), size=dst, mode="bilinear", align_corners=False))
    close(got, ref, what=f"resize {src} -> {dst}")


def test_resize_bilinear_slices_and_accumulate():
    """read a channel slice, write a channel slice of a wider buffer (the rest untouched), and accumulate"""
    from ctrlora_b200 import ops
    wide_src = h16(2, 13, 27, 1024)
    x = wide_src[..., 512:]
    buf = h16(2, 26, 53, 2048)
    before = buf.clone()
    ops.resize_bilinear(x, out=buf[..., 1024:1536])
    ref = nhwc(F.interpolate(x.float().permute(0, 3, 1, 2), size=(26, 53), mode="bilinear", align_corners=False))
    close(buf[..., 1024:1536], ref, what="slice write")
    assert torch.equal(buf[..., :1024], before[..., :1024]) and torch.equal(buf[..., 1536:], before[..., 1536:])
    lat = h16(2, 26, 53, 512)
    lat0 = lat.float()
    ops.resize_bilinear(x, out=lat, accumulate=True)
    close(lat, lat0 + ref, what="accumulate")


@pytest.mark.parametrize("h,w", [(128, 213), (53, 106), (27, 27), (4, 6)])
def test_tap_gather_stride2_truncates_odd_sizes(h, w):
    """the patch embeds' 2 x 2 stride-2 gather: an odd size drops its last row or column, as the Conv2d does"""
    from ctrlora_b200 import ops
    x = h16(2, h, w, 64)
    got = ops.tap_gather_act(x, [(0, 0), (0, 1), (1, 0), (1, 1)], reflect=False, k_pad=256, stride=2)
    assert got.shape == (2, h // 2, w // 2, 256)
    ho, wo = h // 2, w // 2
    ref = x[:, :2 * ho, :2 * wo].reshape(2, ho, 2, wo, 2, 64).permute(0, 1, 3, 2, 4, 5).reshape(2, ho, wo, 256)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("h,w", [(16, 26), (12, 64), (26, 16), (5, 7), (16, 16)])
def test_adaptive_avg_pool(h, w):
    from ctrlora_b200 import ops
    wide = h16(2, h, w, 2560)
    x = wide[..., :512]
    outs = ops.adaptive_avg_pool(x, (1, 2, 3, 6))
    for s, got in zip((1, 2, 3, 6), outs):
        ref = nhwc(F.adaptive_avg_pool2d(x.float().permute(0, 3, 1, 2), s)).reshape(-1, 512)
        close(got, ref, what=f"pool {s} of {h}x{w}")


@pytest.mark.parametrize("h4,net,out", [((128, 213), (512, 853), (384, 640)), ((128, 128), (512, 512), (512, 512)),
                                        ((102, 512), (410, 2048), (200, 1000)), ((213, 128), (853, 512), (640, 384))])
def test_seg_output(h4, net, out):
    from ctrlora_b200 import ops
    logits = torch.zeros(1, *h4, 152, device="cuda")
    logits[..., :150] = torch.randn(1, *h4, 150, device="cuda") * 3
    palette = torch.randint(0, 256, (150, 3), device="cuda", dtype=torch.uint8)
    rgb, labels = ops.seg_output(logits, 150, net, out, palette, want_labels=True)
    ref_labels, margin, ref_rgb = UL.seg_output(logits, 150, net, out, palette)
    differ = labels.long() != ref_labels
    print(f"seg_output {h4} -> {net} -> {out}: {differ.float().mean().item():.2e} of the labels differ, smallest margin "
          f"there {margin[differ].max().item() if differ.any() else 0:.2e}")
    assert not (differ & (margin > UL.SEG_MARGIN)).any()
    assert torch.equal(rgb, palette[labels.long()])


# ------------------------------------------------------------------------------------------------ the network
def _stage_errors(golden, net, size):
    from ctrlora_b200.annotator.uniformer import network_input
    img = ug.image(size)
    assert int(img.astype("int64").sum()) == golden[f"{size}.input_sum"]
    x = network_input(img)
    assert tuple(x.shape[2:]) == tuple(golden[f"{size}.net_size"])
    logits, st = net.forward_stages(x.cuda())
    errs = []
    for i, t in enumerate(st["features"] + [logits]):
        c, h, w = golden[f"{size}.stage{i}.shape"]
        assert tuple(t.shape[1:]) == (h, w, c)
        got = ug.sample_stage(t.permute(0, 3, 1, 2), ug.stage_positions(h, w, c))
        errs.append(norm_rel(got, golden[f"{size}.stage{i}"]))
    errs.append((got - golden[f"{size}.stage4"]).abs().max().item())
    return errs


@pytest.mark.parametrize("size", list(ug.SIZES))
def test_stages_and_logits_against_the_reference(golden, net, size):
    errs = _stage_errors(golden, net, size)
    print(f"{size}: stages " + ", ".join(f"{e:.2e}" for e in errs[:4]) + f"; logits {errs[4]:.2e}, max abs {errs[5]:.3e}")
    assert max(errs[:4]) <= STAGE_BOUND
    assert errs[4] <= LOGITS_BOUND


def _labels(net, img):
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.uniformer import NUM_CLASSES, network_input
    x = network_input(img)
    logits, _ = net._run(x.cuda())
    return ops.seg_output(logits, NUM_CLASSES, tuple(x.shape[2:]), img.shape[:2], net.palette, want_labels=True)


@pytest.mark.parametrize("size", list(ug.SIZES))
def test_labels_against_the_reference(golden, net, size):
    """labels equal the reference's wherever its top-two fp32 logit margin exceeds LABEL_MARGIN (twice
    the largest logit error measured at the sampled positions, plus 20 %): two logits each off by less than half the
    margin cannot swap.  The overall share that differs is bounded and printed"""
    rgb, labels = _labels(net, ug.image(size))
    ref = ug.unband(golden[f"{size}.labels"]).long()
    margin = ug.unband(golden[f"{size}.margin"]).float()
    differ = labels[0].cpu().long() != ref
    share = differ.float().mean().item()
    print(f"{size}: {share:.4%} of the labels differ; the largest margin among them {margin[differ].max().item() if differ.any() else 0:.3f}")
    assert not (differ & (margin > LABEL_MARGIN)).any()
    assert share <= LABEL_SHARE


@pytest.mark.parametrize("size", ["384x640", "200x1000"])
def test_detector_rgb(golden, ckpt_dir, size):
    from ctrlora_b200.annotator.uniformer import UniformerDetector
    det = UniformerDetector(ckpt_dir=ckpt_dir)
    out = det(ug.image(size))
    ref = ug.unband(golden[f"{size}.rgb"]).numpy()
    assert out.shape == ref.shape and out.dtype == np.uint8
    margin = ug.unband(golden[f"{size}.margin"]).float().numpy()
    differ = (out != ref).any(-1)
    assert not (differ & (margin > LABEL_MARGIN)).any()
    # every colour is the checkpoint palette's
    pal = {tuple(p) for p in golden["palette"].tolist()}
    assert {tuple(p) for p in np.unique(out.reshape(-1, 3), axis=0).tolist()} <= pal


def test_two_calls_bit_identical(net):
    from ctrlora_b200.annotator.uniformer import network_input
    x = network_input(ug.image("384x640")).cuda()
    assert torch.equal(net(x), net(x))


def test_batch_of_two_equals_two_batches_of_one(net):
    from ctrlora_b200.annotator.uniformer import network_input
    xs = [network_input(ug.image("512", tag)) for tag in ("", ".b")]
    old = net.split_k
    net.split_k = 1
    try:
        both = net(torch.cat(xs).cuda())
        for i, x in enumerate(xs):
            assert torch.equal(both[i], net(x.cuda())[0])
    finally:
        net.split_k = old


def test_weights_follow_load_state_dict(net):
    """the kernel copies (folded BatchNorms included) come from a PrepCache: new weights change the logits, the old ones
    restore them"""
    from ctrlora_b200.annotator.uniformer import network_input
    x = network_input(ug.image("256x320")).cuda()
    before = net(x).clone()
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    mod = dict(sd)
    mod["backbone.blocks1.0.norm1.running_var"] = sd["backbone.blocks1.0.norm1.running_var"] * 2.0
    net.load_state_dict(mod, strict=True)
    assert not torch.equal(net(x), before)
    net.load_state_dict(sd, strict=True)
    assert torch.equal(net(x), before)


def test_detector_launches(ckpt_dir, monkeypatch):
    """every kernel launch of one UniformerDetector call at 384 x 640 against its fp32 launch reference"""
    from ctrlora_b200.annotator.uniformer import UniformerDetector
    det = UniformerDetector(ckpt_dir=ckpt_dir)
    img = ug.image("384x640")
    det(img)  # builds the kernel-layout weights outside the shadow
    sh = UL.shadow(monkeypatch)
    out = det(img)
    sh.check("UniformerDetector at 384x640")
    assert out.shape == (384, 640, 3)
    recs = [(op, shape) for op, shape, _ in sh.records]
    seen = {op for op, _ in recs}
    assert set(UL.NEW) | {"gemm", "gemm_relu", "attention", "tap_gather_act", "patch_gather_hw", "layernorm_rows",
                          "gelu_"} <= seen, sorted(seen)
    assert any(op == "attention" and "nq=1696 nk=1696 d=64" in s for op, s in recs)
    assert any(op == "dwconv" and "k=5" in s for op, s in recs)
    assert any(op == "resize_bilinear" and "accumulate=True" in s for op, s in recs)
