"""The UniFormer segmentation annotator without a GPU: the module tree against the reference segmentor's state dict,
the mmcv checkpoint layout and its palette, the resize-size rule, the torch restatement of tools/uniformer_bench.py
against the fixture, and the launch references of tests/uniformer_launches.py against index-loop restatements."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from golden_io import load_golden  # noqa: E402
import uniformer_golden as ug  # noqa: E402
import uniformer_launches as UL  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "uniformer_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def _net():
    from ctrlora_b200.annotator.uniformer import UniformerSegmentor
    return UniformerSegmentor()


def _weights(net):
    bn = [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    return ug.weights({k: tuple(v.shape) for k, v in net.state_dict().items()}, bn)


def test_state_dict_is_the_reference_segmentors(golden):
    net = _net()
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == [(k, tuple(s)) for k, s in golden["keys"]]


def test_unsupported_configurations():
    from ctrlora_b200.annotator.uniformer import UniformerSegmentor
    for kw in ({"windows": True}, {"hybrid": True}, {"num_classes": 19}):
        with pytest.raises(NotImplementedError):
            UniformerSegmentor(**kw)


def test_mmcv_checkpoint_loads(golden, tmp_path):
    net = _net()
    sd = _weights(net)
    path = tmp_path / "upernet_global_small.pth"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "meta": {"CLASSES": tuple(map(str, range(150))), "PALETTE": golden["palette"].tolist()}}, path)
    net.load(str(path))
    assert torch.equal(net.palette, golden["palette"])
    assert all(torch.equal(net.state_dict()[k], v) for k, v in sd.items())
    assert "palette" not in net.state_dict()


def test_missing_palette_raises(tmp_path):
    net = _net()
    path = tmp_path / "upernet_global_small.pth"
    torch.save({"state_dict": _weights(net), "meta": {"CLASSES": ()}}, path)
    with pytest.raises(ValueError, match="PALETTE"):
        net.load(str(path))


def test_missing_checkpoint_raises(tmp_path):
    from ctrlora_b200.annotator.uniformer import UniformerDetector
    with pytest.raises(FileNotFoundError, match="upernet_global_small.pth"):
        UniformerDetector(ckpt_dir=str(tmp_path))


def test_resize_rule_matches_the_reference(golden):
    from ctrlora_b200.annotator.uniformer import network_input, rescale_size
    for size, (h, w) in ug.SIZES.items():
        assert rescale_size(h, w) == tuple(golden[f"{size}.net_size"]), size
    x = network_input(ug.image("256x320"))
    assert x.shape == (1, 3, 512, 640) and x.dtype == torch.float32 and x.min() >= 0 and x.max() <= 255


def test_torch_restatement_matches_the_fixture(golden):
    """tools/uniformer_bench.py's torch forward (which the bench compares the kernels with) gives the reference's
    logits: the module tree, Normalize's channel reversal and the resize rule are the reference's"""
    from tools.uniformer_bench import torch_forward
    from ctrlora_b200.annotator.uniformer import network_input
    net = _net()
    net.load_state_dict(_weights(net), strict=True)
    x = network_input(ug.image("256x320"))
    with torch.no_grad():
        logits = torch_forward(net, x)
    c, h, w = golden["256x320.stage4.shape"]
    got = ug.sample_stage(logits, ug.stage_positions(h, w, c))
    ref = golden["256x320.stage4"]
    assert ((got - ref).norm() / ref.norm()).item() < 1e-5


def test_fixture_labels_are_varied(golden):
    for size in ug.SIZES:
        labels = ug.unband(golden[f"{size}.labels"]).long()
        margin = ug.unband(golden[f"{size}.margin"]).float()
        assert len(labels.unique()) > 20 and (margin > 0.1).float().mean() > 0.8
        rgb = ug.unband(golden[f"{size}.rgb"])
        assert torch.equal(rgb, golden["palette"][labels])


# ------------------------------------------------------------------------------------------------ launch references
def _loop_dwconv(x, wt, bias, k, residual):
    b, h, w, c = x.shape
    out = torch.zeros(b, h, w, c, dtype=torch.float64)
    for yy in range(h):
        for xx in range(w):
            acc = bias.double().clone().expand(b, c).clone()
            for ky in range(k):
                for kx in range(k):
                    iy, ix = yy + ky - k // 2, xx + kx - k // 2
                    if 0 <= iy < h and 0 <= ix < w:
                        acc += wt[ky * k + kx].double() * x[:, iy, ix].double()
            out[:, yy, xx] = acc + (residual[:, yy, xx].double() if residual is not None else 0)
    return out


def _src(d, scale, n):
    r = max(scale * (d + 0.5) - 0.5, 0.0)
    i0 = min(int(r), n - 1)
    i1 = i0 + (i0 < n - 1)
    l1 = r - i0
    return i0, i1, 1 - l1, l1


def _loop_resize(x, ho, wo):
    b, hi, wi, c = x.shape
    out = torch.zeros(b, ho, wo, c, dtype=torch.float64)
    xd = x.double()
    for yy in range(ho):
        y0, y1, a0, a1 = _src(yy, hi / ho, hi)
        for xx in range(wo):
            x0, x1, b0, b1 = _src(xx, wi / wo, wi)
            out[:, yy, xx] = a0 * (b0 * xd[:, y0, x0] + b1 * xd[:, y0, x1]) + a1 * (b0 * xd[:, y1, x0] + b1 * xd[:, y1, x1])
    return out


def _loop_pool(x, s):
    b, h, w, c = x.shape
    out = torch.zeros(b, s, s, c, dtype=torch.float64)
    for i in range(s):
        y0, y1 = (i * h) // s, math.ceil((i + 1) * h / s)
        for j in range(s):
            x0, x1 = (j * w) // s, math.ceil((j + 1) * w / s)
            out[:, i, j] = x[:, y0:y1, x0:x1].double().mean(dim=(1, 2))
    return out.reshape(-1, c)


@pytest.mark.parametrize("k", [3, 5])
def test_dwconv_reference(k):
    g = torch.Generator().manual_seed(k)
    x = torch.randn(2, 6, 7, 8, generator=g).half()
    wt, bias = torch.randn(k * k, 8, generator=g), torch.randn(8, generator=g)
    for res in (None, x):
        ref = UL.dwconv(x, wt, bias, k, residual=res).double()
        loop = _loop_dwconv(x, wt, bias, k, res)
        assert (ref - loop).abs().max() <= 2e-3 * loop.abs().max()


@pytest.mark.parametrize("src,dst", [((6, 6), (26, 53)), ((26, 53), (7, 11)), ((1, 1), (5, 4)), ((5, 5), (5, 5)),
                                     ((128, 213), (384, 640))])
def test_resize_reference_and_rule(src, dst):
    """the fp32 reference is torch's F.interpolate(size=...); the loop restates the rule the kernels implement"""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, *src, 8, generator=g).half()
    ref = UL.resize_bilinear(x, size=dst).double()
    loop = _loop_resize(x, *dst)
    assert (ref - loop).abs().max() <= 2e-3 * loop.abs().max()
    acc = torch.randn(1, *dst, 8, generator=g).half()
    ref_acc = UL.resize_bilinear(x, out=acc.clone(), accumulate=True).double()
    assert (ref_acc - (loop + acc.double())).abs().max() <= 2e-3 * (loop + acc.double()).abs().max()


@pytest.mark.parametrize("h,w", [(16, 26), (16, 16), (12, 64), (5, 7), (26, 16)])
def test_pool_reference_and_bins(h, w):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, h, w, 8, generator=g).half()
    for s, ref in zip((1, 2, 3, 6), UL.adaptive_avg_pool(x, (1, 2, 3, 6))):
        loop = _loop_pool(x, s)
        assert (ref.double() - loop).abs().max() <= 2e-3 * loop.abs().max()


def test_seg_output_reference():
    g = torch.Generator().manual_seed(3)
    logits = torch.zeros(1, 8, 10, 12)
    logits[..., :10] = torch.randn(1, 8, 10, 10, generator=g)
    palette = torch.randint(0, 256, (10, 3), generator=g, dtype=torch.uint8)
    labels, margin, rgb = UL.seg_output(logits, 10, (32, 40), (24, 50), palette)
    up = _loop_resize(logits[..., :10], 32, 40)
    up = _loop_resize(up, 24, 50)
    loop_labels = up.argmax(-1)
    top2 = up.topk(2, dim=-1).values
    assert torch.equal(labels[(top2[..., 0] - top2[..., 1] > 1e-5)], loop_labels[(top2[..., 0] - top2[..., 1] > 1e-5)])
    assert torch.allclose(margin.double(), top2[..., 0] - top2[..., 1], atol=1e-5)
    assert torch.equal(rgb, palette[labels])
    assert np.array_equal(rgb.shape, (1, 24, 50, 3))
