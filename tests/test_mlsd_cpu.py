"""The M-LSD line annotator without a GPU: the module tree against the reference network's state dict, the torch
restatement of tools/mlsd_bench.py with the BatchNorms folded as the kernels fold them against the fixture, the size
and threshold rules that return zeros, the host filter and draw against the reference's maps bit for bit, and the
launch references of tests/mlsd_launches.py against index-loop restatements."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from golden_io import load_golden, unband  # noqa: E402
import mlsd_golden as mg  # noqa: E402
import mlsd_launches as MLL  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mlsd_golden.pt")
LIVE = [s for s in mg.SIZES if s not in mg.ZERO_SIZES]


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def _net(weights=True):
    from ctrlora_b200.annotator.mlsd import MobileV2_MLSD_Large
    net = MobileV2_MLSD_Large()
    if weights:
        bn = [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
        net.load_state_dict(mg.weights({k: tuple(v.shape) for k, v in net.state_dict().items()}, bn), strict=True)
    return net


def test_state_dict_is_the_reference_networks(golden):
    net = _net(weights=False)
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == [(k, tuple(s)) for k, s in golden["keys"]]
    assert len(golden["keys"]) == 362


def test_missing_checkpoint_raises(tmp_path):
    from ctrlora_b200.annotator.mlsd import MLSDdetector
    with pytest.raises(FileNotFoundError, match="mlsd_large_512_fp32.pth"):
        MLSDdetector(ckpt_dir=str(tmp_path), device="cpu")


def _folded_forward(net, x):
    """the network with every BatchNorm folded into its conv by mlsd.fold_bn (the kernels' weights, in fp32)"""
    from ctrlora_b200.annotator.mlsd import fold_bn

    def cbr(seq, x, stride=1, act=F.relu, tflite=False):
        c = seq[0]
        w, b = fold_bn(c, seq[1] if len(seq) > 1 else None)
        if tflite:
            x, pad = F.pad(x, (0, 1, 0, 1)), 0
        else:
            pad = c.dilation[0] * (c.kernel_size[0] // 2)
        y = F.conv2d(x, w, b, stride=stride, padding=pad, dilation=c.dilation, groups=c.groups)
        return act(y) if act is not None else y

    relu6 = lambda t: t.clamp(0, 6)  # noqa: E731
    f = net.backbone.features
    y = cbr(f[0], x, 2, relu6, tflite=True)
    feats = []
    for i in range(1, 14):
        blk, layers = f[i], list(f[i].conv)
        t = cbr(layers[0], y, 1, relu6) if len(layers) == 4 else y
        t = cbr(layers[-3], t, blk.stride, relu6, tflite=blk.stride == 2)
        t = cbr([layers[-2], layers[-1]], t, act=None)
        y = y + t if blk.use_res_connect else t
        if i in (1, 3, 6, 10, 13):
            feats.append(y)

    def block_a(blk, a, b):
        b = cbr(blk.conv1, b)
        if blk.upscale:
            b = F.interpolate(b, scale_factor=2.0, mode="bilinear", align_corners=True)
        return torch.cat((cbr(blk.conv2, a), b), 1)

    def block_b(blk, x):
        return cbr(blk.conv2, cbr(blk.conv1, x) + x)

    c1, c2, c3, c4, c5 = feats
    y = block_b(net.block16, block_a(net.block15, c4, c5))
    y = block_b(net.block18, block_a(net.block17, c3, y))
    y = block_b(net.block20, block_a(net.block19, c2, y))
    y = block_b(net.block22, block_a(net.block21, c1, y))
    c = net.block23
    y = cbr([c.conv3], cbr(c.conv2, cbr(c.conv1, y)), act=None)
    return y[:, 7:], feats


@pytest.mark.parametrize("size", ["512", "497x513"])
def test_folded_restatement_matches_the_fixture(golden, size):
    """the BN-folded fp32 restatement (and the unfolded one of tools/mlsd_bench.py) give the reference's features and
    head map at the fixture's sampled positions"""
    from ctrlora_b200.annotator.mlsd import network_input
    from tools.mlsd_bench import torch_forward
    net = _net()
    img = mg.image(size)
    assert int(img.astype("int64").sum()) == golden[f"{size}.input_sum"]
    x = network_input(img)
    with torch.no_grad():
        out, feats = _folded_forward(net, x)
        out2, feats2 = torch_forward(net, x, stages=True)
    for fn_out, fn_feats, bound in ((out, feats, 2e-5), (out2, feats2, 2e-6)):
        for i, f in enumerate(fn_feats + [fn_out]):
            _, c, h, w = f.shape
            assert (c, h, w) == tuple(golden[f"{size}.stage{i}.shape"])
            got = mg.sample_stage(f, mg.stage_positions(h, w, c))
            ref = golden[f"{size}.stage{i}"]
            rel = ((got - ref).norm() / ref.norm()).item()
            assert rel < bound, (size, i, rel)


def test_network_input_is_the_references():
    from ctrlora_b200.annotator.mlsd import network_input
    img = mg.image("512x768")
    x = network_input(img)
    assert x.dtype == torch.float32 and tuple(x.shape) == (1, 4, 512, 768)
    ref = (np.concatenate([img, np.ones([512, 768, 1])], -1).transpose(2, 0, 1)[None].astype("float32") / 127.5) - 1.0
    assert np.array_equal(x.numpy(), ref)
    assert x[0, 3].unique().tolist() == [np.float32(1.0) / np.float32(127.5) - np.float32(1.0)]


@pytest.mark.parametrize("h,w,thr_v,zero", [
    (512, 512, 0.1, False), (497, 513, 0.5, False), (16, 400, 0.1, False), (17, 400, 0.1, False),
    (16, 16, 0.1, True), (16, 48, 0.1, True), (500, 740, 0.1, True), (512, 520, 0.1, True), (15, 512, 0.1, True),
    (512, 512, 1.0, True), (512, 512, 1.7, True), (512, 512, 0.9999, False), (512, 512, float("nan"), True)])
def test_zero_rules(h, w, thr_v, zero):
    from ctrlora_b200.annotator.mlsd import returns_zeros
    assert returns_zeros(h, w, thr_v) == zero


@pytest.mark.parametrize("h,w", [(496, 512), (497, 513), (512, 768), (16, 17)])
def test_zero_rules_agree_with_the_decoder_shapes(h, w):
    """the size rule is exactly 'the x2-upsampled levels match the next one', as the decoder's torch.cat needs"""
    from ctrlora_b200.annotator.mlsd import check_size
    levels = [h]
    for _ in range(4):
        levels.append(levels[-1] // 2)
    ok = all(2 * levels[i + 1] == levels[i] for i in (1, 2, 3)) and levels[4] >= 1
    cols = [w]
    for _ in range(4):
        cols.append(cols[-1] // 2)
    ok = ok and all(2 * cols[i + 1] == cols[i] for i in (1, 2, 3)) and cols[4] >= 1
    assert ok
    check_size(h, w)
    for bad in ((h + 2, w), (h, w + 4)):
        with pytest.raises(ValueError):
            check_size(*bad)


def test_fixture_zero_sizes(golden):
    for size in mg.ZERO_SIZES:
        assert golden[f"{size}.zero"]
        from ctrlora_b200.annotator.mlsd import returns_zeros
        assert returns_zeros(*mg.SIZES[size], 0.1)


@pytest.mark.parametrize("size", LIVE)
def test_host_filter_and_draw_are_the_references(golden, size):
    """the fixture's reference candidates through select_lines and draw_lines give the reference's segments and maps
    bit for bit"""
    from ctrlora_b200.annotator.mlsd import draw_lines, select_lines
    h, w = mg.SIZES[size]
    idx, val = golden[f"{size}.cand_idx"].numpy(), golden[f"{size}.cand_val"].numpy()
    for thr_v, thr_d in mg.THRESHOLDS:
        key = f"{size}.thr{thr_v}_{thr_d}"
        lines = select_lines(idx, val, w // 2, thr_v, thr_d)
        ref_lines = golden[f"{key}.lines"]
        if ref_lines is None:
            assert lines == []
        else:
            assert lines == [tuple(int(v) for v in row) for row in ref_lines.tolist()]
        m = draw_lines(h, w, lines)
        ref = np.zeros((h, w), dtype=np.uint8)
        nz = golden[f"{key}.nonzero"].numpy()
        ref[nz[:, 0], nz[:, 1]] = 255
        assert np.array_equal(m, ref), (key, int((m != ref).sum()))


def test_fixture_is_spread(golden):
    """scores over (0.1, 1), lengths over (0.1, 20), and a reference top 200 that is no near-tie: the 200th score
    exceeds the 201st by over a thousand fp32 units (about 3e-8 at these scores), so neither torch.topk's tie order nor
    a float32 / float64 comparison can change the reference's own set.  That gap is not above the fp16 path's score
    error (up to 7.2e-3 on an H100): with about 5000 peaks per 256 x 256 map, the spacing of the scores near rank 200
    and that error both scale with the head's centre column, so no CENTER_SCALE / CENTER_BIAS separates them, and
    tests/test_mlsd_gpu.py compares candidates against a margin instead."""
    for size in LIVE:
        val = golden[f"{size}.cand_val"]
        assert 0.1 < val[:, 0].min() and val[:, 0].max() < 1
        assert 0.1 < val[:, 1].min() and val[:, 1].max() < 20
        assert val[199, 0] - golden[f"{size}.score201"] > 5e-5


# ---------------------------------------------------------------------------------------------- launch references
def _rand(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("act", [None, "relu", "relu6"])
def test_dwconv_act_reference(stride, act):
    h, w, c, k = 7, 6, 8, 3
    x, wt, b = _rand(1, h, w, c, seed=1) * 4, _rand(k * k, c, seed=2), _rand(c, seed=3)
    ho, wo = (h, w) if stride == 1 else (h // 2, w // 2)
    res = _rand(1, ho, wo, c, seed=4)
    got = MLL.dwconv_act(x, wt, b, k, stride=stride, act=act, residual=res)
    ref = torch.zeros(1, ho, wo, c, dtype=torch.float64)
    p = k // 2 if stride == 1 else 0
    for y in range(ho):
        for xx in range(wo):
            acc = b.double() + res[0, y, xx].double()
            for ky in range(k):
                for kx in range(k):
                    iy, ix = stride * y + ky - p, stride * xx + kx - p
                    if 0 <= iy < h and 0 <= ix < w:
                        acc = acc + wt[ky * k + kx].double() * x[0, iy, ix].double()
            if act == "relu":
                acc = acc.clamp_min(0)
            elif act == "relu6":
                acc = acc.clamp(0, 6)
            ref[0, y, xx] = acc
    assert torch.allclose(got.double(), ref, atol=1e-4)


def test_gemm_mode_references():
    a, w, b = _rand(1, 3, 4, 8, seed=5), _rand(16, 1, 8, seed=6), _rand(16, seed=7)
    res = _rand(1, 3, 4, 16, seed=8)
    y = a.reshape(-1, 8) @ w.reshape(16, 8).t() + b
    assert torch.allclose(MLL.gemm_relu6(a, w, bias=b, residual=res).reshape(-1, 16), (y + res.reshape(-1, 16)).clamp(0, 6),
                          atol=1e-5)
    assert torch.allclose(MLL.gemm_relu_residual(a, w, bias=b, residual=res).reshape(-1, 16),
                          y.clamp_min(0) + res.reshape(-1, 16), atol=1e-5)


def test_upsample_reference():
    x = _rand(1, 3, 5, 8, seed=9)
    got = MLL.upsample_bilinear2x_into(x, None)
    h, w = 3, 5
    for oy in range(6):
        for ox in range(10):
            fy, fx = (h - 1) / 5 * oy, (w - 1) / 9 * ox
            y0, x0 = int(fy), int(fx)
            y1, x1 = min(y0 + 1, h - 1), min(x0 + 1, w - 1)
            ly, lx = fy - y0, fx - x0
            v = (1 - ly) * ((1 - lx) * x[0, y0, x0] + lx * x[0, y0, x1]) + ly * ((1 - lx) * x[0, y1, x0] + lx * x[0, y1, x1])
            assert torch.allclose(got[0, oy, ox], v, atol=1e-5)


def test_decode_reference():
    """peaks, order (score descending, index ascending), zero fill from the lowest indices, lengths"""
    h, w = 16, 20
    tp = _rand(2, h, w, 16, seed=10) * 3
    tp[1, ..., 7] = -50.0                    # image 1: every heat underflows to ~0 except a few peaks
    tp[1, 2, 3, 7], tp[1, 9, 9, 7], tp[1, 9, 12, 7] = 1.0, 2.0, 1.0
    idx, val = MLL.mlsd_decode(tp, 7, 8)
    for b in range(2):
        heat = torch.sigmoid(tp[b, ..., 7])
        s = {}
        for y in range(h):
            for x in range(w):
                win = heat[max(0, y - 1):y + 2, max(0, x - 1):x + 2]
                s[y * w + x] = float(heat[y, x]) if heat[y, x] == win.max() else 0.0
        order = sorted(s, key=lambda i: (-s[i], i))[:MLL.TOPK]
        assert idx[b].tolist() == order
        for j, i in enumerate(order):
            d = tp[b].reshape(-1, 16)[i, 8:12]
            assert val[b, j, 0] == s[i]
            assert torch.allclose(val[b, j, 1], torch.sqrt((d[0] - d[2]) ** 2 + (d[1] - d[3]) ** 2))
            assert torch.equal(val[b, j, 2:], d)
    assert idx[1, :3].tolist() == [9 * w + 9, 2 * w + 3, 9 * w + 12]


def test_full_map_decodes_to_the_reference_candidates(golden):
    """the decode reference on the fixture's full centre and displacement maps gives the reference's 200 candidates"""
    maps = unband(golden[f"{mg.FULL_SIZE}.maps"])  # [h2, w2, 5]: centre, 4 displacements
    tp = torch.zeros(maps.shape[:2] + (16,))
    tp[..., 7:12] = maps
    idx, val = MLL.mlsd_decode(tp[None], 7, 8)
    ref_idx, ref_val = golden[f"{mg.FULL_SIZE}.cand_idx"], golden[f"{mg.FULL_SIZE}.cand_val"]
    assert torch.equal(idx[0], ref_idx)
    assert torch.allclose(val[0], ref_val, rtol=1e-6, atol=1e-6)
