"""The anime line-art annotator's host side: the module tree against the reference's state dict, the refused sizes and
constructor arguments, the checkpoint loader (the `module.` prefix, no network access), the 4 x 4 sub-pixel
decomposition of the transposed convs in plain torch, and the launch references of its new kernel arguments at tiny
shapes."""
import functools
import os
import socket

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from golden_io import load_golden
import launch_refs as R
import lineart_anime_launches as AL
import lineart_anime_golden as lg
from ctrlora_b200.annotator.lineart_anime import (TAPS4, LineartAnimeDetector, UnetGenerator, load_netg,
                                                  phase_taps)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lineart_anime_golden.pt")
NORM = functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def generator(num_downs=lg.NUM_DOWNS):
    return UnetGenerator(3, 1, num_downs, 64, norm_layer=NORM, use_dropout=False)


def test_state_dict_matches_reference(golden):
    """keys, order and shapes of UnetGenerator(3, 1, 8) equal the reference's (recorded from the reference module)"""
    ours = [(k, tuple(v.shape)) for k, v in generator().state_dict().items()]
    assert ours == [(k, tuple(s)) for k, s in golden["keys"]]
    assert len(ours) == 32 and sum(v.numel() for v in generator().state_dict().values()) == 54_405_505


def test_reference_weights_load_strict(golden):
    generator().load_state_dict(lg.weights({k: s for k, s in golden["keys"]}), strict=True)


def test_module_prefixed_checkpoint_loads(golden, tmp_path):
    """a DataParallel checkpoint (`module.` keys) loads through the detector's loader, as the reference strips it"""
    sd = lg.weights({k: s for k, s in golden["keys"]})
    torch.save({"module." + k: v for k, v in sd.items()}, tmp_path / "netG.pth")
    ck = load_netg(str(tmp_path / "netG.pth"))
    assert list(ck) == list(sd)
    model = generator()
    model.load_state_dict(ck, strict=True)
    assert torch.equal(model.model.model[0].weight, sd["model.model.0.weight"])


@pytest.mark.parametrize("hw", [(500, 740), (256, 384), (128, 256), (512, 520)])
def test_size_not_multiple_of_256_is_refused(hw):
    with pytest.raises(NotImplementedError, match="multiples of 256"):
        generator()(torch.zeros(1, 3, *hw))


def test_smaller_unets_need_their_own_multiple():
    with pytest.raises(NotImplementedError, match="multiples of 32"):
        generator(5)(torch.zeros(1, 3, 48, 64))


@pytest.mark.parametrize("args,kwargs", [
    ((4, 1, 8), {"norm_layer": NORM}),
    ((3, 3, 8), {"norm_layer": NORM}),
    ((3, 1, 4), {"norm_layer": NORM}),
    ((3, 1, 8, 32), {"norm_layer": NORM}),
    ((3, 1, 8), {}),                                                     # the reference's default BatchNorm2d
    ((3, 1, 8), {"norm_layer": functools.partial(nn.InstanceNorm2d, affine=True)}),
    ((3, 1, 8), {"norm_layer": functools.partial(nn.InstanceNorm2d, track_running_stats=True)}),
    ((3, 1, 8), {"norm_layer": NORM, "use_dropout": True}),
])
def test_unsupported_constructor_arguments_are_refused(args, kwargs):
    with pytest.raises(NotImplementedError, match="LineartAnimeDetector builds"):
        UnetGenerator(*args, **kwargs)


def test_plain_instance_norm_class_is_accepted():
    UnetGenerator(3, 1, 5, norm_layer=nn.InstanceNorm2d)


def test_missing_checkpoint_raises_without_network(tmp_path, monkeypatch):
    def no_network(*args, **kwargs):
        raise AssertionError("LineartAnimeDetector tried to open a socket")
    monkeypatch.setattr(socket, "socket", no_network)
    monkeypatch.setattr(socket, "create_connection", no_network)
    with pytest.raises(FileNotFoundError) as e:
        LineartAnimeDetector(ckpt_dir=str(tmp_path))
    assert str(tmp_path / "netG.pth") in str(e.value)


def test_subpixel_phases_recompose_conv_transpose():
    """ConvTranspose2d(4, stride 2, padding 1) equals, at output phase (py, px), the sum over phase_taps of the input
    shifted by (dy, dx) (zero outside) through kernel tap (ky, kx)"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 6, 5, 7, generator=g, dtype=torch.float64)
    w = torch.randn(6, 4, 4, 4, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, w, stride=2, padding=1)
    assert ref.shape[2:] == (10, 14)
    xp = F.pad(x, (1, 1, 1, 1))
    h, wd = x.shape[2:]
    for py in (0, 1):
        for px in (0, 1):
            acc = torch.zeros(2, 4, h, wd, dtype=torch.float64)
            for dy, dx, ky, kx in phase_taps(py, px):
                acc += torch.einsum("bihw,io->bohw", xp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + wd], w[:, :, ky, kx])
            torch.testing.assert_close(acc, ref[:, :, py::2, px::2], rtol=1e-12, atol=1e-12)
    assert [len(phase_taps(py, px)) for py in (0, 1) for px in (0, 1)] == [4, 4, 4, 4]


def test_stride2_taps_are_the_down_conv():
    """the 16 stride-2 taps, tap-major and channel-minor, times the conv weight in that order are Conv2d(4, 2, 1)"""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 6, 8, 10, generator=g, dtype=torch.float64)
    w = torch.randn(5, 6, 4, 4, generator=g, dtype=torch.float64)
    cols = AL.tap_gather_act(x, TAPS4, reflect=False, k_pad=16 * 6, stride=2)           # fp64 NCHW source
    got = cols @ w.permute(0, 2, 3, 1).reshape(5, -1).t()
    torch.testing.assert_close(got.permute(0, 3, 1, 2), F.conv2d(x, w, stride=2, padding=1), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("act", [None, "relu", "leaky"])
def test_tap_gather_reference_stride_and_activation(act):
    """lineart_anime_launches.tap_gather_act with stride 2 and an activation: a loop over output pixels and taps, the activation
    applied to the fp16 source in fp32 and rounded once"""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 6, 8, 16, generator=g).half()                               # [B, H, W, C] fp16
    taps = [(-1, 2), (0, 0), (2, -1)]
    got = AL.tap_gather_act(x, taps, reflect=False, k_pad=56, stride=2, act=act)
    assert got.shape == (2, 3, 4, 56) and got.dtype == torch.float16
    f = x.float()
    f = f if act is None else (f.clamp_min(0) if act == "relu" else torch.where(f > 0, f, f * 0.2))
    f = f.half()
    for y in range(3):
        for xx in range(4):
            for t, (dy, dx) in enumerate(taps):
                sy, sx = 2 * y + dy, 2 * xx + dx
                inside = 0 <= sy < 6 and 0 <= sx < 8
                want = f[:, sy, sx] if inside else torch.zeros(2, 16, dtype=torch.float16)
                assert torch.equal(got[:, y, xx, t * 16:(t + 1) * 16], want)
    assert not got[..., 48:].any()
    assert torch.equal(AL.tap_gather_act(x, taps, reflect=False, k_pad=56, stride=1, act=None),
                       R.tap_gather(x, taps, reflect=False, k_pad=56))


def test_lineart_anime_out_reference():
    """lineart_anime_launches.lineart_anime_out against an explicit scatter of every input pixel through the 4 x 4 kernel"""
    g = torch.Generator().manual_seed(3)
    skip = torch.randn(1, 3, 4, 4, generator=g, dtype=torch.float64)
    up = torch.randn(1, 3, 4, 4, generator=g, dtype=torch.float64)
    weight = torch.randn(8, 16, generator=g, dtype=torch.float64)
    bias = torch.tensor([0.3], dtype=torch.float64)
    got = AL.lineart_anime_out(skip, up, weight, bias, scale=127.5, shift=127.5)
    assert got.shape == (1, 1, 6, 8)
    x = torch.cat([skip, up], -1).clamp_min(0)[0]                                  # [h, w, C]
    acc = torch.zeros(2 * 3 + 2, 2 * 4 + 2, dtype=torch.float64)                   # one pixel of margin each side
    for iy in range(3):
        for ix in range(4):
            for ky in range(4):
                for kx in range(4):
                    acc[2 * iy + ky, 2 * ix + kx] += x[iy, ix] @ weight[:, ky * 4 + kx]
    ref = torch.tanh(acc[1:-1, 1:-1] + 0.3) * 127.5 + 127.5
    torch.testing.assert_close(got[0, 0], ref, rtol=1e-12, atol=1e-12)
