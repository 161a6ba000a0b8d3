"""The line-art annotator's host side: the module tree against the reference's state dict, the input-size limits, the
checkpoint lookup without network access, and the sub-pixel decomposition of the transposed convs in plain torch."""
import os
import socket

import pytest
import torch
import torch.nn.functional as F

from golden_io import load_golden
from ctrlora_b200.annotator.lineart import Generator, LineartDetector, phase_taps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lineart_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def test_state_dict_matches_reference(golden):
    """keys, order and shapes of Generator(3, 1, 3) equal the reference's (recorded from the reference module)"""
    ours = [(k, tuple(v.shape)) for k, v in Generator(3, 1, 3).state_dict().items()]
    assert ours == [(k, tuple(s)) for k, s in golden["keys"]]


def test_reference_weights_load_strict(golden):
    import lineart_golden as lg
    model = Generator(3, 1, 3)
    model.load_state_dict(lg.weights({k: s for k, s in golden["keys"]}), strict=True)


@pytest.mark.parametrize("hw", [(66, 64), (64, 62), (30, 30)])
def test_size_not_multiple_of_4_is_refused(hw):
    with pytest.raises(NotImplementedError, match="multiples of 4"):
        Generator(3, 1, 3)(torch.zeros(1, 3, *hw))


def test_missing_checkpoint_raises_without_network(tmp_path, monkeypatch):
    def no_network(*args, **kwargs):
        raise AssertionError("LineartDetector tried to open a socket")
    monkeypatch.setattr(socket, "socket", no_network)
    monkeypatch.setattr(socket, "create_connection", no_network)
    with pytest.raises(FileNotFoundError) as e:
        LineartDetector(ckpt_dir=str(tmp_path))
    assert str(tmp_path / "sk_model.pth") in str(e.value)


def test_subpixel_phases_recompose_conv_transpose():
    """ConvTranspose2d(3, stride 2, padding 1, output_padding 1) equals, at output phase (py, px), the sum over
    phase_taps of the input shifted by (dy, dx) (zero outside) through kernel tap (ky, kx)"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 6, 5, 7, generator=g, dtype=torch.float64)
    w = torch.randn(6, 4, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, w, stride=2, padding=1, output_padding=1)
    xp = F.pad(x, (0, 1, 0, 1))
    h, wd = x.shape[2:]
    for py in (0, 1):
        for px in (0, 1):
            acc = torch.zeros(2, 4, h, wd, dtype=torch.float64)
            for dy, dx, ky, kx in phase_taps(py, px):
                acc += torch.einsum("bihw,io->bohw", xp[:, :, dy:dy + h, dx:dx + wd], w[:, :, ky, kx])
            torch.testing.assert_close(acc, ref[:, :, py::2, px::2], rtol=1e-12, atol=1e-12)
    assert [len(phase_taps(py, px)) for py in (0, 1) for px in (0, 1)] == [1, 2, 2, 4]
