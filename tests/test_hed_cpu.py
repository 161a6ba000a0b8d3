"""The HED annotators' host side: the module tree against the reference's state dict, the input-size limit, the
checkpoint lookup without network access, the resize tables against cv2.resize, and the HED-sketch retry loop against
the reference's (tests/golden/hed_golden.pt)."""
import os
import socket

import cv2
import numpy as np
import pytest
import torch

from golden_io import load_golden
import hed_golden as hg
from ctrlora_b200.annotator.hed import ControlNetHED_Apache2, HEDdetector, level_sizes, resize_tables
from ctrlora_b200.annotator.hedsketch import HEDSketchDetector

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hed_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def test_state_dict_matches_reference(golden):
    """keys, order and shapes of ControlNetHED_Apache2 equal the reference's (recorded from the reference module)"""
    ours = [(k, tuple(v.shape)) for k, v in ControlNetHED_Apache2().state_dict().items()]
    assert ours == [(k, tuple(s)) for k, s in golden["keys"]]


def test_reference_weights_load_strict(golden):
    model = ControlNetHED_Apache2()
    model.load_state_dict(hg.weights({k: s for k, s in golden["keys"]}), strict=True)
    assert 90 <= float(model.norm.min()) and float(model.norm.max()) <= 150


@pytest.mark.parametrize("hw", [(15, 64), (64, 15), (8, 8)])
def test_size_below_16_is_refused(hw):
    with pytest.raises(ValueError, match="at least 16"):
        ControlNetHED_Apache2()(torch.zeros(1, 3, *hw))


def test_missing_checkpoint_raises_without_network(tmp_path, monkeypatch):
    def no_network(*args, **kwargs):
        raise AssertionError("HEDdetector tried to open a socket")
    monkeypatch.setattr(socket, "socket", no_network)
    monkeypatch.setattr(socket, "create_connection", no_network)
    with pytest.raises(FileNotFoundError) as e:
        HEDdetector(ckpt_dir=str(tmp_path))
    assert str(tmp_path / "ControlNetHED.pth") in str(e.value)
    with pytest.raises(FileNotFoundError) as e:
        HEDSketchDetector(ckpt_dir=str(tmp_path))
    assert str(tmp_path / "ControlNetHED.pth") in str(e.value)


def resize_with_tables(s, h, w):
    """the fuse kernel's bilinear resize in float32 numpy: the horizontal pass on two source rows, then the vertical"""
    ri, rf = resize_tables(s.shape[0], h)
    ci, cf = resize_tables(s.shape[1], w)
    r1, c1 = np.minimum(ri + 1, s.shape[0] - 1), np.minimum(ci + 1, s.shape[1] - 1)
    one = np.float32(1)
    t0 = s[ri][:, ci] * (one - cf) + s[ri][:, c1] * cf
    t1 = s[r1][:, ci] * (one - cf) + s[r1][:, c1] * cf
    return t0 * (one - rf)[:, None] + t1 * rf[:, None]


RATIOS = sorted({(lh, lw, h, w) for h, w in hg.SIZES.values() for lh, lw in level_sizes(h, w)[1:]})


@pytest.mark.parametrize("lh,lw,h,w", RATIOS)
def test_resize_tables_reproduce_cv2(lh, lw, h, w):
    """at every (level size -> output size) of the fixture's sizes, including the ragged 200 x 328 whose floors give
    25 x 41 and 12 x 20"""
    rs = np.random.RandomState(lh * 1000 + lw)
    s = rs.standard_normal((lh, lw)).astype(np.float32)
    ref = cv2.resize(s, (w, h), interpolation=cv2.INTER_LINEAR)
    got = resize_with_tables(s, h, w)
    assert got.dtype == np.float32
    assert np.abs(got - ref).max() < 1e-5, np.abs(got - ref).max()


def test_resize_tables_identity_and_clamps():
    idx, frac = resize_tables(7, 7)
    assert np.array_equal(idx, np.arange(7)) and not frac.any()
    idx, frac = resize_tables(12, 200)
    assert idx.min() == 0 and idx.max() == 11 and frac[0] == 0 and frac[-1] == 0
    assert ((frac >= 0) & (frac < 1)).all()


class StubHED:
    def __init__(self, m):
        self.m = m

    def __call__(self, input_image, safe=False):
        return self.m.copy()


@pytest.mark.parametrize("src,seed", [(s, n) for s in hg.SKETCH_SEEDS for n in hg.SKETCH_SEEDS[s]])
def test_hedsketch_loop_matches_reference(golden, src, seed):
    """the restated retry loop on the fixture's HED map gives the reference's sketch and leaves numpy's global RNG
    where the reference leaves it"""
    edge = golden["200x328"]["u8"].numpy()
    det = HEDSketchDetector.__new__(HEDSketchDetector)
    det.hed = StubHED(hg.dark(edge) if src == "dark" else edge)
    case = golden["sketch"][f"{src}.{seed}"]
    old = np.random.get_state()
    try:
        np.random.seed(seed)
        out = det(np.zeros(edge.shape + (3,), np.uint8))
        st = np.random.get_state()
    finally:
        np.random.set_state(old)
    assert out.dtype == np.uint8 and np.array_equal(out, case["out"].numpy())
    assert np.array_equal(st[1].astype(np.int64), case["state_keys"].numpy())
    assert (int(st[2]), (int(st[3]), float(st[4]))) == (case["state_pos"], tuple(case["state_gauss"]))


@pytest.mark.parametrize("size", list(hg.SIZES))
def test_host_post_reproduces_fixture(golden, size):
    """the tests' and the benchmark's restated host post-process gives the reference's mean and uint8 maps bit for bit
    from the reference's own side maps"""
    g = golden[size]
    sides = [hg.golden_map(golden, size, "e1").numpy()] + [g[f"e{i}"].numpy() for i in range(2, 6)]
    mean, u8 = hg.host_post(sides)
    assert np.array_equal(mean, hg.golden_map(golden, size, "mean").numpy())
    assert np.array_equal(u8, g["u8"].numpy())
    _, u8_safe = hg.host_post(sides, safe=True)
    assert np.array_equal(u8_safe, g["u8_safe"].numpy())


def test_resize_table_cache_is_bounded():
    from ctrlora_b200.annotator.hed import TABLE_CACHE_SIZES
    model = ControlNetHED_Apache2()
    sizes = [(16 + i, 40 + 2 * i) for i in range(TABLE_CACHE_SIZES + 4)]
    for h, w in sizes:
        tabs = model._resize_tables(h, w, "cpu")
        assert len(tabs) == 4 and all(idx.numel() == h + w for idx, _ in tabs)
    assert len(model._tables) == TABLE_CACHE_SIZES
    assert [k[:2] for k in model._tables] == sizes[-TABLE_CACHE_SIZES:]
    first = model._resize_tables(*sizes[-TABLE_CACHE_SIZES], "cpu")
    assert first is model._tables[sizes[-TABLE_CACHE_SIZES] + ("cpu",)]
    assert list(model._tables)[-1][:2] == sizes[-TABLE_CACHE_SIZES]
