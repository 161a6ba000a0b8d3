"""OpenPose body annotator, host side: module tree and checkpoint mapping, the no-ReLU list, the resampling tables
against cv2.resize, the Gaussian against scipy, the network input, and the host matching, assembly and drawing against
the reference's fixture.  No GPU needed."""
import os
import socket

import cv2
import numpy as np
import pytest
import scipy.ndimage
import torch

from golden_io import load_golden
import openpose_golden as og
from ctrlora_b200.annotator import openpose as op

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "openpose_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def test_state_dict_keys_and_strict_load(golden):
    model = op.bodypose_model()
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == [tuple(e) for e in golden["keys"]]
    # body_pose_model.pth stores each conv under its own name (no block prefix)
    sd = og.weights({k: tuple(v.shape) for k, v in model.state_dict().items()})
    ckpt = {k.split(".", 1)[1]: v for k, v in sd.items()}
    assert len(ckpt) == len(sd)
    model.load_state_dict(op.checkpoint_state_dict(model, ckpt), strict=True)
    assert torch.equal(model.model6_2.Mconv7_stage6_L2.bias, sd["model6_2.Mconv7_stage6_L2.bias"])


def test_no_relu_list():
    model = op.bodypose_model()
    relu_after = {}
    for block, seq in model.named_children():
        names = [n for n, _ in seq.named_children()]
        for i, (n, m) in enumerate(seq.named_children()):
            if isinstance(m, torch.nn.Conv2d):
                relu_after[n] = i + 1 < len(names) and names[i + 1] == f"relu_{n}"
    no_relu = sorted(n for n, r in relu_after.items() if not r)
    assert no_relu == sorted(["conv5_5_CPM_L1", "conv5_5_CPM_L2"] +
                             [f"Mconv7_stage{s}_L{b}" for s in range(2, 6) for b in (1, 2)] + ["Mconv7_stage6_L1"])
    assert relu_after["Mconv7_stage6_L2"], "the reference ReLUs stage 6's heatmaps (its list names L1 twice)"
    assert op.no_relu_layers().count("Mconv7_stage6_L1") == 2


def _sizes():
    return [og.NET_SIZES[s] for s in og.NET_SIZES] + [og.PP_CASES[c]["size"] for c in og.PP_CASES]


@pytest.mark.parametrize("size", _sizes(), ids=lambda s: f"{s[0]}x{s[1]}")
def test_resize_tables_match_cv2(size):
    """each single resize (x8 LANCZOS4; the second one LANCZOS4 or INTER_AREA) and their composition per axis against
    cv2.resize on float32 maps"""
    h, w = size
    rh, rw, ph, pw = op.geometry(h, w)
    h8, w8 = ph // 8, pw // 8
    rs = np.random.RandomState(h * 1000 + w)
    m = rs.uniform(-1, 1, (h8, w8)).astype(np.float32)
    up = cv2.resize(m, (pw, ph), interpolation=cv2.INTER_LANCZOS4)
    up_t = op.resize_matrix(h8, ph, cv2.INTER_LANCZOS4) @ m @ op.resize_matrix(w8, pw, cv2.INTER_LANCZOS4).T
    assert np.abs(up_t - up).max() < 1e-5
    crop = up[:rh, :rw]
    interp = op.resize_interp(rh, rw, h, w)
    out = cv2.resize(crop, (w, h), interpolation=interp)
    shrink = h <= rh and w <= rw
    out_t = op.resize_matrix(rh, h, interp, shrink) @ crop.astype(np.float64) @ op.resize_matrix(rw, w, interp, shrink).T
    assert np.abs(out_t - out).max() < 1e-5
    a, b = op.axis_matrices(h, w)
    assert np.abs(a @ m.astype(np.float64) @ b.T - out).max() < 1e-5
    (ys, yw), (xs, xw) = op.band(a), op.band(b)
    full = np.zeros_like(a)
    for y in range(h):
        full[y, ys[y]:ys[y] + yw.shape[1]] = yw[y]
    assert np.array_equal(full, a) and yw.shape[1] <= h8 and xw.shape[1] <= w8


@pytest.mark.parametrize("ratio", [(23, 40), (40, 23), (23, 7), (184, 512), (184, 120), (1472, 100)])
def test_area_and_lanczos_rules(ratio):
    """INTER_AREA (shrinking both axes, and its linear rule otherwise) and LANCZOS4 along one axis of a 2-D resize"""
    src, dst = ratio
    m = np.random.RandomState(src + dst).uniform(-1, 1, (src, 5)).astype(np.float32)
    for interp in (cv2.INTER_AREA, cv2.INTER_LANCZOS4):
        other = 3 if interp == cv2.INTER_AREA and dst < src else 7  # a second axis that shrinks / grows with the first
        ref = cv2.resize(m, (other, dst), interpolation=interp)
        shrink = dst <= src and other <= 5
        got = op.resize_matrix(src, dst, interp, shrink) @ m @ op.resize_matrix(5, other, interp, shrink).T
        assert np.abs(got - ref).max() < 1e-5, interp


def test_gaussian_weights_match_scipy():
    w = op.gaussian_weights()
    assert len(w) == 13
    delta = np.zeros(25)
    delta[12] = 1.0
    impulse = scipy.ndimage.gaussian_filter1d(delta, 3.0)
    assert np.array_equal(impulse[12:], w) and np.array_equal(impulse[:13][::-1], w)


@pytest.mark.parametrize("size", list(og.NET_SIZES))
def test_network_input(golden, size):
    g = golden[f"net.{size}"]
    img = og.image(size)
    x = op.network_input(img)
    padded = g["padded"].numpy()
    assert x.shape == (1, 3) + padded.shape[:2]
    ref = np.transpose(np.float32(padded[:, :, :, None]), (3, 2, 0, 1)) / 256 - 0.5
    assert np.array_equal(x, ref)
    assert np.array_equal(x.astype(np.float16).astype(np.float32), x)  # exact in fp16


def _limb_candidates(g):
    cands = [None] * len(op.LIMB_PARTS)
    for k, rows in g["limb_candidates"].items():
        cands[k] = [(int(i), int(j), float(s)) for i, j, s in rows.tolist()]
    return cands


@pytest.mark.parametrize("case", list(og.PP_CASES))
def test_host_assembly_and_drawing_match_reference(golden, case):
    g = golden[f"pp.{case}"]
    h, w = og.PP_CASES[case]["size"]
    cand_ref = g["candidate"].numpy()
    candidate = op.make_candidate(cand_ref[:, 0].astype(int), cand_ref[:, 1].astype(int), cand_ref[:, 2])
    assert np.array_equal(candidate, cand_ref)
    subset = op.assemble(candidate, g["counts"].numpy(), _limb_candidates(g))
    assert np.array_equal(subset, g["subset"].numpy())
    pose = op.pose_dict(candidate, subset, h, w)
    assert pose == g["pose"]
    assert np.array_equal(op.draw_body(pose, h, w), g["canvas"].numpy())


def test_empty_candidate_stays_1d():
    candidate = op.make_candidate([], [], [])
    assert candidate.shape == (0,)
    subset = op.assemble(candidate, np.zeros(18, np.int64), [None] * len(op.LIMB_PARTS))
    pose = op.pose_dict(candidate, subset, 64, 48)
    assert pose == {"bodies": {"candidate": [], "subset": []}, "hands": [], "faces": []}
    assert not op.draw_body(pose, 64, 48).any()


def test_missing_checkpoint_and_hand_and_face(tmp_path, monkeypatch):
    def no_network(*a, **k):
        raise AssertionError("the detector must not open a network connection")
    monkeypatch.setattr(socket.socket, "connect", no_network)
    with pytest.raises(FileNotFoundError, match=str(tmp_path / "body_pose_model.pth")):
        op.OpenposeDetector(ckpt_dir=str(tmp_path), device="cpu")
    det = op.OpenposeDetector.__new__(op.OpenposeDetector)
    with pytest.raises(NotImplementedError):
        det(np.zeros((64, 64, 3), np.uint8), hand_and_face=True)
