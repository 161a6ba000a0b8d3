"""The OpenPose body annotator (annotator/openpose: bodypose_model, Body and OpenposeDetector) on the sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.openpose import OpenposeDetector`.
`bodypose_model` keeps the reference's module tree (model0, model1_1 ... model6_2, each a Sequential of named convs,
ReLUs and pools), so `state_dict()` equals the reference's and body_pose_model.pth loads with strict=True through
`checkpoint_state_dict` (each model key is the checkpoint key behind its first component).  The nn modules only hold
the parameters; forward runs:

- conv1_1 (K = 27): a zero-masked 3x3 tap gather from the fp32 NCHW input (padded to K = 32) and one 1x1
  ctrlora_gemm_f16 with the bias and the ReLU in its epilogue, as HED's first conv;
- every other 3x3 / 7x7 / 1x1 conv (+ ReLU): one implicit ctrlora_gemm_f16 (zero padding is the TMA out-of-bounds fill)
  with the bias (and the ReLU) in its epilogue;
- the three 2x2 max pools: ctrlora_hed_side_pool_f16 without its projection (ops.max_pool2x2);
- each stage's cat([L1, L2, out1]) (185 channels): no copy.  Its producers write straight into one 192-wide fp16
  pixel-major buffer: out1 at columns 0..127, L1 at 128..167 (38 + 2 zero columns), L2 at 168..191 (19 + 5).  The next
  stage's Mconv1 weights are permuted and zero-padded to that order at prepare time, and both branches' Mconv1 (they
  read the same input) run as one N = 256 launch;
- stage 6's Mconv7 outputs are stored in fp32.

Body's post-process runs on the device through openpose_sm90.cu: the two resizes of the stride-8 maps as one banded
float64 table per axis (`axis_matrices`, `band`), the float64 Gaussian of the 18 part maps, the peaks compacted in the
reference's order, and the scores of every candidate limb.  The host keeps the input resize and padding, the greedy
matching, the assembly of people and the drawing, with the reference's float64 expressions.

Activations are fp16 pixel-major with fp32 accumulation (x / 256 - 0.5 of a uint8 image is exact in fp16).  Inference
only, on the current stream.
"""
import collections
import math
import os

import cv2
import numpy as np
import torch
import torch.nn as nn

from .. import ops, prepare
from .common import TAPS3, SizeCache, checkpoint_path, device_input, freeze, linear_src_coord

BOXSIZE, STRIDE, PAD_VALUE = 368, 8, 128
SCALE_SEARCH = 0.5          # the reference's single scale
THRE_PEAK, THRE_PAF = 0.1, 0.05
MID_NUM = 10                # PAF samples per candidate limb
SIGMA, TRUNCATE = 3.0, 4.0  # gaussian_filter(sigma=3) with scipy's default truncate
TABLE_CACHE_SIZES = 8       # image sizes whose device resample tables are kept (least recently used goes first)
CAT_WIDTH, L1_COL, L2_COL = 192, 128, 168  # the stage input buffer: out1 | L1 (38 -> 40) | L2 (19 -> 24)
PAF_PAD, HEAT_PAD = 40, 24
N_PARTS = 18

# limbs as (part A, part B) 1-based, and their PAF channels as 1-based network output indices (19 = first PAF channel)
LIMB_PARTS = ((2, 3), (2, 6), (3, 4), (4, 5), (6, 7), (7, 8), (2, 9), (9, 10), (10, 11), (2, 12), (12, 13), (13, 14),
              (2, 1), (1, 15), (15, 17), (1, 16), (16, 18), (3, 17), (6, 18))
LIMB_PAF = ((31, 32), (39, 40), (33, 34), (35, 36), (41, 42), (43, 44), (19, 20), (21, 22), (23, 24), (25, 26), (27, 28),
            (29, 30), (47, 48), (49, 50), (53, 54), (51, 52), (55, 56), (37, 38), (45, 46))
COLORS = ((255, 0, 0), (255, 85, 0), (255, 170, 0), (255, 255, 0), (170, 255, 0), (85, 255, 0), (0, 255, 0),
          (0, 255, 85), (0, 255, 170), (0, 255, 255), (0, 170, 255), (0, 85, 255), (0, 0, 255), (85, 0, 255),
          (170, 0, 255), (255, 0, 255), (255, 0, 170), (255, 0, 85))
STICK_WIDTH = 4


# ------------------------------------------------------------------------------------------------ network
def _trunk_spec():
    """model0: (name, cin, cout, k) convs and pool names"""
    spec = [("conv1_1", 3, 64, 3), ("conv1_2", 64, 64, 3), "pool1_stage1",
            ("conv2_1", 64, 128, 3), ("conv2_2", 128, 128, 3), "pool2_stage1"]
    spec += [(f"conv3_{i}", 128 if i == 1 else 256, 256, 3) for i in range(1, 5)] + ["pool3_stage1"]
    return spec + [("conv4_1", 256, 512, 3), ("conv4_2", 512, 512, 3), ("conv4_3_CPM", 512, 256, 3),
                   ("conv4_4_CPM", 256, 128, 3)]


def _stage_spec(stage, branch):
    """model{stage}_{branch}: the convs of one branch (branch 1: 38 PAF channels, branch 2: 19 heatmaps)"""
    out = 38 if branch == 1 else 19
    if stage == 1:
        return [(f"conv5_{i}_CPM_L{branch}", 128, 128, 3) for i in (1, 2, 3)] + [
            (f"conv5_4_CPM_L{branch}", 128, 512, 1), (f"conv5_5_CPM_L{branch}", 512, out, 1)]
    return [(f"Mconv{i}_stage{stage}_L{branch}", 185 if i == 1 else 128, 128, 7) for i in range(1, 6)] + [
        (f"Mconv6_stage{stage}_L{branch}", 128, 128, 1), (f"Mconv7_stage{stage}_L{branch}", 128, out, 1)]


def no_relu_layers():
    """The convs without a ReLU, as the reference lists them: each branch's last conv of stages 1-5, and of stage 6
    only L1 (the reference names Mconv7_stage6_L1 twice and Mconv7_stage6_L2 never, so stage 6's heatmaps are ReLU'd)"""
    names = [f"conv5_5_CPM_L{b}" for b in (1, 2)]
    names += [f"Mconv7_stage{s}_L{b}" for s in range(2, 6) for b in (1, 2)]
    return names + ["Mconv7_stage6_L1", "Mconv7_stage6_L1"]


def _sequential(spec, no_relu):
    layers = []
    for item in spec:
        if isinstance(item, str):
            layers.append((item, nn.MaxPool2d(kernel_size=2, stride=2, padding=0)))
            continue
        name, cin, cout, k = item
        layers.append((name, nn.Conv2d(cin, cout, kernel_size=k, stride=1, padding=(k - 1) // 2)))
        if name not in no_relu:
            layers.append((f"relu_{name}", nn.ReLU(inplace=True)))
    return nn.Sequential(collections.OrderedDict(layers))


def checkpoint_state_dict(model, ckpt):
    """body_pose_model.pth's tensors under the model's keys: a model key is `<block>.<checkpoint key>`"""
    return {k: ckpt[k.split(".", 1)[1]] for k in model.state_dict()}


class bodypose_model(nn.Module):
    """The reference's body network with its parameters; forward(x fp32 [B, 3, h, w], h and w multiples of 8) ->
    (PAFs fp32 [B, 38, h / 8, w / 8], heatmaps fp32 [B, 19, h / 8, w / 8]), the reference's (out6_1, out6_2).

    split_k: passed to every GEMM (0 lets the tile model choose; 1 pins one plan per row, so a batch of B equals B
    batches of 1 bit for bit)."""

    def __init__(self):
        super().__init__()
        no_relu = set(no_relu_layers())
        self.model0 = _sequential(_trunk_spec(), no_relu)
        for b in (1, 2):  # the reference's registration order: model1_1 ... model6_1, then model1_2 ... model6_2
            for s in range(1, 7):
                setattr(self, f"model{s}_{b}", _sequential(_stage_spec(s, b), no_relu))
        freeze(self)
        self.__dict__["_no_relu"] = no_relu

    def branch(self, stage, b):
        return getattr(self, f"model{stage}_{b}")

    # ---- kernel-layout weights
    def _conv(self, name, conv, pad_out=None):
        """(fp16 [Cout(pad), taps, Cin], fp32 bias [Cout(pad)]); conv1_1 flat [64, 1, 32] (K zero-padded from 27) for
        the tap gather"""
        def build():
            if name == "conv1_1":
                w = prepare.flat_conv_weight(conv.weight, 32)
            else:
                w = prepare.conv_weight(conv.weight, pad_out=pad_out)
            bias = torch.zeros(w.shape[0], device=w.device, dtype=torch.float32)
            bias[:conv.out_channels] = conv.bias.detach().float()
            return w, bias
        return self._prep.get(name, [conv.weight, conv.bias], build)

    def _pair(self, stage):
        """both branches' first conv of a stage as one N = 256 launch: fp16 [256, taps, Cin], fp32 [256].  Stages 2-6
        read the 192-wide buffer, so their input channels (L1 0..37, L2 38..56, out1 57..184 in the reference's cat)
        are permuted to out1 | L1 | L2 at columns 0 / 128 / 168, with zero weights on the padding columns."""
        c1, c2 = self.branch(stage, 1)[0], self.branch(stage, 2)[0]

        def build():
            ws = []
            for conv in (c1, c2):
                w = prepare.conv_weight(conv.weight)
                if stage > 1:
                    full = torch.zeros((w.shape[0], w.shape[1], CAT_WIDTH), device=w.device, dtype=torch.float16)
                    full[:, :, :128] = w[:, :, 57:185]
                    full[:, :, L1_COL:L1_COL + 38] = w[:, :, 0:38]
                    full[:, :, L2_COL:L2_COL + 19] = w[:, :, 38:57]
                    w = full
                ws.append(w)
            return torch.cat(ws).contiguous(), torch.cat([prepare.bias_f32(c1.bias), prepare.bias_f32(c2.bias)])
        return self._prep.get(f"pair{stage}", [c1.weight, c1.bias, c2.weight, c2.bias], build)

    def _check(self, x):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"input must be [B, 3, H, W], got {tuple(x.shape)}")
        h, w = x.shape[2], x.shape[3]
        if h % STRIDE or w % STRIDE or h < STRIDE or w < STRIDE:
            raise ValueError(f"{h} x {w}: H and W must be positive multiples of {STRIDE} (Body pads the image so)")
        return device_input(self, x, self.model0.conv1_1.weight)

    def _gemm(self, x, conv, name, out=None, out_f32=False, pad_out=None):
        w, b = self._conv(name, conv, pad_out)
        run = ops.gemm if name in self._no_relu else ops.gemm_relu
        return run(x, w, ksize=conv.kernel_size[0], bias=b, out=out, out_f32=out_f32, split_k=self.split_k)

    def run_maps(self, x):
        """(PAFs fp32 pixel-major [B, h / 8, w / 8, 40], heatmaps fp32 [B, h / 8, w / 8, 24]); the columns past 38 / 19
        are zero"""
        x = self._check(x)
        h = None
        for name, m in self.model0.named_children():
            if isinstance(m, nn.MaxPool2d):
                h = ops.max_pool2x2(h)
            elif isinstance(m, nn.Conv2d):
                if name == "conv1_1":
                    w, b = self._conv(name, m)
                    h = ops.gemm_relu(ops.tap_gather(x, TAPS3, reflect=False, k_pad=w.shape[-1]), w, bias=b,
                                      split_k=self.split_k)
                elif name == "conv4_4_CPM":
                    cat = torch.empty(h.shape[:3] + (CAT_WIDTH,), device=h.device, dtype=torch.float16)
                    self._gemm(h, m, name, out=cat[..., :128])
                else:
                    h = self._gemm(h, m, name)
        out1 = cat[..., :128]
        paf = torch.empty(cat.shape[:3] + (PAF_PAD,), device=cat.device, dtype=torch.float32)
        heat = torch.empty(cat.shape[:3] + (HEAT_PAD,), device=cat.device, dtype=torch.float32)
        for s in range(1, 7):
            w, b = self._pair(s)
            both = ops.gemm_relu(out1 if s == 1 else cat, w, ksize=3 if s == 1 else 7, bias=b, split_k=self.split_k)
            for br, (col, n_pad, final) in ((1, (L1_COL, PAF_PAD, paf)), (2, (L2_COL, HEAT_PAD, heat))):
                t = both[..., (br - 1) * 128:br * 128]
                convs = list(self.branch(s, br).named_children())
                convs = [(n, m) for n, m in convs if isinstance(m, nn.Conv2d)][1:]
                for i, (name, m) in enumerate(convs):
                    if i < len(convs) - 1:
                        t = self._gemm(t, m, name)
                    elif s < 6:
                        self._gemm(t, m, name, out=cat[..., col:col + n_pad], pad_out=n_pad)
                    else:
                        self._gemm(t, m, name, out=final, out_f32=True, pad_out=n_pad)
        return paf, heat

    @torch.no_grad()
    def forward(self, x):
        paf, heat = self.run_maps(x)
        return ops.nhwc_to_nchw_f32(paf, channels=38), ops.nhwc_to_nchw_f32(heat, channels=19)


# ------------------------------------------------------------------------------------------------ resampling tables
def _src_coord(dst, src, area_linear):
    """cv2.resize's (sx, fx) per output index along one axis: the generic rule (common.linear_src_coord), or INTER_AREA's
    rule when it does not shrink both axes: sx = floor(d * scale), fx = (float)((d + 1) - (sx + 1) / scale) wrapped to
    [0, 1).  scale = 1 / (dst / src) in float64."""
    if not area_linear:
        return linear_src_coord(src, dst)
    inv = dst / src
    scale = 1.0 / inv
    d = np.arange(dst, dtype=np.float64)
    sx = np.floor(d * scale).astype(np.int64)
    fx = ((d + 1) - (sx + 1) * inv).astype(np.float32)
    fx = np.where(fx <= 0, np.float32(0), fx - np.floor(fx)).astype(np.float32)
    return sx, fx


def _lanczos4_coeffs(fx):
    """cv2's 8 LANCZOS4 weights for fractional offsets fx (float32 [n]): sin-based terms in float64 rounded to float32,
    normalised by their float32 sum; offset 0 (a tap on the sample) gets weight 1"""
    s45 = 0.70710678118654752440084436210485
    cs = ((1, 0), (-s45, -s45), (0, 1), (s45, -s45), (-1, 0), (s45, s45), (0, -1), (-s45, s45))
    x3 = (fx + np.float32(3)).astype(np.float32)
    y0 = -x3.astype(np.float64) * math.pi * 0.25
    s0, c0 = np.sin(y0), np.cos(y0)
    coef = np.empty((fx.size, 8), np.float32)
    for i in range(8):
        yi = (x3 - np.float32(i)).astype(np.float32)
        y = -yi.astype(np.float64) * math.pi * 0.25
        with np.errstate(divide="ignore", invalid="ignore"):
            v = ((cs[i][0] * s0 + cs[i][1] * c0) / (y * y)).astype(np.float32)
        coef[:, i] = np.where(np.abs(yi) >= np.float32(1e-6), v, np.float32(1e30))
    total = np.zeros(fx.size, np.float32)
    for i in range(8):
        total = (total + coef[:, i]).astype(np.float32)
    return (coef * (np.float32(1) / total)[:, None]).astype(np.float32)


def resize_matrix(src, dst, interp, shrink_both=True):
    """cv2.resize along one axis as a float64 [dst, src] matrix (float32 coefficients).  interp: cv2.INTER_LANCZOS4 or
    cv2.INTER_AREA; shrink_both: for INTER_AREA, whether the call shrinks both axes (cv2 then averages cells; otherwise
    it interpolates linearly with its area rule).  Taps past the border clamp to the edge sample, as cv2's resize does."""
    m = np.zeros((dst, src), np.float64)
    rows = np.arange(dst)
    if interp == cv2.INTER_LANCZOS4:
        sx, fx = _src_coord(dst, src, False)
        coef = _lanczos4_coeffs(fx)
        for k in range(8):
            np.add.at(m, (rows, np.clip(sx - 3 + k, 0, src - 1)), coef[:, k].astype(np.float64))
        return m
    assert interp == cv2.INTER_AREA
    scale = src / dst
    if not shrink_both or scale < 1:
        sx, fx = _src_coord(dst, src, True)
        edge = sx >= src - 1
        fx = np.where(sx < 0, np.float32(0), fx)
        sx = np.maximum(sx, 0)
        fx = np.where(edge, np.float32(0), fx)
        sx = np.where(edge, src - 1, sx)
        np.add.at(m, (rows, sx), (np.float32(1) - fx).astype(np.float32).astype(np.float64))
        np.add.at(m, (rows, np.minimum(sx + 1, src - 1)), fx.astype(np.float64))
        return m
    scale = 1.0 / (dst / src)
    for d in range(dst):  # each output cell covers [d * scale, (d + 1) * scale) of the source
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, src - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, src - 1)
        s1 = min(s1, s2)
        if s1 - f1 > 1e-3:
            m[d, s1 - 1] += float(np.float32((s1 - f1) / cell))
        for s in range(s1, s2):
            m[d, s] += float(np.float32(1.0 / cell))
        if f2 - s2 > 1e-3:
            m[d, s2] += float(np.float32(min(min(f2 - s2, 1.0), cell) / cell))
    return m


def resize_interp(ho, wo, ht, wt):
    """util.smart_resize's choice: INTER_AREA when (Ht + Wt) / (Ho + Wo) < 1, else INTER_LANCZOS4"""
    return cv2.INTER_AREA if float(ht + wt) / float(ho + wo) < 1 else cv2.INTER_LANCZOS4


def geometry(h, w):
    """(resized h, resized w, padded h, padded w) of Body's network input for an h x w image"""
    scale = SCALE_SEARCH * BOXSIZE / h
    rh, rw = int(h * scale), int(w * scale)
    return rh, rw, rh + (-rh) % STRIDE, rw + (-rw) % STRIDE


def axis_matrices(h, w):
    """(rows float64 [h, h8], columns float64 [w, w8]): the stride-8 maps -> x8 (LANCZOS4) -> crop to the resized image
    -> h x w (smart_resize), composed per axis"""
    rh, rw, ph, pw = geometry(h, w)
    interp = resize_interp(rh, rw, h, w)
    shrink = h <= rh and w <= rw
    mats = []
    for n, r, p in ((h, rh, ph), (w, rw, pw)):
        up = resize_matrix(p // STRIDE, p, cv2.INTER_LANCZOS4)[:r]
        mats.append(resize_matrix(r, n, interp, shrink) @ up)
    return mats


def band(m):
    """a banded [n, src] matrix -> (int32 [n] starts, float64 [n, t] weights): row i is m[i, s_i : s_i + t]"""
    nz = m != 0
    first = nz.argmax(axis=1)
    last = m.shape[1] - 1 - nz[:, ::-1].argmax(axis=1)
    t = int((last - first).max()) + 1
    start = np.clip(first, 0, m.shape[1] - t)
    idx = start[:, None] + np.arange(t)[None, :]
    return start.astype(np.int32), np.take_along_axis(m, idx, axis=1)


def gaussian_weights(sigma=SIGMA, truncate=TRUNCATE):
    """scipy's gaussian_filter1d kernel (order 0) from the centre tap outwards: exp(-0.5 / sigma^2 * x^2) over x in
    [-r, r], r = int(truncate * sigma + 0.5), divided by its sum"""
    r = int(truncate * float(sigma) + 0.5)
    x = np.arange(-r, r + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    phi = phi / phi.sum()
    return phi[r:]


# ------------------------------------------------------------------------------------------------ host steps
def network_input(ori_img):
    """Body's input: the image scaled to height 184 (one cv2.resize on uint8), padded right / down to multiples of 8
    with 128, as fp32 [1, 3, h, w] = x / 256 - 0.5 (channel order as given)"""
    h, w = ori_img.shape[:2]
    rh, rw, ph, pw = geometry(h, w)
    img = cv2.resize(ori_img, (rw, rh), interpolation=resize_interp(h, w, rh, rw))
    padded = np.full((ph, pw, 3), PAD_VALUE, np.uint8)
    padded[:rh, :rw] = img
    return np.ascontiguousarray(padded.astype(np.float32).transpose(2, 0, 1)[None] / 256 - 0.5)


def match_limb(cand, n_a, n_b, peak_ids_a, peak_ids_b):
    """The greedy matching of one limb: cand = [(i, j, score)] of the pairs that passed both criteria, in (i, j)
    order.  Stable sort by score, descending; take a pair when neither end is taken, until min(nA, nB) are.
    Returns float64 [n, 5] rows (id A, id B, score, i, j)."""
    order = sorted(range(len(cand)), key=lambda c: cand[c][2], reverse=True)
    rows, used_a, used_b = [], set(), set()
    for c in order:
        i, j, s = cand[c]
        if i in used_a or j in used_b:
            continue
        rows.append([peak_ids_a[i], peak_ids_b[j], s, i, j])
        used_a.add(i)
        used_b.add(j)
        if len(rows) >= min(n_a, n_b):
            break
    return np.array(rows, dtype=np.float64).reshape(-1, 5)


def assemble(candidate, part_counts, limb_candidates):
    """People from the matched limbs, as Body.__call__ builds them (body.py :140-197).  candidate: float64 [N, 4] (x, y,
    score, id; the peaks of part 0, then part 1, ...) or the empty 1-D array; part_counts: the number of peaks of each
    part; limb_candidates[k]: None when part A or part B of limb k has no peak, else the (i, j, score) list of its pairs
    that passed both criteria, in (i, j) order.  Returns float64 [n, 20] rows: the candidate index of each of the 18
    parts (-1: none), the total score, the number of parts.  People with fewer than 4 parts or a mean score below 0.4
    are dropped."""
    first = np.concatenate([[0], np.cumsum(part_counts)]).astype(np.int64)
    people = -1 * np.ones((0, 20))
    for k, cand in enumerate(limb_candidates):
        if cand is None:
            continue
        a, b = LIMB_PARTS[k][0] - 1, LIMB_PARTS[k][1] - 1
        ids_a = np.arange(first[a], first[a + 1])
        ids_b = np.arange(first[b], first[b + 1])
        for pa, pb, s, _, _ in match_limb(cand, len(ids_a), len(ids_b), ids_a, ids_b):
            hits = [n for n in range(len(people)) if people[n][a] == pa or people[n][b] == pb]
            if len(hits) > 2:
                raise IndexError("a limb's ends belong to more than two people (the reference fails here too)")
            shared = len(hits) == 2 and np.any((people[hits[0]] >= 0)[:-2] & (people[hits[1]] >= 0)[:-2])
            if len(hits) == 1 or shared:  # extend the first person (always when the two people share a part)
                p = people[hits[0]]
                if shared or p[b] != pb:
                    p[b] = pb
                    p[-1] += 1
                    p[-2] += candidate[int(pb), 2] + s
            elif len(hits) == 2:  # two disjoint people joined by this limb: merge them
                p, q = people[hits[0]], people[hits[1]]
                p[:-2] += q[:-2] + 1
                p[-2:] += q[-2:]
                p[-2] += s
                people = np.delete(people, hits[1], 0)
            elif k < 17:  # a new person (the last two limbs, shoulder-ear, never start one)
                new = -1 * np.ones(20)
                new[a], new[b] = pa, pb
                new[-1] = 2
                new[-2] = sum(candidate[np.array([pa, pb]).astype(int), 2]) + s
                people = np.vstack([people, new])
    drop = [n for n in range(len(people)) if people[n][-1] < 4 or people[n][-2] / people[n][-1] < 0.4]
    return np.delete(people, drop, axis=0)


def make_candidate(px, py, score):
    """Body's candidate array from the peaks in id order: float64 [N, 4] (x, y, score, id), or the empty 1-D array"""
    if len(px) == 0:
        return np.array([])
    n = len(px)
    return np.stack([np.asarray(px, np.float64), np.asarray(py, np.float64), np.asarray(score, np.float64),
                     np.arange(n, dtype=np.float64)], axis=1)


def pose_dict(candidate, subset, h, w):
    """OpenposeDetector's pose: candidate x / W, y / H (a 2-D candidate only; an empty one stays as it is), empty hands
    and faces"""
    if candidate.ndim == 2 and candidate.shape[1] == 4:
        candidate = candidate[:, :2].copy()
        candidate[:, 0] /= float(w)
        candidate[:, 1] /= float(h)
    return dict(bodies=dict(candidate=candidate.tolist(), subset=subset.tolist()), hands=[], faces=[])


def draw_body(pose, h, w):
    """The reference's body drawing on a black h x w x 3 canvas: an ellipse per limb of each person (cv2.ellipse2Poly
    + fillConvexPoly), the canvas x 0.6, then a filled circle per part.  Pixel positions are recomputed from the
    normalised candidate as the reference does (x * W, int truncation), so the canvas is the reference's bit for bit."""
    canvas = np.zeros((h, w, 3), np.uint8)
    cand = np.array(pose["bodies"]["candidate"])
    subset = np.array(pose["bodies"]["subset"])
    for k in range(17):
        for person in subset:
            idx = person[np.array(LIMB_PARTS[k]) - 1]
            if -1 in idx:
                continue
            px = cand[idx.astype(int), 0] * float(w)
            py = cand[idx.astype(int), 1] * float(h)
            my, mx = np.mean(px), np.mean(py)
            length = ((py[0] - py[1]) ** 2 + (px[0] - px[1]) ** 2) ** 0.5
            angle = math.degrees(math.atan2(py[0] - py[1], px[0] - px[1]))
            poly = cv2.ellipse2Poly((int(my), int(mx)), (int(length / 2), STICK_WIDTH), int(angle), 0, 360, 1)
            cv2.fillConvexPoly(canvas, poly, COLORS[k])
    canvas = (canvas * 0.6).astype(np.uint8)
    for part in range(N_PARTS):
        for person in subset:
            i = int(person[part])
            if i == -1:
                continue
            x, y = cand[i][0:2]
            cv2.circle(canvas, (int(x * w), int(y * h)), 4, COLORS[part], thickness=-1)
    return canvas


# ------------------------------------------------------------------------------------------------ device post-process
class PostProcess:
    """Body's post-process of one image's stride-8 maps on the device; keeps the resample tables of the last
    TABLE_CACHE_SIZES image sizes"""

    def __init__(self):
        self._tables = SizeCache(TABLE_CACHE_SIZES)
        self._gauss = gaussian_weights()

    def tables(self, h, w, device):
        def build():
            (ys, yw), (xs, xw) = [band(m) for m in axis_matrices(h, w)]
            return tuple(torch.from_numpy(np.ascontiguousarray(t)).to(device) for t in (ys, yw, xs, xw))
        return self._tables.fetch((h, w, str(device)), build)

    def peaks(self, heat_px, h, w):
        """(heatmaps fp32 [18, h, w], smoothed float64 [18, h, w], device peaks (x, y, part, score))"""
        tabs = self.tables(h, w, heat_px.device)
        heat = ops.openpose_resample(heat_px, tabs, N_PARTS)
        smooth = ops.openpose_smooth(heat, self._gauss)
        return heat, smooth, ops.openpose_peaks(smooth, heat, THRE_PEAK)

    def __call__(self, paf_px, heat_px, h, w):
        """(candidate, subset) of one image: paf_px / heat_px fp32 pixel-major [h8, w8, ld] (38 PAF / 19 heatmap
        channels first), for an h x w image"""
        _, _, (px, py, part, score) = self.peaks(heat_px, h, w)
        part_h = part.cpu().numpy()
        counts = np.bincount(part_h, minlength=N_PARTS) if len(part_h) else np.zeros(N_PARTS, np.int64)
        first = np.concatenate([[0], np.cumsum(counts)])
        limbs, ranges, pairs = [], [], 0
        for k, ((a, b), (cx, cy)) in enumerate(zip(LIMB_PARTS, LIMB_PAF)):
            n_a, n_b = int(counts[a - 1]), int(counts[b - 1])
            if n_a and n_b:
                limbs.append((pairs, int(first[a - 1]), n_a, int(first[b - 1]), n_b, cx - 19, cy - 19))
                ranges.append((k, pairs, n_a, n_b))
                pairs += n_a * n_b
        limb_candidates = [None] * len(LIMB_PARTS)
        if limbs:
            sc, ok = ops.openpose_limbs(paf_px, self.tables(h, w, paf_px.device), px, py, limbs, h, THRE_PAF)
            sc, ok = sc.cpu().numpy(), ok.cpu().numpy()
            for k, base, n_a, n_b in ranges:
                limb_candidates[k] = [(q // n_b, q % n_b, float(sc[base + q])) for q in range(n_a * n_b)
                                      if ok[base + q]]
        candidate = make_candidate(px.cpu().numpy(), py.cpu().numpy(), score.cpu().numpy())
        return candidate, assemble(candidate, counts, limb_candidates)


# ------------------------------------------------------------------------------------------------ public API
class Body:
    """The reference's Body: body_pose_model.pth at `model_path`; __call__(BGR uint8 image) -> (candidate float64 [N, 4]
    (x, y, score, id) or the empty 1-D array, subset float64 [n, 20])"""

    def __init__(self, model_path, device="cuda"):
        checkpoint_path(*os.path.split(model_path))
        self.model = bodypose_model()
        ckpt = torch.load(model_path, map_location="cpu", weights_only=True)
        self.model.load_state_dict(checkpoint_state_dict(self.model, ckpt), strict=True)
        self.model = self.model.to(device).eval()
        self.post = PostProcess()

    def __call__(self, ori_img):
        h, w = ori_img.shape[:2]
        x = torch.from_numpy(network_input(ori_img)).to(self.model.model0.conv1_1.weight.device)
        with torch.no_grad():
            paf, heat = self.model.run_maps(x)
        return self.post(paf[0], heat[0], h, w)


class OpenposeDetector:
    """The reference's OpenposeDetector for bodies: body_pose_model.pth from `ckpt_dir` (default: the reference's
    checkpoint directory); __call__(HWC uint8 RGB image, hand_and_face=False, return_is_index=False) -> the drawn
    uint8 canvas, or the pose dict with return_is_index.  Nothing is downloaded: a missing checkpoint raises
    FileNotFoundError with the path it was expected at.  The hand and face estimators are not provided:
    hand_and_face=True raises NotImplementedError."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        self.body_estimation = Body(checkpoint_path(ckpt_dir, "body_pose_model.pth"), device=device)

    def __call__(self, oriImg, hand_and_face=False, return_is_index=False):
        if hand_and_face:
            raise NotImplementedError("ctrlora_b200's OpenposeDetector estimates bodies only: the hand and face "
                                      "estimators are not ported (call with hand_and_face=False)")
        img = oriImg[:, :, ::-1].copy()
        h, w = img.shape[:2]
        candidate, subset = self.body_estimation(img)
        pose = pose_dict(candidate, subset, h, w)
        return pose if return_is_index else draw_body(pose, h, w)
