"""Every kernel launch of the paths the benchmarked steps do not take, against a plain fp32 reference of the same call
(tests/launch_refs.py, through the shadow of tests/launch_shadow.py).

The annotators, the multi-LoRA sampling pass, the pretrain model's sampling pass and the VAE encoder are checked end to
end by their own tests: norm-relative bounds on stage outputs after up to 26 layers, or on the network's result.  An
error confined to one call -- one 128-row M tile of a 393 216-row conv, one phase of a transposed conv, the border row
of a reflect gather -- moves such a figure by less than its bound.  Here each call is compared on its own, with a
max-abs guard as a fraction of the call's own max|ref|, and named at its call site when it fails.

Scenarios: the 2-LoRA inference pass on the DDIM sampler's CFG batch with unequal LoRA weights, the pretrain model's
sampling pass with a task's LoRA set switched in, the VAE encoder at 512^2 (bench.py's random weights for these three),
and the line-art, HED and OpenPose detectors on their fixtures' synthetic weights at a 512 x 768 image and at an image
whose pixel count is not a multiple of 128.  Each scenario asserts that it took the path it claims.  The fault-injection
tests corrupt one call's result in Python and assert that the shadow reports exactly that call.  `pytest -s` prints one
line per distinct call signature with its plan and errors.
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from launch_shadow import Models, Shadow, _assert_reported, _corrupt_once, _gen, _randn, _signature  # noqa: E402
import hed_golden as hg  # noqa: E402
import lineart_golden as lg  # noqa: E402
import openpose_golden as og  # noqa: E402

pytestmark = pytest.mark.gpu
full = pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")

# 512 x 768, and a size whose pixel count is not a multiple of 128 (the line-art Generator needs multiples of 4)
SIZES = {"lineart": [(512, 768), (508, 764)], "hed": [(512, 768), (500, 740)], "openpose": [(512, 768), (500, 740)]}
T_CFG = [981, 901, 781, 641, 501, 341, 181, 21]


def _ids(size):
    return f"{size[0]}x{size[1]}"


def _has(sh, op, *texts):
    return any(o == op and all(t in shape for t in texts) for o, shape, _ in sh.records)


@pytest.fixture(scope="module")
def models():
    m = Models()
    yield m
    m.free()


# ------------------------------------------------------------------------------------------------ SD1.5 paths
@full
def test_multi_lora_sampling_pass(models, monkeypatch):
    """ControlInferenceLDM with two LoRA sets: forward_grouped runs the ControlNet on the batch 2 x the CFG batch, then
    one weighted_sum per control residual.  The weights are unequal and the hints differ, so a swapped set shows."""
    import bench
    model = models.get("inference_2loras")
    model.eval()
    model.lora_weights = [0.7, 0.45]
    cn = type(model.control_model)
    real_grouped, ran = cn.forward_grouped, []

    def grouped(self, hints, *args, **kwargs):
        ran.append(len(hints))
        return real_grouped(self, hints, *args, **kwargs)
    monkeypatch.setattr(cn, "forward_grouped", grouped)
    b = 2 * bench.BATCH
    g = _gen(41)
    x = _randn(g, b, 4, bench.LATENT, bench.LATENT)
    hints = [_randn(g, b, 4, bench.LATENT, bench.LATENT) for _ in range(2)]
    ctx = _randn(g, b, bench.CTX_TOKENS, bench.CTX_DIM)
    t = torch.tensor(T_CFG, device="cuda")[:b]
    sh = Shadow(monkeypatch)
    with torch.no_grad():
        eps = model.apply_model(x, t, [{"c_crossattn": [ctx], "c_concat": [h]} for h in hints])
    torch.cuda.synchronize()
    assert eps.shape == x.shape and torch.isfinite(eps).all()
    sh.check(f"multi-LoRA sampling pass (2 sets, CFG batch {b}, ControlNet batch {2 * b})")
    assert ran == [2]
    assert sh.calls["weighted_sum"] == len(model.control_scales) == 13
    assert all("w=0.7,0.45" in shape for op, shape, _ in sh.records if op == "weighted_sum")


@full
def test_pretrain_sampling_pass(models, monkeypatch):
    """ControlPretrainLDM.apply_model with one task's LoRA set switched in, another timestep and context per image"""
    import bench
    model = models.get("pretrain")
    model.eval()
    cn = model.control_model
    task = cn.tasks[1]
    real_switch, switched = type(cn).switch_lora, []

    def switch(self, name):
        switched.append(name)
        return real_switch(self, name)
    monkeypatch.setattr(type(cn), "switch_lora", switch)
    b = 2 * bench.BATCH
    g = _gen(42)
    x, hint = _randn(g, b, 4, bench.LATENT, bench.LATENT), _randn(g, b, 4, bench.LATENT, bench.LATENT)
    ctx = _randn(g, b, bench.CTX_TOKENS, bench.CTX_DIM)
    t = torch.tensor(T_CFG, device="cuda")[:b]
    sh = Shadow(monkeypatch)
    with torch.no_grad():
        model.prepare_context(ctx)
        twin = model.twin_enabled()
        eps = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [hint], "task": task})
    torch.cuda.synchronize()
    assert eps.shape == x.shape and torch.isfinite(eps).all()
    sh.check(f"pretrain sampling pass (task {task}, CFG batch {b}, twin encoder {twin})")
    assert switched == [task]
    assert all(m.lora_layer is lora for m, lora in zip(cn.lora_linears(), cn.loras_dict[task]))


@full
def test_vae_encode(models, monkeypatch):
    """encode_first_stage + get_first_stage_encoding at 512^2: the largest GroupNorm (262 144 pixels at 128 channels),
    the pad_lo = 0 stride-2 gathers of the Downsamples, the 4096-key softmax of the mid-block attention, and the
    posterior sample"""
    import bench
    model = models.get("finetune")
    side = 8 * bench.LATENT
    x = torch.rand(bench.BATCH, 3, side, side, device="cuda", generator=_gen(43)) * 2 - 1
    sh = Shadow(monkeypatch)
    torch.manual_seed(0)  # the posterior's host-side noise
    with torch.no_grad():
        z = model.get_first_stage_encoding(model.encode_first_stage(x))
    torch.cuda.synchronize()
    assert z.shape == (bench.BATCH, 4, bench.LATENT, bench.LATENT) and torch.isfinite(z).all()
    sh.check(f"VAE encode (batch {bench.BATCH}, {side}^2)")
    assert _has(sh, "im2col_s2", "pad_lo=0")
    assert _has(sh, "groupnorm", f"{bench.BATCH}x{side}x{side}x128")
    assert _has(sh, "softmax_rows", f"{bench.LATENT ** 2}x{bench.LATENT ** 2} ")
    assert _has(sh, "gaussian_sample", ",noise")


# ------------------------------------------------------------------------------------------------ annotators
@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    """a checkpoint directory with the fixtures' synthetic weights: sk_model.pth (fine), sk_model2.pth (coarse: the
    fine weights x 0.9), ControlNetHED.pth and body_pose_model.pth"""
    from ctrlora_b200.annotator.hed import ControlNetHED_Apache2
    from ctrlora_b200.annotator.lineart import Generator
    from ctrlora_b200.annotator.openpose import bodypose_model
    d = tmp_path_factory.mktemp("annotator_ckpts")
    shapes = lambda m: {k: tuple(v.shape) for k, v in m.state_dict().items()}
    fine = lg.weights(shapes(Generator(3, 1, lg.N_RESIDUAL)))
    torch.save(fine, d / "sk_model.pth")
    torch.save({k: v * 0.9 for k, v in fine.items()}, d / "sk_model2.pth")
    torch.save(hg.weights(shapes(ControlNetHED_Apache2())), d / "ControlNetHED.pth")
    torch.save({k.split(".", 1)[1]: v for k, v in og.weights(shapes(bodypose_model())).items()},
               d / "body_pose_model.pth")
    return str(d)


def _lineart_batch(n, h, w):
    imgs = [lg.image((h, w), tag=f".batch{i}") for i in range(n)]
    return torch.stack([torch.from_numpy(i).float() / 255.0 for i in imgs]).permute(0, 3, 1, 2).contiguous().cuda()


@pytest.mark.parametrize("size", SIZES["lineart"], ids=_ids)
def test_lineart_detector(ckpts, size, monkeypatch):
    from ctrlora_b200.annotator.lineart import LineartDetector
    det = LineartDetector(ckpt_dir=ckpts)
    img = lg.image(size)
    sh = Shadow(monkeypatch)
    fine, coarse = det(img, coarse=False), det(img, coarse=True)
    sh.check(f"LineartDetector fine + coarse at {_ids(size)}")
    assert fine.shape == coarse.shape == size and fine.dtype == np.uint8 and not np.array_equal(fine, coarse)
    assert _has(sh, "instance_norm", ",phases")
    assert _has(sh, "instance_norm", ",residual")
    assert _has(sh, "tap_gather", "f32nchw", "reflect")
    assert _has(sh, "tap_gather", "f16", "zero")
    assert _has(sh, "lineart_out", ",want_u8")
    assert _has(sh, "im2col_s2", "pad_lo=1")


def test_lineart_generator_batch_3(ckpts, monkeypatch):
    """Generator.forward on three different images: the per-image statistics of every instance norm"""
    from ctrlora_b200.annotator.lineart import LineartDetector
    model = LineartDetector(ckpt_dir=ckpts).model
    x = _lineart_batch(3, 256, 384)
    sh = Shadow(monkeypatch)
    y = model(x)
    torch.cuda.synchronize()
    assert y.shape == (3, 1, 256, 384) and torch.isfinite(y).all()
    sh.check("line-art Generator at batch 3, 256 x 384")
    assert _has(sh, "instance_norm", "4x3x", ",phases")
    assert _has(sh, "lineart_out", "3x256x384x64")


@pytest.mark.parametrize("safe", [False, True])
@pytest.mark.parametrize("size", SIZES["hed"], ids=_ids)
def test_hed_detector(ckpts, size, safe, monkeypatch):
    from ctrlora_b200.annotator.hed import HEDdetector
    det = HEDdetector(ckpt_dir=ckpts)
    img = hg.image(size)
    sh = Shadow(monkeypatch)
    edge = det(img, safe=safe)
    sh.check(f"HEDdetector at {_ids(size)}, safe={safe}")
    assert edge.shape == size and edge.dtype == np.uint8
    assert sh.calls["hed_fuse"] == 1
    assert _has(sh, "tap_gather", "f32nchw", "zero")
    assert _has(sh, "gemm_relu", "K=9x")
    assert _has(sh, "hed_side_pool", ",pool")
    assert any(op == "hed_side_pool" and ",pool" not in shape for op, shape, _ in sh.records)  # block5: side only


@pytest.mark.parametrize("size", SIZES["openpose"], ids=_ids)
def test_openpose_detector(ckpts, size, monkeypatch):
    from ctrlora_b200.annotator.openpose import OpenposeDetector
    det = OpenposeDetector(ckpt_dir=ckpts)
    img = og.image(size)
    sh = Shadow(monkeypatch)
    canvas = det(img)
    sh.check(f"OpenposeDetector at {_ids(size)}")
    assert canvas.shape == img.shape and canvas.dtype == np.uint8
    assert _has(sh, "gemm_relu", "K=49x")
    assert _has(sh, "gemm", "f32")
    assert _has(sh, "max_pool2x2")
    assert sh.calls["openpose_peaks"] == 1


# --------------------------------------------------------------------------------------------- the check notices
def _only(monkeypatch, op, wrapped):
    return Shadow(monkeypatch, replace={op: wrapped}, only=(op,))


def _assert_only_this(sh, op, text):
    _assert_reported(sh, op, text)
    assert len(sh.failures) == 1, sh.failures


def test_notices_swapped_phases_of_an_instance_norm(ckpts, monkeypatch):
    """phases 1 (py 0, px 1) and 2 (py 1, px 0) of one transposed conv's instance norm written to each other's pixels"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart import LineartDetector
    model = LineartDetector(ckpt_dir=ckpts).model
    real = ops.instance_norm

    def swap(p, args, kwargs):
        y = real(*args, **kwargs)
        _, b, h, w, c = p["x"].shape
        v = y.view(b, h, 2, w, 2, c)
        one = v[:, :, 0, :, 1].clone()
        v[:, :, 0, :, 1] = v[:, :, 1, :, 0]
        v[:, :, 1, :, 0] = one
        return y
    wrapped = _corrupt_once(real, lambda p: p["phases"], swap)
    sh = _only(monkeypatch, "instance_norm", wrapped)
    model(_lineart_batch(1, 64, 96))
    torch.cuda.synchronize()
    assert wrapped.state["done"]
    _assert_only_this(sh, "instance_norm", "y image 0")


def test_notices_a_zeroed_reflected_bottom_row(ckpts, monkeypatch):
    """one residual block's reflect gather with the taps of its last row that read below the border (mirrored from the
    row above it) zeroed, as zero padding would give"""
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart import LineartDetector
    model = LineartDetector(ckpt_dir=ckpts).model
    real = ops.tap_gather

    def zero_bottom(p, args, kwargs):
        out = real(*args, **kwargs)
        c = p["channels"] or p["x"].shape[-1]
        for t, (dy, _) in enumerate(p["taps"]):
            if dy > 0:
                out[:, -1, :, t * c:(t + 1) * c] = 0
        return out
    wrapped = _corrupt_once(real, lambda p: p["reflect"] and p["x"].dtype == torch.float16, zero_bottom)
    sh = _only(monkeypatch, "tap_gather", wrapped)
    model(_lineart_batch(1, 64, 96))
    torch.cuda.synchronize()
    assert wrapped.state["done"]
    _assert_only_this(sh, "tap_gather", "elements differ")


def test_notices_negatives_left_in_the_last_partial_m_tile(ckpts, monkeypatch):
    """one conv + ReLU (HED's first, 100 x 164 = 16 400 rows) whose last partial 128-row tile keeps its negatives"""
    import inspect
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.hed import HEDdetector
    det = HEDdetector(ckpt_dir=ckpts)
    real = ops.gemm_relu

    def rows(p):
        a = p["a"]
        return a.shape[0] if a.dim() == 2 else a.shape[0] * a.shape[1] * a.shape[2]

    def keep_negatives(p, args, kwargs):
        out = real(*args, **kwargs)
        plain = ops.gemm(*args, **kwargs)
        tail = rows(p) // 128 * 128
        out.view(-1, out.shape[-1])[tail:] = plain.view(-1, plain.shape[-1])[tail:]
        return out
    sig = _signature(dict(inspect.getmembers(ops, inspect.isfunction)), "gemm_relu")
    wrapped = _corrupt_once(real, lambda p: p["seg_outs"] is None and p["out"] is None and rows(p) % 128 != 0,
                            keep_negatives, sig=sig)
    sh = _only(monkeypatch, "gemm_relu", wrapped)
    det(hg.image((100, 164)))
    torch.cuda.synchronize()
    assert wrapped.state["done"]
    _assert_only_this(sh, "gemm_relu", "out")
