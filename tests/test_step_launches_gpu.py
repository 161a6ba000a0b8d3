"""Every kernel launch of the benchmarked steps against a plain fp32 reference of the same call (tests/launch_refs.py).

The per-kernel tests check each kernel at shapes their authors picked.  The steps pick others, and with them plans no
per-kernel test lists: the grouped batch-16 encoder pass, split-K tails, GroupNorm's partial statistics at batch 16,
wgrad at M = 65536, pointer alignments that choose between the TMA epilogue and the row-per-thread one.  Here the real
steps run eagerly (no CUDA graph) at SD1.5 size with bench.py's random weights while a shadow replaces the `ops`
wrappers the references cover: each call runs the real kernel, and its outputs are compared with the reference computed
from the inputs the kernel actually received (pre-call copies of the operands the call overwrites and also reads).

Scenarios: the sampling pass on the DDIM sampler's CFG batch, the VAE decode, the finetune step at bench.TRAIN_BATCH and
the pretrain step at bench.PRETRAIN_BATCH.  The `ops` functions a step calls that no shadow covers must be listed in
UNCHECKED with the reason.  The fault-injection tests corrupt one call's *result* in Python and assert that the shadow
names that call.  `pytest -s` prints one line per distinct call signature with its plan and error.  The shadow itself
lives in tests/launch_shadow.py.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from launch_shadow import Models, Shadow, _assert_reported, _corrupt_once, _gen, _randn  # noqa: E402

pytestmark = pytest.mark.gpu
full = pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")


@pytest.fixture(scope="module")
def models():
    m = Models()
    yield m
    m.free()


def _sampling_pass(model, seed=21):
    """apply_model on the CFG batch of the DDIM sampler (2 x bench.BATCH latents), with a different timestep and
    context per image so that a row term or a context read from the wrong image shows"""
    import bench
    b = 2 * bench.BATCH
    g = _gen(seed)
    x, hint = _randn(g, b, 4, bench.LATENT, bench.LATENT), _randn(g, b, 4, bench.LATENT, bench.LATENT)
    ctx = _randn(g, b, bench.CTX_TOKENS, bench.CTX_DIM)
    t = torch.tensor([981, 901, 781, 641, 501, 341, 181, 21], device="cuda")[:b]
    with torch.no_grad():
        model.prepare_context(ctx)
        assert model.twin_enabled()
        return model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [hint]})


def _train_inputs(b, seed):
    import bench
    g = _gen(seed)
    x0, hint = _randn(g, b, 4, bench.LATENT, bench.LATENT), _randn(g, b, 4, bench.LATENT, bench.LATENT)
    ctx, noise = _randn(g, b, bench.CTX_TOKENS, bench.CTX_DIM), _randn(g, b, 4, bench.LATENT, bench.LATENT)
    t = torch.randint(0, 1000, (b,), device="cuda", generator=g)
    return x0, hint, ctx, t, noise


@full
def test_sampling_pass(models, monkeypatch):
    model = models.get("finetune")
    model.eval()
    sh = Shadow(monkeypatch)
    eps = _sampling_pass(model)
    torch.cuda.synchronize()
    assert torch.isfinite(eps).all()
    sh.check("sampling pass (CFG batch 8, twin encoder at 16)")
    for op in ("gemm", "groupnorm"):
        assert 16 in sh.grouped[op], dict(sh.grouped)
    assert sh.grouped["layernorm"], dict(sh.grouped)


@full
def test_vae_decode(models, monkeypatch):
    import bench
    model = models.get("finetune")
    z = _randn(_gen(22), bench.BATCH, 4, bench.LATENT, bench.LATENT)
    sh = Shadow(monkeypatch)
    with torch.no_grad():
        img = model.decode_first_stage(z)
    torch.cuda.synchronize()
    assert img.shape == (bench.BATCH, 3, 8 * bench.LATENT, 8 * bench.LATENT) and torch.isfinite(img).all()
    sh.check("VAE decode (batch 4)")


@full
def test_finetune_step(models, monkeypatch):
    import bench
    from ctrlora_b200.train import FinetuneTrainer
    model = models.get("finetune")
    trainer = FinetuneTrainer(model, lr=1e-5)
    args = _train_inputs(bench.TRAIN_BATCH, 23)
    sh = Shadow(monkeypatch)
    loss = trainer.loss_and_grads(*args)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    sh.check(f"finetune step (batch {bench.TRAIN_BATCH})")
    m = bench.TRAIN_BATCH * bench.LATENT * bench.LATENT
    assert any(op == "wgrad_tn" and shape.startswith(f"M={m} ") for op, shape, _ in sh.records)


@full
def test_pretrain_step(models, monkeypatch):
    import bench
    from ctrlora_b200.train import PretrainTrainer
    model = models.get("pretrain")
    trainer = PretrainTrainer(model, lr=1e-5)
    args = _train_inputs(bench.PRETRAIN_BATCH, 24)
    sh = Shadow(monkeypatch)
    loss = trainer.loss_and_grads(*args, task=trainer.tasks[0])
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    sh.check(f"pretrain step (batch {bench.PRETRAIN_BATCH}, task {trainer.tasks[0]})")
    # the dense 3x3 conv weight gradients: wgrad over im2col columns, Q = 9 * Cin
    assert any(op == "wgrad_tn" and f"Q={9 * 320} " in shape for op, shape, _ in sh.records)


# --------------------------------------------------------------------------------------------- the check notices
def _run_sampling_with(models, monkeypatch, op, corrupt_fn, seed=21):
    """the sampling pass with one call of `op` corrupted and only `op` checked"""
    from ctrlora_b200 import ops
    model = models.get("finetune")
    model.eval()
    wrapped = corrupt_fn(getattr(ops, op))
    sh = Shadow(monkeypatch, replace={op: wrapped}, only=(op,))
    _sampling_pass(model, seed)
    torch.cuda.synchronize()
    assert wrapped.state["done"], "no call took the corruption"
    return sh


@full
def test_notices_grouped_gemm_upper_half_with_the_lower_bias(models, monkeypatch):
    """the upper half of one grouped GEMM's output recomputed with the lower half's bias"""
    def corrupt(real):
        def lower_bias(p, args, kwargs):
            out = real(*args, **kwargs)
            h = out.shape[0] // 2
            out[h:] += ((p["bias"] - p["hi"]["bias"]) * p["out_scale"]).to(out.dtype)
            return out
        return _corrupt_once(real, lambda p: p["hi"] is not None and p["bias"] is not None and
                             p["hi"].get("bias") is not None and not p["geglu"] and p["seg_outs"] is None, lower_bias)
    sh = _run_sampling_with(models, monkeypatch, "gemm", corrupt)
    _assert_reported(sh, "gemm", "out hi")


@full
def test_notices_an_unwritten_partial_m_tile(models, monkeypatch):
    """the context's K | V^T projection (8 x 77 = 616 rows): K rows 512..615, the last partial 128-row tile, keep their
    pre-call contents -- another context's keys, as the sampling pass ran on a different context before"""
    def corrupt(real):
        def restore(p, args, kwargs):
            k = p["seg_outs"][0]
            tail = k.shape[0] // 128 * 128
            keep = k[tail:].clone()
            ret = real(*args, **kwargs)
            k[tail:] = keep
            return ret
        return _corrupt_once(real, lambda p: p["seg_outs"] is not None and not p["transposed"][0] and
                             p["seg_outs"][0].shape[0] % 128 != 0, restore)
    _sampling_pass(models.get("finetune"), seed=30)
    sh = _run_sampling_with(models, monkeypatch, "gemm", corrupt, seed=31)
    _assert_reported(sh, "gemm", "segment 0")


@full
def test_notices_a_grouped_groupnorm_image_with_the_lower_gamma(models, monkeypatch):
    """the last image of one grouped GroupNorm (an upper-half image) normalised with the lower half's gamma and beta"""
    def corrupt(real):
        def lower(p, args, kwargs):
            ret = real(*args, **kwargs)
            y = ret[0] if isinstance(ret, tuple) else ret
            sl = slice(p["x1"].shape[0] - 1, None)
            cut = {k: (None if p[k] is None else p[k][sl]) for k in ("add1", "x2", "add2")}
            y[sl] = real(p["x1"][sl], p["gamma"], p["beta"], p["eps"], p["silu"], add1_scale=p["add1_scale"],
                         add2_scale=p["add2_scale"], groups=p["groups"], **cut)
            return ret
        return _corrupt_once(real, lambda p: p["gamma_hi"] is not None, lower)
    sh = _run_sampling_with(models, monkeypatch, "groupnorm", corrupt)
    _assert_reported(sh, "groupnorm", "y hi")


@full
def test_notices_wgrad_dropping_beta(models, monkeypatch):
    """one accumulating weight gradient (beta = 1, a second micro-batch of an accumulation window) that overwrites"""
    import bench
    from ctrlora_b200 import ops
    from ctrlora_b200.train import FinetuneTrainer
    real = ops.wgrad_tn

    def drop_beta(p, args, kwargs):
        return real(p["a"], p["b"], out=p["out"], alpha=p["alpha"], beta=0.0)
    wrapped = _corrupt_once(real, lambda p: p["beta"] != 0.0 and bool(p["out"].any()), drop_beta)
    trainer = FinetuneTrainer(models.get("finetune"), lr=1e-5)
    args = _train_inputs(bench.TRAIN_BATCH, 25)
    trainer.loss_and_grads(*args)
    sh = Shadow(monkeypatch, replace={"wgrad_tn": wrapped}, only=("wgrad_tn",))
    trainer.loss_and_grads(*args, accumulate=True)
    torch.cuda.synchronize()
    assert wrapped.state["done"]
    _assert_reported(sh, "wgrad_tn", "dW")


@full
def test_notices_a_zeroed_last_head_of_the_last_image(models, monkeypatch):
    def corrupt(real):
        def zero(p, args, kwargs):
            out = real(*args, **kwargs)
            out.view(p["batch"], p["nq"], -1)[-1, :, -p["head_dim"]:] = 0
            return out
        return _corrupt_once(real, lambda p: True, zero)
    sh = _run_sampling_with(models, monkeypatch, "attention", corrupt)
    _assert_reported(sh, "attention", "out image ")
    hit = next(f for f in sh.failures if f[0] == "attention")
    batch = int(hit[2].split()[0][len("B="):])
    assert f"out image {batch - 1} " in hit[3], hit  # the last image, and only it
