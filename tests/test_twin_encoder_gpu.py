"""The twin pass: the ControlNet and the UNet encoder as one batch-2B pass (cldm/cldm.py ControlLDM._control_and_unet).

A grouped launch computes every element of a tile as a plain launch over the same half does, so with the split
factor pinned a grouped GEMM equals two plain launches bit for bit, and grouped GroupNorm / LayerNorm (statistics per
image / per row) equal two plain calls.  At SD1.5 size the twin apply_model then differs from the sequential one only
where doubling M changes a GEMM's automatic split-K plan.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

pytestmark = pytest.mark.gpu


def _rand(*shape, s=1.0):
    return (torch.randn(*shape, device="cuda") * s).half()


def _f32(*shape):
    return torch.randn(*shape, device="cuda") * 0.1


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16) if a.dtype == torch.float16 else a,
                       b.contiguous().view(torch.int16) if b.dtype == torch.float16 else b)


# (batch per half, H, W, Cin, N, ksize)
GEMM_SHAPES = [(8, 8, 8, 1280, 1280, 3), (8, 16, 16, 640, 640, 3), (8, 64, 64, 320, 320, 1), (8, 16, 16, 640, 1280, 1)]


@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("epi", ["plain", "residual", "rowbias", "skipconv"])
@pytest.mark.parametrize("split", [1, 3])
def test_grouped_gemm_equals_two_launches(shape, epi, split):
    """split 3: every tile of the grouped launch and of the half launches splits K the same way (split tiles, whose
    last CTA picks the group's bias and row term, run the row-per-thread epilogue)"""
    from ctrlora_b200 import ops
    b, h, w, cin, n, k = shape
    if split > 1 and h * w * b > 16 * 16 * 8:
        pytest.skip("the split-K workspace holds the partial tiles of the coarse levels only")
    torch.manual_seed(0)
    a = _rand(2 * b, h, w, cin)
    wl, wh = _rand(n, k * k, cin, s=cin ** -0.5 / k), _rand(n, k * k, cin, s=cin ** -0.5 / k)
    bl, bh = _f32(n), _f32(n)
    kw_lo, kw_hi, hi = {}, {}, {"w": wh, "bias": bh}
    if epi == "residual":
        res = _rand(2 * b * h * w, n)
        kw_lo["residual"], kw_hi["residual"] = res[:b * h * w], res[b * h * w:]
    if epi == "rowbias":
        rl, rh = _f32(b, 2 * n)[:, :n], _f32(b, 2 * n)[:, :n]  # slices of wider rows, as the time embedding's
        kw_lo["rowbias"], kw_hi["rowbias"], hi["rowbias"] = rl, rh, rh
    if epi == "skipconv":
        a2, w2l, w2h = _rand(2 * b, h, w, 320), _rand(n, 320, s=0.05), _rand(n, 320, s=0.05)
        kw_lo.update(a2=a2[:b], w2=w2l)
        kw_hi.update(a2=a2[b:], w2=w2h)
        hi["w2"] = w2h
    both = dict(kw_lo)
    if epi == "residual":
        both["residual"] = res
    if epi == "skipconv":
        both["a2"] = a2
    g = ops.gemm(a, wl, ksize=k, bias=bl, split_k=split, hi=hi, **both)
    lo = ops.gemm(a[:b], wl, ksize=k, bias=bl, split_k=split, **kw_lo)
    up = ops.gemm(a[b:], wh, ksize=k, bias=bh, split_k=split, **kw_hi)
    torch.cuda.synchronize()
    assert _bits_equal(g[:b], lo) and _bits_equal(g[b:], up)


@pytest.mark.parametrize("rows", [64 * 64, 16 * 16, 8 * 8])
def test_grouped_linear_geglu_and_qkv_equal_two_launches(rows):
    """[M, K] operands (the transformer's linears) group by rows: GEGLU, and q | k | V^T with a transposed segment"""
    from ctrlora_b200 import ops
    b, c = 8, 320
    torch.manual_seed(1)
    x = _rand(2 * b * rows, c)
    w1l, w1h = _rand(2 * 4 * c, c, s=c ** -0.5), _rand(2 * 4 * c, c, s=c ** -0.5)
    b1l, b1h = _f32(8 * c), _f32(8 * c)
    g = ops.gemm(x, w1l, bias=b1l, geglu=True, split_k=1, hi={"w": w1h, "bias": b1h})
    assert _bits_equal(g[:b * rows], ops.gemm(x[:b * rows], w1l, bias=b1l, geglu=True, split_k=1))
    assert _bits_equal(g[b * rows:], ops.gemm(x[b * rows:], w1h, bias=b1h, geglu=True, split_k=1))
    heads, d = 8, c // 8
    nk_pad = (rows + 7) // 8 * 8
    wl, wh = _rand(3 * c, c, s=c ** -0.5), _rand(3 * c, c, s=c ** -0.5)

    def qkv(xx, ww, batch, hi=None):
        q = torch.empty((batch * rows, c), device="cuda", dtype=torch.float16)
        k = torch.empty_like(q)
        vt = torch.zeros((batch, heads, d, nk_pad), device="cuda", dtype=torch.float16)
        ops.gemm(xx, ww, seg_outs=[q, k, vt], seg_width=c, transposed=(0, 0, 1), rows_per_img=rows, head_dim=d,
                 tok_pad=nk_pad, split_k=1, hi=hi)
        return q, k, vt

    q, k, vt = qkv(x, wl, 2 * b, hi={"w": wh})
    for sl, ww, half in ((slice(0, b), wl, x[:b * rows]), (slice(b, 2 * b), wh, x[b * rows:])):
        q1, k1, vt1 = qkv(half, ww, b)
        r = slice(sl.start * rows, sl.stop * rows)
        assert _bits_equal(q[r], q1) and _bits_equal(k[r], k1) and _bits_equal(vt[sl], vt1)


def test_row_terms_of_different_strides_are_refused():
    from ctrlora_b200 import ops
    a = _rand(16, 8, 8, 64)
    wl, wh = _rand(64, 9, 64, s=0.05), _rand(64, 9, 64, s=0.05)
    with pytest.raises(AssertionError):
        ops.gemm(a, wl, ksize=3, rowbias=_f32(8, 128)[:, :64], hi={"w": wh, "rowbias": _f32(8, 64)})


def test_ungroupable_launch_falls_back():
    """4x4 images: one tile covers 8 images, so halves of 2 images cannot be tiled apart -- two launches instead"""
    from ctrlora_b200 import ops
    torch.manual_seed(2)
    a = _rand(4, 4, 4, 64)
    wl, wh = _rand(64, 9, 64, s=0.05), _rand(64, 9, 64, s=0.05)
    bl, bh = _f32(64), _f32(64)
    rl, rh = _f32(2, 64), _f32(2, 64)
    before = ops.LAUNCHES
    g = ops.gemm(a, wl, ksize=3, bias=bl, rowbias=rl, hi={"w": wh, "bias": bh, "rowbias": rh})
    assert ops.LAUNCHES - before == 2
    assert _bits_equal(g[:2], ops.gemm(a[:2], wl, ksize=3, bias=bl, rowbias=rl))
    assert _bits_equal(g[2:], ops.gemm(a[2:], wh, ksize=3, bias=bh, rowbias=rh))


@pytest.mark.parametrize("shape", [(8, 64, 64, 320), (8, 32, 32, 640), (8, 16, 16, 1280), (8, 8, 8, 1280)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("concat", [False, True])
def test_grouped_groupnorm_equals_two_calls(shape, concat):
    from ctrlora_b200 import ops
    b, h, w, c = shape
    torch.manual_seed(3)
    x1 = _rand(2 * b, h, w, c)
    x2 = _rand(2 * b, h, w, c) if concat else None
    add2 = _rand(2 * b, h, w, c) if concat else None
    ct = 2 * c if concat else c
    gl, bl, gh, bh = 1 + _f32(ct), _f32(ct), 1 + _f32(ct), _f32(ct)

    def gn(sl, g, be, **hi):
        kw = {} if not concat else {"x2": x2[sl], "add2": add2[sl], "add2_scale": 0.5}
        return ops.groupnorm(x1[sl], g, be, 1e-5, True, **kw, **hi)

    y = gn(slice(None), gl, bl, gamma_hi=gh, beta_hi=bh)
    assert _bits_equal(y[:b], gn(slice(0, b), gl, bl)) and _bits_equal(y[b:], gn(slice(b, None), gh, bh))


@pytest.mark.parametrize("cols", [320, 640, 1280])
def test_grouped_layernorm_equals_two_calls(cols):
    from ctrlora_b200 import ops
    torch.manual_seed(4)
    x = _rand(2 * 8 * 256, cols)
    gl, bl, gh, bh = 1 + _f32(cols), _f32(cols), 1 + _f32(cols), _f32(cols)
    y = ops.layernorm(x, gl, bl, 1e-5, gamma_hi=gh, beta_hi=bh)
    half = x.shape[0] // 2
    assert _bits_equal(y[:half], ops.layernorm(x[:half], gl, bl, 1e-5))
    assert _bits_equal(y[half:], ops.layernorm(x[half:], gh, bh, 1e-5))


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def sd15():
    from bench import build_model
    model = build_model(torch.device("cuda"), seed=0)
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(8, 4, 64, 64, device="cuda", generator=g)
    hint = torch.randn(8, 4, 64, 64, device="cuda", generator=g)
    ctx = torch.randn(8, 77, 768, device="cuda", generator=g)
    t = torch.full((8,), 501, device="cuda", dtype=torch.long)
    return model, x, hint, ctx, t


def test_sd15_twin_matches_sequential(sd15, monkeypatch):
    """13 control residuals and eps of the twin pass against the sequential one (random weights, batch 8).  The blocks
    above the first Downsample run at batch 8 as before: their residuals are bit-identical.  Below it only GEMMs whose
    automatic split-K plan changes with the doubled M round differently (measured: at most 1.2e-3)."""
    model, x, hint, ctx, t = sd15
    cond = {"c_crossattn": [ctx], "c_concat": [hint]}
    with torch.no_grad():
        model.prepare_context(ctx)
        assert model.twin_enabled()
        control, _, _, _, _ = model._control_and_unet(x, hint, t, ctx)
        eps_twin = model.apply_model(x, t, cond)
        monkeypatch.setenv("CTRLORA_TWIN_ENCODER", "0")
        assert not model.twin_enabled()
        ref = model.control_model(hint=hint, timesteps=t, context=ctx)
        eps_seq = model.apply_model(x, t, cond)
    torch.cuda.synchronize()
    rels = [_rel(c, r) for c, r in zip(control, ref)]
    e = _rel(eps_twin, eps_seq)
    print(f"control max rel {max(rels):.2e}, eps rel {e:.2e}, bitwise residuals "
          f"{sum(_bits_equal(c, r) for c, r in zip(control, ref))}/13")
    above = 4  # input blocks above the fork: conv_in, 2 x (ResBlock + ST), Downsample
    assert all(_bits_equal(c, r) for c, r in zip(control[:above], ref[:above]))
    assert max(rels) < 2.5e-3 and e < 2.5e-3


def _tiny(name, lora_num=None, seed=0):
    from bench import random_weights_
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import load_config
    from ldm.util import instantiate_from_config
    cfg = load_config(os.path.join(ROOT, "tests", "golden", name))
    if lora_num is not None:
        cfg["model"]["params"]["control_stage_config"]["params"]["lora_num"] = lora_num
    model = instantiate_from_config(cfg["model"]).cuda().eval()
    random_weights_(model, seed)
    return model


def _tiny_inputs(model, b=2):
    """latents of the tiny configs (16 x 16) and a context of their cross-attention width"""
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(b, 4, 16, 16, device="cuda", generator=g)
    hint = torch.randn(b, 4, 16, 16, device="cuda", generator=g)
    width = model._twin_pairs()["cross"][0][1].to_k.in_features
    ctx = torch.randn(b, 77, width, device="cuda", generator=g)
    t = torch.full((b,), 321, device="cuda", dtype=torch.long)
    return x, hint, ctx, t


class _NoTwin(Exception):
    pass


def _forbid_twin(model, monkeypatch):
    def fail(*a, **k):
        raise _NoTwin
    monkeypatch.setattr(model, "_control_and_unet", fail)


def test_fallbacks_take_the_sequential_path(monkeypatch):
    """apply_model never enters the twin pass with the knob off, in training mode, under autograd, or with grouped
    multi-LoRA inference (two LoRA sets)"""
    model = _tiny("tiny_finetune.yaml")
    x, hint, ctx, t = _tiny_inputs(model)
    cond = {"c_crossattn": [ctx], "c_concat": [hint]}
    with torch.no_grad():
        assert model.twin_enabled()
        _forbid_twin(model, monkeypatch)
        with pytest.raises(_NoTwin):
            model.apply_model(x, t, cond)
        monkeypatch.setenv("CTRLORA_TWIN_ENCODER", "0")
        model.apply_model(x, t, cond)
        monkeypatch.delenv("CTRLORA_TWIN_ENCODER")
        model.train()
        model.apply_model(x, t, cond)
        model.eval()
    model.apply_model(x, t, cond)  # autograd on: a training forward
    two = _tiny("tiny_inference.yaml")
    assert two.control_model.lora_num == 2
    _forbid_twin(two, monkeypatch)
    with torch.no_grad():
        two.apply_model(x, t, [cond, cond])


def test_one_set_inference_takes_the_twin_pass(monkeypatch):
    """The inference ControlNet's transformer norms are Switchable* shells; the eps that counts is the attached
    layer's, which equals the UNet's.  A one-set apply_model runs the twin pass and matches the sequential one."""
    model = _tiny("tiny_inference.yaml", lora_num=1)
    x, hint, ctx, t = _tiny_inputs(model)
    cond = {"c_crossattn": [ctx], "c_concat": [hint]}
    calls = []
    orig = model._control_and_unet
    monkeypatch.setattr(model, "_control_and_unet", lambda *a, **k: calls.append(1) or orig(*a, **k))
    with torch.no_grad():
        eps_twin = model.apply_model(x, t, cond)
        assert calls and model.twin_enabled()
        monkeypatch.setenv("CTRLORA_TWIN_ENCODER", "0")
        eps_seq = model.apply_model(x, t, cond)
    torch.cuda.synchronize()
    assert len(calls) == 1
    e = _rel(eps_twin, eps_seq)
    print(f"tiny one-set inference: eps rel {e:.2e}")
    assert e < 2.5e-3


def test_style_variant_is_not_twinned():
    """The IP-Adapter UNet's cross-attention class differs from the ControlNet's: no twin pairs, while the inference
    variant it derives from has them"""
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    model = create_model(os.path.join(ROOT, "tests", "golden", "tiny_style.yaml")).cuda().eval()
    assert model._twin_pairs() is None
    inference = create_model(os.path.join(ROOT, "tests", "golden", "tiny_inference.yaml")).cuda().eval()
    assert inference._twin_pairs() is not None
    tiny = create_model(os.path.join(ROOT, "tests", "golden", "tiny_finetune.yaml")).cuda().eval()
    assert tiny._twin_pairs() is not None
