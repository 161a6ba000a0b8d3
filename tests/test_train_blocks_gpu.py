"""The training backward at SD1.5 size, block by block, against fp32 autograd through the oracle.

The trainer's own functions (train.seq_fwd / seq_bwd / zero_conv_bwd / unet_bwd / emb_mlp_backward) run every
TimestepEmbedSequential of the ControlNet and of the UNet decoder at B = 2, 64x64 latent, 77 x 768 context, on synthetic
weights of the SD1.5 finetune and pretrain configs.  The reference is ctrlora_oracle (pinned to the reference by
test_oracle_golden.py) under torch autograd in fp32 on the GPU, TF32 off, fed the same fp16-rounded activations and upstream
gradients; it reads the fp32 master weights, so the product's fp16 weight rounding counts as its error.  Every input gradient
and every gradient tensor the optimizer's sink holds for a block is compared per tensor (tolerances.close: norm-relative
bound plus a max-abs guard); `pytest -s` prints each measured error.  Last, one full pretraining step against
oracle.apply_model + p_losses: the loss and every gradient tensor of the base ControlNet and of the active task's LoRA set.
"""
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

from tolerances import TOL, close  # noqa: E402

B, RES, SEED, TASK = 2, 64, 0, "canny"
HEADS, MC = 8, 320                        # SD1.5: num_heads 8, model_channels 320
S_MID, S_CTRL = 0.7, 1.3                  # control scales != 1 on the decoder's mid-control add and skip-half add
# (channels, resolution) entering ControlNet input_blocks.0 .. 11 and middle_block, and (h, skip channels, resolution)
# entering UNet output_blocks.0 .. 11
CN_IN = [(4, 64), (320, 64), (320, 64), (320, 64), (320, 32), (640, 32), (640, 32), (640, 16), (1280, 16), (1280, 16),
         (1280, 8), (1280, 8), (1280, 8)]
UNET_IN = [(1280, 1280, 8), (1280, 1280, 8), (1280, 1280, 8), (1280, 1280, 16), (1280, 1280, 16), (1280, 640, 16),
           (1280, 640, 32), (640, 640, 32), (640, 320, 32), (640, 320, 64), (320, 320, 64), (320, 320, 64)]


@pytest.fixture(scope="module", autouse=True)
def fp32_reference_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _pm(gen, b, h, w, c):
    """N(0, 1) rounded to fp16, pixel-major [B, H, W, C] (the trainer's activation layout)"""
    return torch.randn(b, h, w, c, device="cuda", generator=gen).half()


def _nchw32(buf):
    return buf.permute(0, 3, 1, 2).float()


def _build(mode, config, trainer_cls):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from oracle import synth
    model = create_model(os.path.join(ROOT, "configs", config), init_weights=False)
    for sub, prefix in ((model.control_model, "control_model."), (model.model.diffusion_model, "model.diffusion_model.")):
        shapes = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
        sub.load_state_dict(synth.synth_state_dict(shapes, SEED, prefix))
    model = model.cuda().eval()
    cn = model.control_model
    ups = [(n, p) for n, p in cn.named_parameters() if "lora" in n and n.endswith("up.weight")]
    assert ups and all(p.detach().abs().sum().item() > 0 for _, p in ups), "a LoRA up weight is zero: dDown would be untested"
    trainer = trainer_cls(model)
    if mode == "pretrain":
        cn.switch_lora(TASK)
    gen = torch.Generator(device="cuda").manual_seed(SEED)
    t = torch.tensor([981, 420], device="cuda")
    ctx = torch.randn(B, 77, 768, device="cuda", generator=gen).half()
    # oracle names: after switch_lora the attached set is also reachable as <linear>.lora_layer.* -- the names oracle.linear
    # reads; the other tasks' sets have no such alias
    alias = {}
    for n, p in cn.named_parameters(remove_duplicate=False):
        if not n.startswith("loras_dict."):
            alias[id(p)] = n
    sd = {n: p.detach().requires_grad_(True) for n, p in cn.named_parameters(remove_duplicate=False)
          if not n.startswith("loras_dict.")}
    unet = model.model.diffusion_model
    usd = {n: p.detach() for n, p in unet.named_parameters()}
    from ldm.modules.diffusionmodules.openaimodel import ResBlock
    resblocks = [(n, m) for n, m in cn.named_modules() if isinstance(m, ResBlock)]
    emb = cn.embed(t)
    d_all = torch.zeros((B, sum(m.out_channels for _, m in resblocks)), device="cuda")
    emb_grads, off = {}, 0
    for _, m in resblocks:
        emb_grads[id(m)] = d_all[:, off:off + m.out_channels]
        off += m.out_channels
    return dict(model=model, cn=cn, unet=unet, trainer=trainer, G=trainer.G, t=t, ctx16=ctx, alias=alias, sd=sd, usd=usd,
                resblocks=resblocks, emb=emb, d_all=d_all, emb_grads=emb_grads, done=set(), gen=gen, mode=mode)


@pytest.fixture(scope="module")
def finetune():
    from ctrlora_b200.train import FinetuneTrainer
    return _build("finetune", "ctrlora_finetune_sd15_rank128.yaml", FinetuneTrainer)


@pytest.fixture(scope="module")
def pretrain():
    from ctrlora_b200.train import PretrainTrainer
    return _build("pretrain", "ctrlora_pretrain_sd15_9tasks_rank128.yaml", PretrainTrainer)


def _errors(got, ref):
    got, ref = got.detach().float(), ref.detach().float()
    nrel = ((got - ref).norm() / (ref.norm() + 1e-20)).item()
    return nrel, (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)


class _Report:
    """collects (label, got, ref, bound) so that every error of a case is printed before the first assertion"""

    def __init__(self, title):
        self.title, self.rows = title, []

    def add(self, label, got, ref, bound):
        assert ref is not None, f"{self.title}: no reference gradient for {label}"
        self.rows.append((label, got, ref, bound) + _errors(got, ref))

    def check(self):
        worst = max(self.rows, key=lambda r: r[4] / TOL[r[3]])
        print(f"\n{self.title}: {len(self.rows)} tensors, worst {worst[0]} norm-rel {worst[4]:.2e} (bound {TOL[worst[3]]:.1e})")
        for label, _, _, bound, nrel, mx in self.rows:
            print(f"    {label:<72s} norm-rel {nrel:.2e}  max-abs {mx:.2e}  [{bound}]")
        for label, got, ref, bound, _, _ in self.rows:  # max-abs guard: 1.5x the bound (measured max-abs / norm-rel <= 1.25)
            close(got, ref, tol=1.5 * TOL[bound], nrel=TOL[bound], what=f"{self.title} {label}")
        return worst[4]


def _zero_ref_grads(sd):
    for v in sd.values():
        v.grad = None


def _emb_to_input(sd, prefix, seq, e, emb_grads):
    """product d(emb): the block's d(rowbias) slices mapped through its ResBlocks' emb_layers (SiLU, LoRA linear) in fp32"""
    from oracle import ctrlora_oracle as O
    from ldm.modules.diffusionmodules.openaimodel import ResBlock
    outs, grads = [], []
    for j, layer in enumerate(seq):
        if isinstance(layer, ResBlock):
            outs.append(O.linear(sd, f"{prefix}.{j}.emb_layers.1", F.silu(e)))
            grads.append(emb_grads[id(layer)])
    if not outs:
        return None
    return torch.autograd.grad(outs, e, grads)[0]


def _controlnet_block(s, i):
    """one ControlNet block (input_blocks.i, i = 12: middle_block) and its zero conv, product vs oracle.  The block's
    d(rowbias) slices stay in d_all for emb_mlp_backward; s["done"] records which blocks have filled theirs."""
    from ctrlora_b200 import train
    from ctrlora_b200.runtime import nchw_view
    from oracle import ctrlora_oracle as O
    cn, G, sd, gen = s["cn"], s["G"], s["sd"], s["gen"]
    seq, zc = (cn.input_blocks[i], cn.zero_convs[i]) if i < 12 else (cn.middle_block, cn.middle_block_out)
    prefix, zprefix = (f"input_blocks.{i}", f"zero_convs.{i}") if i < 12 else ("middle_block", "middle_block_out")
    c, r = CN_IN[i]
    x16 = _pm(gen, B, r, r, c)
    G.zero()
    ids = {id(rb) for rb in seq}
    for rb_id, sl in s["emb_grads"].items():
        if rb_id in ids:
            sl.zero_()
    # product: the trainer's forward tape, the zero conv's backward with the gradient arriving from the next block
    x_in = _nchw32(x16) if i == 0 else nchw_view(x16)
    out, tape = train.seq_fwd(seq, x_in, s["emb"], s["ctx16"])
    bo, co, ho, wo = out.shape
    d_zc, d_up = _pm(gen, bo, ho, wo, co), _pm(gen, bo, ho, wo, co)
    d_h = train.zero_conv_bwd(zc, out, nchw_view(d_zc), G, nchw_view(d_up))
    dx = train.seq_bwd(tape, d_h, G, s["emb_grads"])
    torch.cuda.synchronize()
    # reference
    _zero_ref_grads(sd)
    xr = _nchw32(x16).requires_grad_(True)
    er = s["emb"].raw.detach().clone().requires_grad_(True)
    h = O.sequential_block(sd, prefix, xr, er, s["ctx16"].float(), HEADS)
    loss = (O.conv(sd, zprefix + ".0", h) * _nchw32(d_zc)).sum() + (h * _nchw32(d_up)).sum()
    loss.backward()
    mode = s["mode"]
    rep = _Report(f"[{mode}] ControlNet {prefix}")
    if i > 0:
        rep.add("d(input)", dx, xr.grad, "sd15_blk_dx")
    d_emb = _emb_to_input(sd, prefix, seq, er.detach().requires_grad_(True), s["emb_grads"])
    if d_emb is not None:
        rep.add("d(emb) through emb_layers", d_emb, er.grad, "sd15_blk_demb")
    grads = G.named_grads()
    n_owned = 0
    for n, p in zip(G.names, G.params):
        on = s["alias"].get(id(p))
        if on is None or not on.startswith((prefix + ".", zprefix + ".")) or ".emb_layers." in on:
            continue  # another block's, another task's, or the time-embedding MLP's (emb_mlp_backward)
        n_owned += 1
        rep.add(on, grads[n], sd[on].grad, "sd15_blk_grad")
    assert n_owned > 0
    s["done"].add(i)
    return rep


@pytest.mark.parametrize("mode", ["finetune", "pretrain"])
@pytest.mark.parametrize("i", list(range(13)), ids=[f"input_blocks.{i}" for i in range(12)] + ["middle_block"])
def test_controlnet_block_backward(request, mode, i):
    s = request.getfixturevalue(mode)
    t0 = time.perf_counter()
    rep = _controlnet_block(s, i)
    print(f"    ({time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB)")
    rep.check()


@pytest.mark.parametrize("j", list(range(12)))
def test_unet_decoder_block_backward(finetune, j):
    """UNet output_blocks.j fed a runtime.CatSpec as unet_fwd builds it: [h (+ S_MID * c_mid on block 0) | skip + S_CTRL * c];
    backward with want_dx2 and, on block 0, dx1_scale = S_MID (the gradient of the mid control), G = None as in unet_bwd"""
    from ctrlora_b200 import train
    from ctrlora_b200.runtime import CatSpec, nchw_view
    from oracle import ctrlora_oracle as O
    s = finetune
    unet, usd, gen = s["unet"], s["usd"], s["gen"]
    ch, cs, r = UNET_IN[j]
    h16, skip16, add16 = _pm(gen, B, r, r, ch), _pm(gen, B, r, r, cs), _pm(gen, B, r, r, cs)
    cmid16 = _pm(gen, B, r, r, ch) if j == 0 else None
    uemb = unet.embed(s["t"])
    spec = CatSpec(nchw_view(h16), add1=nchw_view(cmid16) if j == 0 else None, s1=S_MID, x2=nchw_view(skip16),
                   add2=nchw_view(add16), s2=S_CTRL)
    out, tape = train.seq_fwd(unet.output_blocks[j], spec, uemb, s["ctx16"])
    bo, co, ho, wo = out.shape
    d16 = _pm(gen, bo, ho, wo, co)
    dx1, dadd = train.seq_bwd(tape, nchw_view(d16), None, None,
                              first_res_kw=dict(want_dx2=True, dx1_scale=S_MID if j == 0 else 1.0))
    hr, ar = _nchw32(h16).requires_grad_(True), _nchw32(add16).requires_grad_(True)
    cr = _nchw32(cmid16).requires_grad_(True) if j == 0 else None
    x1 = hr + S_MID * cr if j == 0 else hr
    x = torch.cat([x1, _nchw32(skip16) + S_CTRL * ar], 1)
    y = O.sequential_block(usd, f"output_blocks.{j}", x, uemb.raw.detach(), s["ctx16"].float(), HEADS)
    (y * _nchw32(d16)).sum().backward()
    rep = _Report(f"UNet output_blocks.{j}")
    rep.add("d(c_mid) = S_MID d(h)" if j == 0 else "d(h)", dx1, cr.grad if j == 0 else hr.grad, "sd15_blk_dx")
    rep.add("d(control) = S_CTRL d(skip half)", dadd, ar.grad, "sd15_blk_dx")
    rep.check()


def test_out_head_and_mse_loss_backward(finetune):
    """GroupNorm + SiLU + conv 320 -> 4 (n_pad = 16) as unet_fwd runs it, ops.mse_loss_grad with the trainer's c_pad and loss
    scale, unet_bwd's head backward"""
    from ctrlora_b200 import ops, prepare, train
    from oracle import ctrlora_oracle as O
    s = finetune
    unet, usd, gen = s["unet"], s["usd"], s["gen"]
    h16 = _pm(gen, B, RES, RES, MC)
    noise = torch.randn(B, 4, RES, RES, device="cuda", generator=gen).half().float()
    gn, conv = unet.out[0], unet.out[2]
    f32 = prepare.bias_f32
    a, stats = ops.groupnorm(h16, f32(gn.weight), f32(gn.bias), gn.eps, True, want_stats=True)
    n_pad = (unet.out_channels + 15) // 16 * 16
    bias = torch.cat([conv.bias.detach().float(), torch.zeros(n_pad - unet.out_channels, device="cuda")])
    eps = ops.nhwc_to_nchw_f32(ops.gemm(a, conv.kernel_weight(pad_out=n_pad), ksize=3, bias=bias, out_f32=True), unet.out_channels)
    scale = s["trainer"]._scale_for(eps.numel())
    loss, d_eps = ops.mse_loss_grad(eps, noise, c_pad=n_pad, grad_scale=scale)
    d_h = train.unet_bwd(unet, {"tapes": [], "stats": stats, "hp": h16, "n_pad": n_pad, "only_mid": False}, d_eps)[12]
    hr = _nchw32(h16).requires_grad_(True)
    eps_ref = O.conv(usd, "out.2", F.silu(O.group_norm(usd, "out.0", hr, 1e-5)), padding=1)
    loss_ref = O.p_losses(eps_ref, noise)
    loss_ref.backward()
    e_loss = abs(loss.item() - loss_ref.item()) / loss_ref.item()
    print(f"\nout head: n_pad {n_pad}, loss scale {scale:g}, loss rel err {e_loss:.2e}")
    rep = _Report("UNet out head + MSE")
    rep.add("eps", eps, eps_ref, "sd15_blk_dx")
    rep.add("d(h) / loss scale", d_h.float() / scale, hr.grad, "sd15_blk_dx")
    rep.check()
    assert e_loss < TOL["sd15_loss"]


@pytest.mark.parametrize("mode", ["finetune", "pretrain"])
def test_time_embedding_mlp_backward(request, mode):
    """train.emb_mlp_backward fed the d(rowbias) the ControlNet blocks produced (the block cases above) against autograd of
    oracle.time_embed and every ResBlock's emb_layers: the sink's time_embed.* and *.emb_layers.* gradients"""
    from ctrlora_b200 import train
    from ldm.modules.diffusionmodules.util import timestep_embedding
    from oracle import ctrlora_oracle as O
    s = request.getfixturevalue(mode)
    for i in range(13):
        if i not in s["done"]:
            _controlnet_block(s, i)
    assert all(s["emb_grads"][id(m)].abs().sum().item() > 0 for _, m in s["resblocks"])
    G, sd = s["G"], s["sd"]
    G.zero()
    train.emb_mlp_backward(s["cn"], timestep_embedding(s["t"], MC), s["emb"].raw, s["d_all"], s["emb_grads"], G)
    torch.cuda.synchronize()
    _zero_ref_grads(sd)
    e = O.time_embed(sd, s["t"], MC)
    loss = sum((O.linear(sd, f"{n}.emb_layers.1", F.silu(e)) * s["emb_grads"][id(m)]).sum() for n, m in s["resblocks"])
    loss.backward()
    rep = _Report(f"[{mode}] time-embedding MLP")
    grads = G.named_grads()
    for n, p in zip(G.names, G.params):
        on = s["alias"].get(id(p))
        if on is not None and (on.startswith("time_embed.") or ".emb_layers." in on):
            rep.add(on, grads[n], sd[on].grad, "sd15_emb_mlp_grad")
    assert len(rep.rows) > 0
    rep.check()


@pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")
def test_sd15_pretrain_step_vs_oracle(pretrain):
    """PretrainTrainer.loss_and_grads at SD1.5 size (B = 2, one task) against fp32 autograd through oracle.apply_model +
    p_losses on the same x_noisy, noise, t, context and hint latent: the loss, every gradient tensor of the base ControlNet
    and of the active task's LoRA set; every other task's set stays exactly zero"""
    from oracle import ctrlora_oracle as O
    s = pretrain
    model, tr, G, gen = s["model"], s["trainer"], s["G"], s["gen"]
    mk = lambda *shape: torch.randn(*shape, device="cuda", generator=gen).half().float()
    x0, hint, noise = mk(B, 4, RES, RES), mk(B, 4, RES, RES), mk(B, 4, RES, RES)
    ctx, t = s["ctx16"].float(), s["t"]
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    loss = tr.loss_and_grads(x0, hint, ctx, t, noise, task=TASK)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    peak_product = torch.cuda.max_memory_allocated()
    inv = 1.0 / tr._scale_used
    grads = {n: g * inv for n, g in G.named_grads().items()}
    x_noisy = model.q_sample(x_start=x0, t=t, noise=noise)
    sd = {"control_model." + n: v for n, v in s["sd"].items()}
    sd.update({"model.diffusion_model." + n: v for n, v in s["usd"].items()})
    _zero_ref_grads(s["sd"])
    torch.cuda.reset_peak_memory_stats()
    eps = O.apply_model(sd, x_noisy, t, ctx, hint, HEADS, MC, model.control_scales, model.only_mid_control)
    loss_ref = O.p_losses(eps, noise)
    loss_ref.backward()
    torch.cuda.synchronize()
    print(f"\nfull pretrain step: product {t1 - t0:.1f} s, peak {peak_product / 2**30:.1f} GiB; fp32 reference "
          f"{time.perf_counter() - t1:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
    e_loss = abs(loss.item() - loss_ref.item()) / loss_ref.item()
    print(f"loss {loss.item():.6f} vs {loss_ref.item():.6f}: rel err {e_loss:.2e}; eps norm-rel "
          f"{_errors(tr.last_eps, eps)[0]:.2e}")
    rep = _Report("full pretrain step")
    n_other = 0
    for n, p in zip(G.names, G.params):
        on = s["alias"].get(id(p))
        if on is None:  # another task's LoRA set: never reached
            assert n.startswith("loras_dict.") and not n.startswith(f"loras_dict.{TASK}.")
            assert torch.count_nonzero(grads[n]).item() == 0, n
            n_other += 1
            continue
        rep.add(on, grads[n], s["sd"][on].grad, "sd15_pt_grad_tensor")
    assert n_other == (len(s["cn"].tasks) - 1) * 2 * len(s["cn"].lora_linears())
    by_kind = {}
    for label, _, _, _, nrel, _ in rep.rows:
        kind = "lora" if ".lora_layer." in label else label.rsplit(".", 1)[-1]
        by_kind[kind] = max(by_kind.get(kind, 0.0), nrel)
    print("worst norm-rel by tensor kind:", {k: f"{v:.2e}" for k, v in by_kind.items()})
    rep.check()
    assert e_loss < TOL["sd15_loss"]
