"""Training-step parity: loss and the gradients of the optimizer's parameter set (246 tensors: LoRA down/up, zero-convs,
'norm' layers) from the CUDA forward+backward, against the gradients the UNMODIFIED reference produced with autograd
(tests/golden/tiny_finetune_golden.pt: loss, per-tensor gradient norms for all 246, full tensors for a sample)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu

from tolerances import TOL  # noqa: E402
from golden_io import load_golden  # noqa: E402


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


@pytest.fixture(scope="module")
def setup():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ctrlora_b200.train import FinetuneTrainer
    from oracle import synth
    g = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = create_model(os.path.join(GOLD, "tiny_finetune.yaml"), init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(g["control_shapes"], g["seed"], "control_model."))
    model.model.diffusion_model.load_state_dict(synth.synth_state_dict(g["unet_shapes"], g["seed"], "model.diffusion_model."))
    model = model.cuda().eval()
    trainer = FinetuneTrainer(model, lr=1e-3)
    B, H, seed = g["B"], g["H"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    data = dict(x0=mk("x", (B, 4, H, H)), hint=mk("hint", (B, 4, H, H)), ctx=mk("ctx", (B, 77, 64)),
                noise=mk("noise", (B, 4, H, H)), t=g["t"].cuda())
    return g, model, trainer, data


def test_loss_and_gradients_vs_reference_autograd(setup):
    g, model, trainer, d = setup
    assert trainer.G.names == g["trainable_names"]  # same parameter set, same order as the reference optimizer
    loss = trainer.loss_and_grads(d["x0"], d["hint"], d["ctx"], d["t"], d["noise"])
    torch.cuda.synchronize()
    e_eps = rel(trainer.last_eps, g["train_eps"])
    e_loss = abs(loss.item() - g["loss"].item()) / abs(g["loss"].item())
    print(f"train eps rel err {e_eps:.2e}, loss rel err {e_loss:.2e}")
    assert e_eps < TOL["tiny_eps"] and e_loss < TOL["tiny_loss"]
    grads = trainer.unscaled_grads()  # the loss scale divided out
    # four tensors (input_blocks.{1,2}.0.emb_layers.1 LoRA) have mathematically zero gradients in this config (32
    # channels / 32 groups: the GroupNorm cancels the time-embedding offset; reference norms ~1e-9)
    norms = sorted(g["grad_norms"].values())
    median, biggest = norms[len(norms) // 2], norms[-1]
    worst, n_zero = 0.0, 0
    for n, ref in g["grad_norms"].items():
        got = grads[n].norm().item()
        if ref < 1e-5 * biggest:  # mathematically zero: ours must be noise (< 1 % of the median gradient norm)
            assert got < 1e-2 * median, (n, got, ref)
            n_zero += 1
            continue
        err = abs(got - ref) / ref
        worst = max(worst, err)
        assert err < TOL["tiny_grad_norm"], (n, got, ref)
    assert n_zero == 4
    errs = {n: rel(grads[n], ref) for n, ref in g["grads"].items()}
    print("grad norm worst rel err %.2e; full-tensor rel errs:" % worst, {k[-40:]: "%.1e" % v for k, v in errs.items()})
    # fp16 activations/gradients through ~60 layers: 2e-2 norm-relative on individual tensors
    assert max(errs.values()) < TOL["tiny_grad_tensor"]


def test_optimizer_step_changes_outputs_and_matches_adamw(setup):
    g, model, trainer, d = setup
    names, before = trainer.G.names, trainer.G.flat_p.clone()
    loss0 = trainer.step(d["x0"], d["hint"], d["ctx"], d["t"], d["noise"]).item()
    grads = trainer.G.flat_g.clone() / trainer._scale_used  # AdamW sees the un-scaled gradient
    # torch.optim.AdamW on the same (params, grads), first step
    p_ref = torch.nn.Parameter(before.clone())
    opt = torch.optim.AdamW([p_ref], lr=1e-3)
    p_ref.grad = grads
    opt.step()
    assert (trainer.G.flat_p - p_ref.detach()).abs().max().item() < 2e-6  # (g * 1/scale) vs (g / scale): 1 ulp
    losses = [loss0]
    for _ in range(5):
        losses.append(trainer.step(d["x0"], d["hint"], d["ctx"], d["t"], d["noise"]).item())
    print("losses over 6 steps on one batch:", ["%.5f" % v for v in losses])
    assert losses[-1] < losses[0]  # the folded-weight caches follow the updated LoRA / zero-conv / norm parameters


def test_loss_scale_invariance_and_overflow_skip(setup):
    """ADVICE r1 (fp16 backward without loss scaling): gradients must not depend on the scale over a wide range, a
    scale that overflows fp16 must be detected, the update skipped and the scale halved."""
    g, model, trainer, d = setup
    args = (d["x0"], d["hint"], d["ctx"], d["t"], d["noise"])
    saved = trainer.loss_scale
    ref = None
    for scale in (None, 4.0, 4096.0):
        trainer.loss_scale = scale
        trainer.loss_and_grads(*args)
        flat = (trainer.G.flat_g / trainer._scale_used).clone()
        if ref is None:
            ref = flat
        else:
            e = rel(flat, ref)
            print(f"loss scale {scale}: gradient rel diff vs default scale {e:.2e}")
            assert e < 5e-3
    # the un-scaled regime the advisor flagged: d_eps ~ 1e-5 (batch 16 x 4 x 64 x 64 numerics emulated with a 1/128 scale)
    trainer.loss_scale = 1.0 / 128
    trainer.loss_and_grads(*args)
    e_small = rel(trainer.G.flat_g / trainer._scale_used, ref)
    print(f"loss scale 1/128 (underflowing fp16 gradients): rel diff {e_small:.2e}")
    assert e_small > 5e-3  # this is the failure the default scale avoids
    # overflow: inf/nan in the flat gradient -> skipped step, halved scale
    trainer.loss_scale = 1e9
    trainer.CHECK_OVERFLOW_EVERY = 1  # poll the device-side skipped-steps counter after this very step (default: every 16th)
    before = trainer.G.flat_p.clone()
    steps = trainer.step_count
    trainer.step(*args)
    assert trainer.skipped_steps >= 1 and trainer.step_count == steps
    assert torch.equal(trainer.G.flat_p, before)
    assert trainer.loss_scale == 0.5e9
    trainer.loss_scale = saved
    del trainer.CHECK_OVERFLOW_EVERY


@pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")
def test_sd15_training_step_vs_reference_golden():
    """SD1.5-size training step (rank 128, B = 2) against the unmodified reference's autograd:
    tests/golden/sd15_rank128_train_golden.pt from `tools/make_golden.py --full-train` (loss, 246 gradient norms, 7 tensors)."""
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ctrlora_b200.train import FinetuneTrainer
    from oracle import synth
    g = load_golden(os.path.join(GOLD, "sd15_rank128_train_golden.pt"))
    gs = torch.load(os.path.join(GOLD, "sd15_rank128_golden.pt"), weights_only=False)
    model = create_model(os.path.join(ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml"), init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(gs["control_shapes"], g["seed"], "control_model."))
    model.model.diffusion_model.load_state_dict(synth.synth_state_dict(gs["unet_shapes"], g["seed"], "model.diffusion_model."))
    model = model.cuda().eval()
    tr = FinetuneTrainer(model)
    assert tr.G.names == g["trainable_names"]
    B, seed = g["B"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    loss = tr.loss_and_grads(mk("x", (B, 4, 64, 64)), mk("hint", (B, 4, 64, 64)), mk("ctx", (B, 77, 768)), g["t"].cuda(),
                             mk("noise", (B, 4, 64, 64)))
    torch.cuda.synchronize()
    e_eps = rel(tr.last_eps, g["eps"])
    e_loss = abs(loss.item() - g["loss"].item()) / abs(g["loss"].item())
    grads = tr.unscaled_grads()
    nerr = {n: abs(grads[n].norm().item() - r) / r for n, r in g["grad_norms"].items()}
    worst = max(nerr, key=nerr.get)
    terr = {n: rel(grads[n], r) for n, r in g["grads"].items()}
    print(f"SD1.5 training step: eps {e_eps:.2e}, loss {e_loss:.2e}, worst grad-norm err {nerr[worst]:.2e} ({worst}), "
          f"median {sorted(nerr.values())[len(nerr) // 2]:.2e}; tensors", {k[-44:]: "%.1e" % v for k, v in terr.items()})
    assert e_eps < TOL["sd15_eps"] and e_loss < TOL["sd15_loss"]
    assert nerr[worst] < TOL["sd15_grad_norm"] and max(terr.values()) < TOL["sd15_grad_tensor"]


@pytest.mark.parametrize("rank", [4, 16, 32])
def test_rank_sweep_training_parity(rank, tmp_path):
    """BASELINE.json configs[4]: the finetune step at other LoRA ranks (rank 4 is not a multiple of 8: the fold and the
    factored gradient GEMMs zero-pad it) against the reference's autograd (tests/golden/tiny_ranks_golden.pt)."""
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ctrlora_b200.train import FinetuneTrainer
    from oracle import synth
    g = torch.load(os.path.join(GOLD, "tiny_ranks_golden.pt"), weights_only=False)
    ref = g["ranks"][rank]
    cfg = tmp_path / f"tiny_rank{rank}.yaml"
    cfg.write_text(open(os.path.join(GOLD, "tiny_finetune.yaml")).read().replace("lora_rank: 8", f"lora_rank: {rank}"))
    model = create_model(str(cfg), init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(ref["control_shapes"], g["seed"], "control_model."))
    model.model.diffusion_model.load_state_dict(synth.synth_state_dict(g["unet_shapes"], g["seed"], "model.diffusion_model."))
    model = model.cuda().eval()
    tr = FinetuneTrainer(model)
    B, H, seed = g["B"], g["H"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    loss = tr.loss_and_grads(mk("x", (B, 4, H, H)), mk("hint", (B, 4, H, H)), mk("ctx", (B, 77, 64)), g["t"].cuda(),
                             mk("noise", (B, 4, H, H)))
    e_eps = rel(tr.last_eps, ref["eps"])
    e_loss = abs(loss.item() - ref["loss"].item()) / abs(ref["loss"].item())
    grads = tr.unscaled_grads()
    norms = sorted(ref["grad_norms"].values())
    biggest, median = norms[-1], norms[len(norms) // 2]
    worst = 0.0
    for n, rn in ref["grad_norms"].items():
        got = grads[n].norm().item()
        if rn < 1e-5 * biggest:
            assert got < 1e-2 * median, (n, got, rn)
        else:
            worst = max(worst, abs(got - rn) / rn)
    print(f"rank {rank}: eps {e_eps:.2e}, loss {e_loss:.2e}, worst grad-norm err {worst:.2e}")
    assert e_eps < TOL["tiny_eps"] and e_loss < TOL["tiny_loss"] and worst < TOL["tiny_grad_norm"]
