"""One place for the parity tolerances (test infrastructure).

north_star: "within 1e-3 relative fp16, bit-exact for timestep/index ops".  Two kinds of bound live here:

* per-kernel bounds (`close`): every kernel is compared with an fp32 torch reference on the SAME fp16-rounded inputs, so
  the only error is the kernel's own arithmetic + one fp16 rounding of its output (rms 2.8e-4).  Primary criterion:
  NORM-RELATIVE error ||got - ref|| / ||ref|| <= 1e-3 (the north_star figure) unless a test states otherwise; the older
  max-abs criterion (|err|_max <= tol * |ref|_max) is kept as a second guard against localised damage.
* end-to-end bounds (`TOL`): norm-relative error against the reference's own outputs (golden fixtures), set about 20 %
  above the error measured when each bound was introduced, so a regression of the accumulated rounding error fails the
  suite.  The tests print the errors they measure (`pytest -s`).  Where a bound is above 1e-3 the entry says why
  (tests/precision_study.py attributes the SD1.5 figure to the fp16 roundings).
"""
import torch

NORM_REL = 1e-3

# name: bound  -- what the compared quantity is, and why the bound exceeds 1e-3 where it does
TOL = {
    "tiny_eps": 2.6e-3,          # width-32 network, ~60 layers of fp16 operand rounding
    "tiny_control": 2.5e-3,      # 13 residuals x 5 attached LoRA sets, worst residual
    "tiny_sample": 4.7e-3,       # 4-step sampling and pred_x0 (which divides the eps error by sqrt(alpha_t) ~ 0.07 at t = 981)
    "tiny_loss": 2e-4,           # training loss
    "tiny_grad_norm": 4.6e-3,    # worst of 246 (finetune) / 816 (pretrain) gradient-tensor norms
    "tiny_grad_tensor": 7e-3,    # worst of the full gradient tensors kept in the goldens
    "mid_eps": 1.7e-3,           # mid-size network eps
    "mid_cfg_step": 3.9e-3,      # x_prev of one CFG-7.5 DDIM step of a 4-step schedule, non-square latent
    "mid_ragged_eps": 2.05e-3,   # worst of six ragged / non-square shapes
    "sd15_eps": 1.9e-3,          # SD1.5 + ControlNet rank 128, forward and training forward (B = 2)
    "sd15_control": 1.8e-3,      # ControlNet residuals, worst of control[0..12]
    "sd15_loss": 1e-4,           # training loss
    "sd15_grad_norm": 1.2e-3,    # worst of the 246 gradient norms
    "sd15_grad_tensor": 2.3e-3,  # worst of the full gradient tensors kept in the golden
    # training backward per SD1.5 block (test_train_blocks_gpu.py, B = 2, 64x64, vs fp32 autograd of the oracle): a block is
    # a handful of fp16 roundings of activations and gradients, so bounds of a few 1e-3
    "sd15_blk_dx": 1.1e-3,       # input gradients of ControlNet / decoder blocks and of the out head (worst: middle_block)
    "sd15_blk_demb": 1.15e-3,    # d(emb) of a block, its d(rowbias) mapped through the emb_layers in fp32
    "sd15_blk_grad": 2e-3,       # every sink gradient of a block, finetune and pretrain (worst: LoRA of the middle block's
                                 # self-attention)
    "sd15_emb_mlp_grad": 5.2e-4,  # time_embed / emb_layers gradients of emb_mlp_backward
    "sd15_pt_grad_tensor": 4.3e-3,  # full pretrain step: worst of the 488 base and active-LoRA gradient tensors (the whole
                                    # network's fp16 roundings, like sd15_grad_tensor)
    "vae_encode": 2e-3,          # first-stage VAE moments, tiny and SD VAE at 512x512
    "vae_decode": 3.5e-3,        # tiny decode, encode->decode round trip, SD VAE decode
}


def norm_rel(got, ref):
    got, ref = got.detach().float(), ref.detach().float()
    return ((got - ref).norm() / (ref.norm() + 1e-20)).item()


def close(got, ref, tol=2e-3, nrel=NORM_REL, what=""):
    """max-abs guard (tol * max|ref|) AND norm-relative bound (nrel)."""
    got, ref = got.detach().float(), ref.detach().float()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    nr = norm_rel(got, ref)
    assert err <= tol * scale, f"{what} max err {err:.4e} vs scale {scale:.4e}"
    assert nr <= nrel, f"{what} norm-relative err {nr:.3e} > {nrel:.1e}"
    return nr
