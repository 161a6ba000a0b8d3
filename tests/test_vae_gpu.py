"""First-stage VAE parity (SURVEY.md §8 rows f1 / f3): the drop-in AutoencoderKL (encoder, decoder, posterior) on the
sm_90a kernels against outputs of the unmodified reference (ldm/models/autoencoder.py:82-91,
ldm/modules/diffusionmodules/model.py:452-654; fixtures from `tools/make_golden.py --vae / --vae-full`)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu

from tolerances import TOL  # noqa: E402


def rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / (ref.norm() + 1e-20)).item()


def vae_image(name, shape, seed):
    from oracle import synth
    x = synth.synth_input(name, shape, seed)
    x = torch.nn.functional.avg_pool2d(x, 3, stride=1, padding=1) * 2.0
    return torch.tanh(x)


@pytest.fixture(scope="module")
def tiny():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from oracle import synth
    g = torch.load(os.path.join(GOLD, "tiny_vae_golden.pt"), weights_only=False)
    gt = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = create_model(os.path.join(GOLD, "tiny_finetune.yaml"), init_weights=False)
    vae = model.first_stage_model
    assert vae is not None and list(vae.state_dict().keys()) == g["key_order"]
    vae.load_state_dict(synth.synth_state_dict(g["shapes"], g["seed"], "first_stage_model."), strict=True)
    model.control_model.load_state_dict(synth.synth_state_dict(gt["control_shapes"], gt["seed"], "control_model."))
    model.model.diffusion_model.load_state_dict(synth.synth_state_dict(gt["unet_shapes"], gt["seed"], "model.diffusion_model."))
    return g, gt, model.cuda().eval()


def test_tiny_vae_encode_decode_vs_reference(tiny):
    from oracle import synth
    g, _, model = tiny
    vae = model.first_stage_model
    img = vae_image("vae_img", (2, 3, 32, 32), g["seed"]).cuda()
    z = synth.synth_input("vae_z", (2, 4, 16, 16), g["seed"]).cuda()
    post = vae.encode(img)
    e_mom, e_mode = rel(post.parameters, g["moments"]), rel(post.mode(), g["mode"])
    torch.manual_seed(123)  # the posterior draws its noise from the host generator like the reference
    e_smp = rel(post.sample(), g["sample_seed123"])
    e_dec = rel(vae.decode(z), g["decode"])
    e_rt = rel(vae.decode(post.mode()), g["roundtrip"])
    print(f"tiny VAE: moments {e_mom:.2e}, mode {e_mode:.2e}, sample {e_smp:.2e}, decode {e_dec:.2e}, roundtrip {e_rt:.2e}")
    assert max(e_mom, e_mode, e_smp) < TOL["vae_encode"] and max(e_dec, e_rt) < TOL["vae_decode"]
    # the LDM-level helpers: scale_factor folded into the sample / post_quant kernels
    torch.manual_seed(123)
    lat = model.get_first_stage_encoding(model.encode_first_stage(img))
    assert rel(lat, model.scale_factor * g["sample_seed123"]) < TOL["vae_encode"]
    dec = model.decode_first_stage(z * model.scale_factor)
    assert rel(dec, g["decode"]) < TOL["vae_decode"]


def test_image_space_hint_through_apply_model(tiny):
    """c_concat holds the 3-channel condition IMAGE (the reference's real calling convention,
    cldm/cldm_ctrlora_finetune.py:76-77): apply_model == apply_model on the latent the VAE kernels produce."""
    from oracle import synth
    g, gt, model = tiny
    B, H = 2, 16
    x = synth.synth_input("x", (B, 4, H, H), gt["seed"]).cuda()
    ctx = synth.synth_input("ctx", (B, 77, 64), gt["seed"]).cuda()
    img = vae_image("vae_img", (B, 3, 2 * H, 2 * H), g["seed"]).cuda()
    t = gt["t"].cuda()
    with torch.no_grad():
        torch.manual_seed(7)
        eps_img = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [img]})
        torch.manual_seed(7)
        lat = model.get_first_stage_encoding(model.encode_first_stage(img))
        eps_lat = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [lat]})
        # same latent, same kernels: every statistic is summed in a fixed order, so the two are bit-equal (measured on an
        # H100); the tolerance is a margin, not noise the check expects
        assert rel(eps_img, eps_lat) < 2 * TOL["tiny_eps"]
        # reference semantics: a fresh posterior sample per call; opt-in cache: one encode per distinct hint tensor
        l1 = model.get_first_stage_encoding(model.encode_first_stage(img))
        l2 = model.get_first_stage_encoding(model.encode_first_stage(img))
        assert rel(l1, l2) > 1e-3  # a fresh posterior draw per call
        model.cache_hint_latent = True
        a = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [img]})
        b = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [img]})
        model.cache_hint_latent = False
        assert rel(a, b) < 2 * TOL["tiny_eps"]


@pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")
def test_sd_vae_512_vs_reference():
    """The SD first stage (ch 128, mult 1-2-4-4, mid attention d = 512) at 512x512, B = 1."""
    from ctrlora_b200 import dropin
    dropin.activate()
    from ldm.models.autoencoder import AutoencoderKL
    from oracle import synth
    g = torch.load(os.path.join(GOLD, "sd_vae_golden.pt"), weights_only=False)
    vae = AutoencoderKL(ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128,
                                      ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0),
                        lossconfig={"target": "torch.nn.Identity"}, embed_dim=4)
    assert list(vae.state_dict().keys()) == g["key_order"]
    vae.load_state_dict(synth.synth_state_dict(g["shapes"], g["seed"], "first_stage_model."), strict=True)
    vae = vae.cuda().eval()
    img = vae_image("vae_img", (1, 3, 512, 512), g["seed"]).cuda()
    z = synth.synth_input("vae_z", (1, 4, 64, 64), g["seed"]).cuda()
    post = vae.encode(img)
    e_mom = rel(post.parameters, g["moments"])
    dec = vae.decode(z)
    e_crop = rel(dec[:, :, 192:320, 192:320], g["decode_crop"])
    e_str = rel(dec[:, :, ::8, ::8], g["decode_strided"])
    e_norm = abs(dec.norm().item() - g["decode_norm"]) / g["decode_norm"]
    print(f"SD VAE 512x512: moments {e_mom:.2e}, decode crop {e_crop:.2e}, strided {e_str:.2e}, norm {e_norm:.2e}")
    assert e_mom < TOL["vae_encode"] and max(e_crop, e_str) < TOL["vae_decode"]
