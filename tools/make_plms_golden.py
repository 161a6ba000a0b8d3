"""Generate tests/golden/tiny_plms_golden.pt and sd15_plms_golden.pt by running the UNMODIFIED reference `PLMSSampler`
(/root/reference, ldm/models/diffusion/plms.py) on the reference's model classes, through tools/ref_shims.py.

    python tools/make_plms_golden.py          # tiny configs (samples) + host schedule for the SD1.5 alphas_cumprod
    python tools/make_plms_golden.py --full   # SD1.5 rank 128, batch 2, 20 steps, CFG 7.5 (CPU, takes minutes)

The reference's PLMSSampler cannot run on a CtrLoRA model as it is (DESIGN.md §7): `sample()` calls `.shape` on the
conditioning's first entry, the list `c_concat` / `c_crossattn` (plms.py:85-91), and its guidance branch `torch.cat`s
the cond dicts (plms.py:188-190).  Two substitutions make it run, and nothing else is changed:
  * the sampler gets a thin model proxy (`GuidanceProxy`), and `conditioning` / `unconditional_conditioning` are
    marker tensors of the batch's size, so the `.shape` check only ever sees a marker and the `torch.cat` runs;
  * the proxy's `apply_model` splits the reference's `x_in` / `t_in` into the uncond and cond halves and calls the
    real `apply_model` with each dict, then concatenates the two eps in the reference's [uncond | cond] order.
All other attributes are the model's.  As for DDIM in tools/make_golden.py, `register_buffer` keeps the buffers where
they are (the reference moves them to a hard-coded 'cuda', plms.py:19-23; there is no GPU here).

Weights and inputs are regenerated from names by oracle/synth.py, so the fixtures hold outputs only; running the tool
twice gives identical bytes.
"""
import argparse
import os
import sys
import time
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from tools.make_golden import _sd15_reference_ldm, build_reference  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests"))
from golden_io import save_golden  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SCHEDULE_STEPS = (1, 2, 3, 4, 5, 20, 50)   # 3 does not divide 1000, and the reference's schedule fails there
TINY_STEPS = (1, 4, 20)


class GuidanceProxy:
    """The model as the reference's PLMSSampler sees it, with `cond` / `ucond` standing behind marker tensors."""

    def __init__(self, model, cond, ucond, batch):
        self._model, self._cond, self._ucond = model, cond, ucond
        self.c_mark = torch.ones(batch)
        self.u_mark = None if ucond is None else torch.zeros(batch)

    def __getattr__(self, name):
        return getattr(self._model, name)

    def apply_model(self, x, t, c):
        if c is self.c_mark:
            return self._model.apply_model(x, t, self._cond)
        b = x.shape[0] // 2   # c is torch.cat([u_mark, c_mark]) (plms.py:190)
        assert torch.equal(c, torch.cat([self.u_mark, self.c_mark]))
        e_u = self._model.apply_model(x[:b], t[:b], self._ucond)
        e_c = self._model.apply_model(x[b:], t[b:], self._cond)
        return torch.cat([e_u, e_c])


def reference_sampler(model):
    from ldm.models.diffusion.plms import PLMSSampler
    sampler = PLMSSampler(model)
    sampler.register_buffer = lambda name, attr: setattr(sampler, name, attr)
    return sampler


def plms_sample(model, x_T, steps, cond, ucond, scale, **kw):
    """PLMSSampler.sample of the reference on `model`, guidance through GuidanceProxy: (samples, intermediates)."""
    proxy = GuidanceProxy(model, cond, ucond if scale != 1. else None, x_T.shape[0])
    sampler = reference_sampler(proxy)
    with torch.no_grad():
        return sampler.sample(steps, x_T.shape[0], tuple(x_T.shape[1:]), proxy.c_mark, verbose=False, x_T=x_T.clone(),
                              unconditional_guidance_scale=scale, unconditional_conditioning=proxy.u_mark, eta=0., **kw)


def schedule_record(model, steps):
    """The reference's tables for `steps` (make_schedule, plms.py:25-55) and, per step of plms_sampling, the values the
    loop forms: `ts` / `ts_next` (:150-151) and the four `torch.full` scalars of get_x_prev_and_pred_x0 (:204-207),
    read from the reference's own calls on a model whose eps is zero, with the derived per-step scalars a_t.sqrt(),
    a_prev.sqrt() and (1 - a_prev - sigma_t**2).sqrt() (:210, :216, :220) evaluated from them as the reference does."""
    fulls, real_full = [], torch.full

    def full(size, fill, **kw):
        out = real_full(size, fill, **kw)
        fulls.append(out)
        return out
    proxy = GuidanceProxy(model, None, None, 1)
    proxy.apply_model = lambda x, t, c: torch.zeros_like(x)
    sampler = reference_sampler(proxy)
    with torch.no_grad(), mock.patch.object(torch, "full", full):
        sampler.sample(steps, 1, (1, 1, 1), None, verbose=False, x_T=torch.zeros(1, 1, 1, 1), eta=0.)
    rec = {"ddim_timesteps": np.asarray(sampler.ddim_timesteps), "ddim_alphas": sampler.ddim_alphas.clone(),
           "ddim_alphas_prev": np.asarray(sampler.ddim_alphas_prev),
           "ddim_sqrt_one_minus_alphas": torch.as_tensor(sampler.ddim_sqrt_one_minus_alphas).clone(),
           "ddim_sigmas": torch.as_tensor(sampler.ddim_sigmas).clone(),
           "t": [], "t_next": [], "a_t": [], "a_prev": [], "sigma_t": [], "sqrt_one_minus_at": [],
           "sqrt_a_t": [], "sqrt_a_prev": [], "dir_coef": []}
    pos = 0
    for i in range(len(sampler.ddim_timesteps)):
        ts, ts_next = fulls[pos], fulls[pos + 1]
        a_t, a_prev, sigma_t, s1m = fulls[pos + 2:pos + 6]
        pos += 10 if i == 0 else 6   # step 0 forms the scalars twice (provisional and final update)
        rec["t"].append(int(ts[0]))
        rec["t_next"].append(int(ts_next[0]))
        for k, v in (("a_t", a_t), ("a_prev", a_prev), ("sigma_t", sigma_t), ("sqrt_one_minus_at", s1m),
                     ("sqrt_a_t", a_t.sqrt()), ("sqrt_a_prev", a_prev.sqrt()),
                     ("dir_coef", (1. - a_prev - sigma_t ** 2).sqrt())):
            rec[k].append(float(v.flatten()[0]))
    assert pos == len(fulls)
    return rec


def _no_vae(model):
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    return model


def tiny(seed=0):
    B, H = 2, 16
    mk = lambda n, s: synth.synth_input(n, s, seed)
    x_T, hint, hint2 = mk("plms_xT", (B, 4, H, H)), mk("hint", (B, 4, H, H)), mk("hint2", (B, 4, H, H))
    ctx, uc = mk("ctx", (B, 77, 64)), mk("uc_ctx", (B, 77, 64))
    ip, uc_ip = mk("ip", (B, 4, 64)), mk("uc_ip", (B, 4, 64))
    g = {"seed": seed, "B": B, "H": H, "scale": 7.5, "finetune": {}, "pretrain": {}}

    model = _no_vae(build_reference(os.path.join(GOLD, "tiny_finetune.yaml"), seed))
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    for S in TINY_STEPS:
        for scale in (1.0, 7.5):
            g["finetune"][(S, scale)] = plms_sample(model, x_T, S, cond, ucond, scale)[0]
    _, inter = plms_sample(model, x_T, 4, cond, ucond, 7.5, log_every_t=1)
    g["finetune_intermediates"] = {"steps": 4, "log_every_t": 1, "x_inter": inter["x_inter"],
                                   "pred_x0": inter["pred_x0"]}
    g["alphas_cumprod"] = model.alphas_cumprod.clone()
    g["schedule"] = {}
    for S in SCHEDULE_STEPS:
        try:
            g["schedule"][S] = schedule_record(model, S)
        except IndexError as e:   # S = 3: the last DDIM timestep is 1000, past the table (util.py:46-65)
            g["schedule"][S] = {"error": type(e).__name__}

    model = _no_vae(build_reference(os.path.join(GOLD, "tiny_pretrain.yaml"), seed))
    for task in ("canny", "depth", "seg"):
        c = {"c_crossattn": [ctx], "c_concat": [hint], "task": task}
        u = {"c_crossattn": [uc], "c_concat": [hint], "task": task}
        g["pretrain"][task] = plms_sample(model, x_T, 4, c, u, 7.5)[0]

    model = _no_vae(build_reference(os.path.join(GOLD, "tiny_inference.yaml"), seed))
    model.lora_weights = [0.7, 0.3]
    g["inference_lora_weights"] = [0.7, 0.3]
    conds = [{"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [ctx], "c_concat": [hint2]}]
    uconds = [{"c_crossattn": [uc], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint2]}]
    g["inference"] = plms_sample(model, x_T, 4, conds, uconds, 7.5)[0]

    # style model: image-prompt tokens in both halves; guess mode as the style app sets it
    # (app/gradio_ctrlora_style_transfer.py:426-432), with the hint-less uncond in the form the reference's
    # apply_model accepts, c_concat [None] (cldm/cldm_ctrlora_style_inference.py:169)
    model = _no_vae(build_reference(os.path.join(GOLD, "tiny_style.yaml"), seed))
    cond = {"c_crossattn": [ctx], "c_concat": [hint], "c_ip": [ip]}
    ucond = {"c_crossattn": [uc], "c_concat": [hint], "c_ip": [uc_ip]}
    g["style"] = plms_sample(model, x_T, 4, cond, ucond, 7.5)[0]
    guess_scales = [1.0 * (0.825 ** float(12 - i)) for i in range(13)]
    model.control_scales = guess_scales
    g["style_guess_control_scales"] = guess_scales
    g["style_guess"] = plms_sample(model, x_T, 4, cond, dict(ucond, c_concat=[None]), 7.5)[0]

    out = os.path.join(GOLD, "tiny_plms_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


def full(seed=0):
    B, R, S = 2, 64, 20
    model = _no_vae(_sd15_reference_ldm(seed))
    mk = lambda n, s: synth.synth_input(n, s, seed)
    x_T, hint = mk("plms_xT", (B, 4, R, R)), mk("hint", (B, 4, R, R))
    cond = {"c_crossattn": [mk("ctx", (B, 77, 768))], "c_concat": [hint]}
    ucond = {"c_crossattn": [mk("uc_ctx", (B, 77, 768))], "c_concat": [hint]}
    t0 = time.time()
    g = {"seed": seed, "B": B, "R": R, "steps": S, "scale": 7.5,
         "samples": plms_sample(model, x_T, S, cond, ucond, 7.5)[0]}
    print("sampled in", time.time() - t0, "s")
    out = os.path.join(GOLD, "sd15_plms_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    full() if a.full else tiny()
