"""The DPM_Solver cases of tests/golden/dpm_solver_golden.pt, shared by tools/make_dpm_solver_golden.py (which runs
them through the reference's unmodified dpm_solver module on the CPU) and the tests (which run them through the
drop-in).  A scripted model returns pre-drawn tensors by call index and records the model input times it is called
with, so a trajectory depends on the solver's update path only: the same case through two implementations that
compute the same updates gives the same bits.
"""
import torch

from oracle import synth

SEED = 0
B, SHAPE = 2, (4, 8, 8)
N_DRAWS = 64


class ScriptedModel:
    """model(x, t_input[, cond]) -> base + 0.05 * draw[k]: a smooth field plus a small per-call perturbation, so
    the data predictions stay large (thresholding bites) and the adaptive solver accepts steps."""

    def __init__(self, device):
        base = synth.synth_input("dpms_base", (2 * B,) + SHAPE, SEED)
        self.draws = [(base + 0.05 * synth.synth_input(f"dpms_draw{k}", (2 * B,) + SHAPE, SEED)).to(device)
                      for k in range(N_DRAWS)]
        self.t_inputs = []

    def __call__(self, x, t_input, cond=None):
        k = len(self.t_inputs)
        self.t_inputs.append(float(t_input.reshape(-1)[0]))
        return self.draws[k % N_DRAWS][:x.shape[0]].clone()


def classifier(device):
    """log p(cond | x_t) = sum(w * x): its gradient is w exactly, on any device"""
    w = synth.synth_input("dpms_classifier_w", (B,) + SHAPE, SEED).to(device)
    return lambda x, t_input, cond: (x * w).sum((1, 2, 3))


def x_T(device):
    return synth.synth_input("dpms_xT", (B,) + SHAPE, SEED).to(device)


def _cases():
    c = {}
    for method, orders in (("multistep", (1, 2, 3)), ("singlestep", (1, 2, 3)), ("singlestep_fixed", (2, 3))):
        for order in orders:
            for px in (False, True):
                for st in ("dpm_solver", "taylor"):
                    c[f"{method}-{order}-{'x0' if px else 'eps'}-{st}"] = dict(
                        predict_x0=px, sample=dict(steps=6, order=order, method=method, solver_type=st))
    for skip in ("logSNR", "time_quadratic"):
        for method, order in (("multistep", 2), ("multistep", 3), ("singlestep", 3), ("singlestep_fixed", 2)):
            for px in (False, True):
                c[f"{method}-{order}-{'x0' if px else 'eps'}-{skip}"] = dict(
                    predict_x0=px, sample=dict(steps=6, order=order, method=method, skip_type=skip))
    for steps in (7, 8):
        c[f"singlestep-3-eps-steps{steps}"] = dict(predict_x0=False, sample=dict(steps=steps, order=3))
    c["singlestep-2-x0-steps7"] = dict(predict_x0=True, sample=dict(steps=7, order=2))
    c["multistep-3-x0-steps16"] = dict(predict_x0=True, sample=dict(steps=16, order=3, method="multistep"))
    c["multistep-2-x0-no-lower-final"] = dict(predict_x0=True, sample=dict(steps=6, order=2, method="multistep",
                                                                           lower_order_final=False))
    c["multistep-3-x0-partial"] = dict(predict_x0=True, sample=dict(steps=6, order=3, method="multistep",
                                                                    t_start=0.7, t_end=0.05))
    c["singlestep-3-eps-partial"] = dict(predict_x0=False, sample=dict(steps=6, order=3, t_start=0.8, t_end=0.01))
    c["multistep-3-x0-threshold"] = dict(predict_x0=True, thresholding=True, max_val=1.0,
                                         sample=dict(steps=6, order=3, method="multistep"))
    c["singlestep-3-x0-threshold"] = dict(predict_x0=True, thresholding=True, max_val=1.5,
                                          sample=dict(steps=6, order=3, method="singlestep"))
    c["multistep-2-x0-denoise-to-zero"] = dict(predict_x0=True, sample=dict(steps=6, order=2, method="multistep",
                                                                            denoise_to_zero=True))
    c["singlestep-2-eps-denoise-to-zero"] = dict(predict_x0=False, sample=dict(steps=6, order=2,
                                                                               denoise_to_zero=True))
    c["multistep-3-x0-cfg-x_start"] = dict(predict_x0=True, model_type="x_start", guidance="classifier-free",
                                           scale=3.0, sample=dict(steps=6, order=3, method="multistep"))
    c["singlestep-3-eps-cfg-v"] = dict(predict_x0=False, model_type="v", guidance="classifier-free", scale=3.0,
                                       sample=dict(steps=6, order=3))
    c["multistep-2-x0-cfg-noise"] = dict(predict_x0=True, guidance="classifier-free", scale=7.5,
                                         sample=dict(steps=6, order=2, method="multistep"))
    c["multistep-2-eps-classifier"] = dict(predict_x0=False, guidance="classifier", scale=2.0,
                                           sample=dict(steps=6, order=2, method="multistep"))
    c["multistep-3-x0-linear"] = dict(schedule="linear", predict_x0=True,
                                      sample=dict(steps=6, order=3, method="multistep", skip_type="logSNR"))
    c["singlestep-3-eps-cosine"] = dict(schedule="cosine", predict_x0=False,
                                        sample=dict(steps=6, order=3, skip_type="logSNR"))
    return c


CASES = _cases()
ADAPTIVE = {f"adaptive-{order}-{'x0' if px else 'eps'}": dict(predict_x0=px, sample=dict(order=order, method="adaptive"))
            for order in (2, 3) for px in (False, True)}


def run_case(mod, spec, alphas_cumprod, device):
    """one case through module `mod` (NoiseScheduleVP / model_wrapper / DPM_Solver): (x, model input times)"""
    sched = spec.get("schedule", "discrete")
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=alphas_cumprod) if sched == "discrete" else \
        mod.NoiseScheduleVP(sched)
    model = ScriptedModel(device)
    kw = dict(model_type=spec.get("model_type", "noise"), guidance_type=spec.get("guidance", "uncond"))
    if kw["guidance_type"] == "classifier-free":
        kw.update(condition=torch.ones(B, 1, device=device), unconditional_condition=torch.zeros(B, 1, device=device),
                  guidance_scale=spec["scale"])
    elif kw["guidance_type"] == "classifier":
        kw.update(classifier_fn=classifier(device), guidance_scale=spec["scale"])
    dpm = mod.DPM_Solver(mod.model_wrapper(model, ns, **kw), ns, predict_x0=spec["predict_x0"],
                         thresholding=spec.get("thresholding", False), max_val=spec.get("max_val", 1.))
    with torch.no_grad():
        x = dpm.sample(x_T(device), **spec["sample"])
    return x, model.t_inputs


# end-to-end samples on the tiny finetune model: (predict_x0, sample kwargs)
E2E = {
    "3M++": (True, dict(steps=6, order=3, method="multistep")),
    "singlestep-3": (False, dict(steps=6, order=3, method="singlestep")),
    "singlestep_fixed-2": (True, dict(steps=6, order=2, method="singlestep_fixed")),
    "2M-eps": (False, dict(steps=6, order=2, method="multistep")),
    "adaptive-3": (False, dict(order=3, method="adaptive")),
}
E2E_SCALES = (1.0, 7.5)
