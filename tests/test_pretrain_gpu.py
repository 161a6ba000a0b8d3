"""Pretraining step parity (BASELINE.json configs[3]; reference cldm/cldm_ctrlora_pretrain.py:88-111,174-182): loss and
the gradient of EVERY ControlNet parameter (dense conv / linear weights and biases, norms, zero-convs, time-embedding MLP)
plus the mini-batch task's LoRA set, against the unmodified reference's autograd on the tiny config
(tests/golden/tiny_variants_golden.pt: norms for all tensors, full tensors for a sample)."""
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
    from ctrlora_b200.train import PretrainTrainer
    from oracle import synth
    g = load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))
    model = create_model(os.path.join(GOLD, "tiny_pretrain.yaml"), init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(g["pretrain_control_shapes"], g["seed"], "control_model."))
    model.model.diffusion_model.load_state_dict(synth.synth_state_dict(g["unet_shapes"], g["seed"], "model.diffusion_model."))
    model = model.cuda().eval()
    trainer = PretrainTrainer(model, lr=1e-3)
    B, H, seed = g["B"], g["H"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    d = dict(x0=mk("x", (B, 4, H, H)), hint=mk("hint", (B, 4, H, H)), ctx=mk("ctx", (B, 77, 64)),
             noise=mk("noise", (B, 4, H, H)), t=g["t"].cuda())
    return g, model, trainer, d


def test_parameter_set_is_the_reference_optimizers(setup):
    g, model, trainer, d = setup
    # the reference lists control_model.parameters() before any switch_lora: ControlNet parameters, then loras_dict.*
    names = trainer.G.names
    assert all(".lora_layer." not in n for n in names)
    base = [n for n in names if not n.startswith("loras_dict.")]
    assert names[:len(base)] == base and len(names) - len(base) == 3 * 2 * 82
    assert trainer.G.numel == sum(p.numel() for p in model.control_model.parameters())
    # state-dict contract survives the kernel-order storage of conv weights
    sd = model.control_model.state_dict()
    assert list(sd.keys()) == g["pretrain_key_order"]
    w = sd["input_blocks.1.0.in_layers.2.weight"]
    assert tuple(w.shape) == (32, 32, 3, 3)
    from oracle import synth
    ref = synth.synth_param("control_model.input_blocks.1.0.in_layers.2.weight", w.shape, g["seed"])
    assert torch.equal(w.cpu(), ref)


def test_pretrain_loss_and_all_gradients_vs_reference_autograd(setup):
    g, model, trainer, d = setup
    loss = trainer.loss_and_grads(d["x0"], d["hint"], d["ctx"], d["t"], d["noise"], task="depth")
    torch.cuda.synchronize()
    e_eps = rel(trainer.last_eps, g["pretrain_train_eps"])
    e_loss = abs(loss.item() - g["pretrain_loss"].item()) / abs(g["pretrain_loss"].item())
    print(f"pretrain eps rel err {e_eps:.2e}, loss rel err {e_loss:.2e}")
    assert e_eps < TOL["tiny_eps"] and e_loss < TOL["tiny_loss"]
    inv = 1.0 / trainer._scale_used
    api = trainer.G._api_grad
    grads = {n: api[id(p)] * inv for n, p in model.control_model.named_parameters()}  # same aliasing as the reference's names
    assert list(grads.keys()) == g["pretrain_param_names"]
    ref_norms = g["pretrain_grad_norms"]
    live = sorted(v for v in ref_norms.values() if v is not None)
    median, biggest = live[len(live) // 2], live[-1]
    worst, worst_name, n_unused, n_zero = 0.0, None, 0, 0
    for n, rn in ref_norms.items():
        got = grads[n].norm().item()
        if rn is None:  # LoRA sets of the other tasks: never reached
            assert got == 0.0, (n, got)
            n_unused += 1
        elif rn < 1e-5 * biggest:  # exactly-cancelled gradients (32 channels / 32 groups, see test_train_gpu.py)
            assert got < 1e-2 * median, (n, got, rn)
            n_zero += 1
        else:
            err = abs(got - rn) / rn
            if err > worst:
                worst, worst_name = err, n
    errs = {n: rel(grads[n], r) for n, r in g["pretrain_grads"].items()}
    print(f"{len(ref_norms)} tensors: worst grad-norm err {worst:.2e} ({worst_name}), {n_unused} unused, {n_zero} cancelled")
    print("full-tensor rel errs:", {k[-46:]: "%.1e" % v for k, v in errs.items()})
    assert n_unused == 2 * 2 * 82
    assert worst < TOL["tiny_grad_norm"] and max(errs.values()) < TOL["tiny_grad_tensor"]


def test_pretrain_step_switches_tasks_and_skips_unused_sets(setup):
    g, model, trainer, d = setup
    args = (d["x0"], d["hint"], d["ctx"], d["t"], d["noise"])
    lay = trainer.layout
    snap = lambda key: trainer.G.flat_p[lay["lora"][key][0]:lay["lora"][key][0] + lay["lora"][key][1]].clone()
    before = {t: snap(t) for t in trainer.tasks}
    base0 = trainer.G.flat_p[:lay["base"][1]].clone()
    l0 = trainer.step(*args, task="canny").item()
    assert not torch.equal(snap("canny"), before["canny"])
    assert torch.equal(snap("depth"), before["depth"]) and torch.equal(snap("seg"), before["seg"])  # no decay, no moments
    assert not torch.equal(trainer.G.flat_p[:lay["base"][1]], base0)
    trainer.step(*args, task="seg")
    assert trainer.seg_steps == {"base": 2, "canny": 1, "seg": 1}
    losses = [l0] + [trainer.step(*args, task="canny").item() for _ in range(4)]
    print("pretrain losses on one batch (task canny):", ["%.5f" % v for v in losses])
    assert losses[-1] < losses[0]
    # graph replay per task gives the same loss as the eager step would on the same weights
    trainer.capture(*args, tasks=["canny", "depth"], warmup=1)
    a = trainer.step(*args, task="depth").item()
    b = trainer.step(*args, task="canny").item()
    assert a == a and b == b and b < losses[0]


def test_full_parameter_finetune_is_refused_by_the_lora_sink_and_served_by_the_dense_trainer():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.cldm_ctrlora_finetune import ControlNetFinetune
    from ctrlora_b200.train import GradSink
    from test_variants_gpu import KW, randomize_
    cn = ControlNetFinetune(ft_with_lora=False, **KW)
    randomize_(cn, 3)
    cn = cn.cuda()
    with pytest.raises(NotImplementedError):
        GradSink(cn)


@pytest.mark.parametrize("kind", ["pretrain", "finetune"])
def test_gradient_buckets_are_final_when_their_stage_fires(setup, kind):
    """The overlapped exchange starts a bucket's all-reduce when the backward reaches its stage: every gradient of the
    bucket must already hold its final value then (single GPU: snapshot at the stage, compare after the backward).  The
    ResBlocks' emb_layers are differentiated after the last block and therefore belong to the final bucket."""
    g, model, trainer, d = setup
    if kind == "finetune":
        from ctrlora_b200 import dropin
        dropin.activate()
        from cldm.model import create_model
        from ctrlora_b200.train import FinetuneTrainer
        from oracle import synth
        g2 = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
        m2 = create_model(os.path.join(GOLD, "tiny_finetune.yaml"), init_weights=False)
        m2.control_model.load_state_dict(synth.synth_state_dict(g2["control_shapes"], g2["seed"], "control_model."))
        m2.model.diffusion_model.load_state_dict(synth.synth_state_dict(g2["unet_shapes"], g2["seed"], "model.diffusion_model."))
        trainer = FinetuneTrainer(m2.cuda().eval(), lr=1e-3)
    trainer.allreduce_cuts = "middle,ib9,ib6,ib3"
    buckets = dict(trainer.merged_buckets())
    assert set(buckets) == {"middle", "ib9", "ib6", "ib3", "final"}
    covered = sorted(r for rs in buckets.values() for r in rs)
    assert sum(n for _, n in covered) == trainer.G.numel and all(a[0] + a[1] <= b[0] for a, b in zip(covered, covered[1:]))
    snaps = {}

    def on_stage(name):
        snaps[name] = [trainer.G.flat_g[off:off + n].clone() for off, n in buckets[name]]

    trainer._on_stage = on_stage
    try:
        args = (d["x0"], d["hint"], d["ctx"], d["t"], d["noise"])
        trainer.loss_and_grads(*args, task="depth") if kind == "pretrain" else trainer.loss_and_grads(*args)
    finally:
        trainer._on_stage = None
        trainer.allreduce_cuts = None
    torch.cuda.synchronize()
    assert set(snaps) == {"middle", "ib9", "ib6", "ib3"}
    for name, tensors in snaps.items():
        nonzero = 0
        for (off, n), snap in zip(buckets[name], tensors):
            assert torch.equal(snap, trainer.G.flat_g[off:off + n]), f"bucket {name} changed after its stage"
            nonzero += int(snap.abs().sum().item() > 0)
        assert nonzero > 0, f"bucket {name} was still empty at its stage"
