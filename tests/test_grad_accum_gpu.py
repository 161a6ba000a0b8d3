"""Gradient accumulation (accumulate_grad_batches = k, Lightning 1.5 semantics) in FinetuneTrainer / PretrainTrainer:
k = 1 runs the plain trainer's kernels in the same order, a window matches the reference's explicit emulation of Lightning
(tests/golden/tiny_accum_golden.pt from `tools/make_golden.py --accum`), k micro-batches of b match one batch of k*b,
graph replay equals the eager window, an overflow anywhere skips the window, the trainable-weight copies are built once
per window, and flush() applies a partial window with the 1/k factor."""
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

# Bounds of the accumulation comparisons (norm-relative, set about 20 % above the errors measured on an H100 when they were
# introduced, like tolerances.TOL; the tests print what they measure with `pytest -s`).  The shared end-to-end bounds
# (tiny_loss, tiny_grad_norm) come from tolerances.TOL.
ACCUM_TOL = {
    "update": 0.19,         # AdamW update (after - before) of the sampled tensors vs the reference's, after one window
    #                         (worst tensor): the first Adam step is ~lr * g / |g| per element, so elements whose gradient
    #                         is near zero turn the gradients' fp16 noise into sign differences of size ~2 lr; a tensor
    #                         left unstepped or stepped with another set's gradient is off by ~1
    "kb_grad": 2e-3,        # 4 micro-batches of 1 vs one batch of 4: unscaled gradient, same arithmetic summed in another
    #                         order (GEMM tiles / split-K and reductions over M = 4x tokens); the fp32 sums differ in the
    #                         last bits, which flips fp16 roundings of activations downstream
    "kb_update": 0.13,      # the same comparison on the AdamW update (sign noise of near-zero gradients, as above)
    "grad_tensor": 8.5e-3,  # worst full gradient tensor of a 3-micro-batch window vs the reference (sum of three backward
    #                         passes, each at the tiny_grad_tensor level)
    "rerun_grad": 6e-3,     # two runs of the same training steps (float-atomic reductions: GroupNorm / LayerNorm
    #                         statistics and affine gradients, bias column sums, the loss): flat gradient buffer;
    #                         ~1.6e-3 in a first window, ~5e-3 in the second (the first update's noise adds in)
    "rerun_update": 0.13,   # the same, on the AdamW update (after - before) of the flat parameter buffer
}


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


@pytest.fixture(scope="module")
def gold():
    from ctrlora_b200 import dropin
    dropin.activate()
    return load_golden(os.path.join(GOLD, "tiny_accum_golden.pt"))


def make(gold, kind, **kw):
    """a fresh tiny model (synth weights of the golden) and its trainer"""
    from cldm.model import create_model
    from ctrlora_b200.train import FinetuneTrainer, PretrainTrainer
    from oracle import synth
    sub = gold[kind]
    model = create_model(os.path.join(GOLD, f"tiny_{kind}.yaml"), init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(sub["control_shapes"], gold["seed"], "control_model."))
    model.model.diffusion_model.load_state_dict(
        synth.synth_state_dict(gold["finetune"]["unet_shapes"], gold["seed"], "model.diffusion_model."))
    model = model.cuda().eval()
    cls = FinetuneTrainer if kind == "finetune" else PretrainTrainer
    return cls(model, lr=gold["lr"], **kw)


def micro(gold, i):
    """(x0, hint, ctx, t, noise) of the golden's micro-batch i"""
    from oracle import synth
    B, H, seed = gold["B"], gold["H"], gold["seed"]
    mk = lambda n, s: synth.synth_input(f"{n}_acc{i}", s, seed).cuda()
    return (mk("x", (B, 4, H, H)), mk("hint", (B, 4, H, H)), mk("ctx", (B, 77, 64)), gold["t"][i].cuda(),
            mk("noise", (B, 4, H, H)))


def state(tr):
    return [tr.G.flat_p.clone(), tr.G.exp_avg.clone(), tr.G.exp_avg_sq.clone()]


def check_grads(grads, ref_norms, ref_grads):
    """gradient norms of every tensor and the full sampled tensors against the reference; returns the worst errors"""
    live = sorted(v for v in ref_norms.values() if v is not None)
    median, biggest = live[len(live) // 2], live[-1]
    worst, n_unused = 0.0, 0
    for n, rn in ref_norms.items():
        got = grads[n].norm().item()
        if rn is None:  # a LoRA set no micro-batch of the window used
            assert got == 0.0, (n, got)
            n_unused += 1
        elif rn < 1e-5 * biggest:  # exactly-cancelled gradients (32 channels / 32 groups, see test_train_gpu.py)
            assert got < 1e-2 * median, (n, got, rn)
        else:
            err = abs(got - rn) / rn
            worst = max(worst, err)
            assert err < TOL["tiny_grad_norm"], (n, got, rn)
    errs = {n: rel(grads[n], r) for n, r in ref_grads.items()}
    assert max(errs.values()) < ACCUM_TOL["grad_tensor"], errs
    return worst, max(errs.values()), n_unused


def check_update(tr, sub):
    """parameter update (after - before) of the sampled tensors against the reference's AdamW step"""
    params = dict(zip(tr.G.names, tr.G.params))
    errs = {}
    for n, after in sub["after"].items():
        errs[n] = rel(params[n].detach().float().cpu() - sub["before"][n], after - sub["before"][n])
    print("update rel errs:", {k[-40:]: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < ACCUM_TOL["update"], errs


def record_ops(monkeypatch):
    """every ops.* call, in order (what a captured graph contains, or what an eager step launches)"""
    import inspect
    from ctrlora_b200 import ops
    seq = []

    def wrap(name, fn):
        def rec(*a, **kw):
            seq.append(name)
            return fn(*a, **kw)
        return rec

    for name, fn in list(vars(ops).items()):
        if inspect.isfunction(fn) and fn.__module__ == ops.__name__ and not name.startswith("_"):
            monkeypatch.setattr(ops, name, wrap(name, fn))
    return seq


def rerun_close(a, b, p0):
    """Two runs of the same training step are not bit-identical: the GroupNorm / LayerNorm statistics and affine
    gradients, the bias column sums and the loss reduce across CTAs with float atomics, so their fp32 sums (and the fp16
    activations rounded from them) differ in the last bits from run to run.  Bounds: ACCUM_TOL["rerun_*"]."""
    e_g = rel(a.G.flat_g, b.G.flat_g)
    e_u = rel(a.G.flat_p - p0, b.G.flat_p - p0)
    print(f"rerun: gradient rel diff {e_g:.2e}, update rel diff {e_u:.2e}")
    assert e_g < ACCUM_TOL["rerun_grad"] and e_u < ACCUM_TOL["rerun_update"]


@pytest.mark.parametrize("graphed", [False, True])
def test_k1_is_the_plain_trainer(gold, graphed, monkeypatch):
    """accumulate_grad_batches=1 runs the same kernels in the same order as a trainer built without it (recorded ops
    sequence of the eager steps, or of the captures), and reaches the same state up to the run-to-run atomics noise.
    Every step returns a loss tensor of its own (a replayed graph's loss is overwritten by its next replay)."""
    a, b = make(gold, "finetune"), make(gold, "finetune", accumulate_grad_batches=1)
    p0 = a.G.flat_p.clone()
    seqs, losses = [], []
    for tr in (a, b):
        seq = record_ops(monkeypatch)
        if graphed:
            tr.capture(*micro(gold, 0))
        losses.append([tr.step(*micro(gold, i)) for i in range(2)])
        seqs.append(list(seq))
        monkeypatch.undo()
    torch.cuda.synchronize()
    assert len(seqs[0]) > 100 and seqs[0] == seqs[1]
    for first, second in losses:
        assert first is not second and first.item() != second.item()
    rerun_close(a, b, p0)
    assert a.step_count == b.step_count == 2 and b.micro_step == 0


def test_finetune_window_vs_reference(gold):
    sub = gold["finetune"]
    tr = make(gold, "finetune", accumulate_grad_batches=3)
    assert tr.G.names == sub["trainable_names"]
    losses = []
    for i in range(3):
        assert tr.step_count == 0 and tr.micro_step == i
        losses.append(tr.step(*micro(gold, i)).item())
    assert tr.step_count == 1 and tr.micro_step == 0
    e_loss = max(abs(l - r) / abs(r) for l, r in zip(losses, sub["losses"].tolist()))
    inv = 1.0 / (tr._scale_used * 3)
    grads = {n: g * inv for n, g in tr.G.named_grads().items()}
    worst, worst_t, _ = check_grads(grads, sub["grad_norms"], sub["grads"])
    print(f"finetune window: loss rel err {e_loss:.2e}, grad norm {worst:.2e}, tensor {worst_t:.2e}")
    assert e_loss < TOL["tiny_loss"]
    check_update(tr, sub)


def test_pretrain_mixed_task_window_vs_reference(gold):
    sub = gold["pretrain"]
    tr = make(gold, "pretrain", accumulate_grad_batches=3)
    assert tr.G.names == sub["param_names"]
    off, n = tr.layout["lora"]["seg"]
    seg0 = [t[off:off + n].clone() for t in state(tr)]
    losses = [tr.step(*micro(gold, i), task=task).item() for i, task in enumerate(sub["tasks"])]
    torch.cuda.synchronize()
    e_loss = max(abs(l - r) / abs(r) for l, r in zip(losses, sub["losses"].tolist()))
    inv = 1.0 / (tr._scale_used * 3)
    grads = {n: g * inv for n, g in tr.G.named_grads().items()}
    worst, worst_t, n_unused = check_grads(grads, sub["grad_norms"], sub["grads"])
    print(f"pretrain window: loss rel err {e_loss:.2e}, grad norm {worst:.2e}, tensor {worst_t:.2e}")
    assert e_loss < TOL["tiny_loss"] and n_unused == 2 * 82
    for before, now in zip(seg0, state(tr)):
        assert torch.equal(before, now[off:off + n])  # seg: no update, no decay, no moments
    assert tr.seg_steps == {"base": 1, "canny": 1, "depth": 1} and tr.step_count == 1
    check_update(tr, sub)


def test_k_micro_batches_equal_one_batch_of_k_b(gold):
    """4 micro-batches of 1 vs one batch of 4 from the same samples, timesteps and noise.  Same arithmetic; the GEMM tile
    and split-K choices and the weight-gradient / column-sum reductions run over M = 4 * tokens instead of 4 separate M,
    so the fp32 sums are ordered differently: last-bit differences, bounded by ACCUM_TOL["kb_grad"]."""
    big = make(gold, "finetune")
    acc = make(gold, "finetune", accumulate_grad_batches=4)
    full = [torch.cat([micro(gold, 0)[j], micro(gold, 1)[j]]) for j in range(5)]
    p0 = big.G.flat_p.clone()
    big.step(*full)
    for i in range(4):
        acc.step(*[v[i:i + 1] for v in full])
    torch.cuda.synchronize()
    g_big = big.G.flat_g / big._scale_used
    g_acc = acc.G.flat_g / (acc._scale_used * 4)
    e_g = rel(g_acc, g_big)
    e_u = rel(acc.G.flat_p - p0, big.G.flat_p - p0)
    print(f"k*b equivalence: gradient rel diff {e_g:.2e}, update rel diff {e_u:.2e}")
    assert e_g < ACCUM_TOL["kb_grad"] and e_u < ACCUM_TOL["kb_update"]


def test_captured_window_equals_eager_window(gold):
    """Captured windows (pretrain, mixed tasks; finetune, segmented at the overlap cuts) against eager ones: the same
    kernels in the same order, equal up to the run-to-run noise of the float-atomic reductions (rerun_close)."""
    tasks = [["canny", "depth", "canny"], ["seg", "seg", "depth"]]
    eager, graph = (make(gold, "pretrain", accumulate_grad_batches=3) for _ in range(2))
    p0 = eager.G.flat_p.clone()
    graph.capture(*micro(gold, 0))
    for window in tasks:
        for i, task in enumerate(window):
            le = eager.step(*micro(gold, i), task=task)
            lg = graph.step(*micro(gold, i), task=task)
            assert abs(le.item() - lg.item()) <= TOL["tiny_loss"] * abs(le.item()), (window, i)
        torch.cuda.synchronize()
        rerun_close(eager, graph, p0)
    assert eager.seg_steps == graph.seg_steps == {"base": 2, "canny": 1, "depth": 2, "seg": 1}

    eager, graph = (make(gold, "finetune", accumulate_grad_batches=3) for _ in range(2))
    p0 = eager.G.flat_p.clone()
    for tr in (eager, graph):
        tr.allreduce_cuts = "middle,ib9,ib6,ib3"
    graph._segmented = lambda: True  # one graph per bucket even on one GPU (the all-reduces are no-ops there)
    graph.capture(*micro(gold, 0))
    assert isinstance(graph._graphs["compute"][None][0], list) and len(graph._graphs["compute"][None][0]) == 5
    for _ in range(2):
        for i in range(3):
            le, lg = eager.step(*micro(gold, i)), graph.step(*micro(gold, i))
            assert abs(le.item() - lg.item()) <= TOL["tiny_loss"] * abs(le.item())
        torch.cuda.synchronize()
        rerun_close(eager, graph, p0)


def test_overflow_anywhere_in_the_window_skips_it(gold):
    tr = make(gold, "finetune", accumulate_grad_batches=3)
    tr.CHECK_OVERFLOW_EVERY = 1
    for i in range(3):
        tr.step(*micro(gold, i))
    before, steps, scale = state(tr), tr.step_count, tr._scale_used
    x0, hint, ctx, t, noise = micro(gold, 1)
    for i, args in enumerate((micro(gold, 0), (x0, hint, ctx, t, noise * 1e6), micro(gold, 2))):
        tr.step(*args)  # the middle micro-batch's fp16 loss gradient overflows
    torch.cuda.synchronize()
    assert tr.skipped_steps == 1 and tr.step_count == steps == tr.seg_steps["all"] == 1
    for x, y in zip(before, state(tr)):
        assert torch.equal(x, y)
    assert tr.loss_scale == 0.5 * scale
    for i in range(3):
        tr.step(*micro(gold, i))
    torch.cuda.synchronize()
    assert tr._scale_used == 0.5 * scale and tr.step_count == 2 and tr.skipped_steps == 1
    assert not torch.equal(tr.G.flat_p, before[0])


def test_weight_copies_built_once_per_window(gold, monkeypatch):
    from ctrlora_b200 import prepare
    calls = []
    orig = prepare.effective_linear_weight

    def counting(lin, out=None):
        calls.append(id(lin))
        return orig(lin, out=out)

    monkeypatch.setattr(prepare, "effective_linear_weight", counting)
    one = make(gold, "finetune")
    one.step(*micro(gold, 0))        # first step also builds the frozen copies
    calls.clear()
    one.step(*micro(gold, 1))
    per_step = len(calls)
    acc = make(gold, "finetune", accumulate_grad_batches=4)
    for i in range(4):
        acc.step(*micro(gold, i % 3))
    per_micro = []
    for i in range(4):
        calls.clear()
        acc.step(*micro(gold, i % 3))
        per_micro.append(len(calls))
    print("effective_linear_weight calls: one step", per_step, "micro-batches of a window", per_micro)
    assert per_step > 0 and per_micro == [per_step, 0, 0, 0]


def test_flush_applies_a_partial_window_with_1_over_k(gold):
    four = make(gold, "finetune", accumulate_grad_batches=4)
    two = make(gold, "finetune", accumulate_grad_batches=2)
    p0 = four.G.flat_p.clone()
    for i in range(2):
        four.step(*micro(gold, i))
        two.step(*micro(gold, i))
    assert four.step_count == 0 and four.micro_step == 2
    four.flush()
    torch.cuda.synchronize()
    assert four.step_count == 1 and four.micro_step == 0
    e_g = rel(four.G.flat_g, two.G.flat_g)  # same kernels and order; atomics noise only (rerun_close)
    assert e_g < ACCUM_TOL["rerun_grad"], e_g
    p_ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([p_ref], lr=gold["lr"])
    p_ref.grad = four.G.flat_g / four._scale_used / 4
    opt.step()
    assert (four.G.flat_p - p_ref.detach()).abs().max().item() < 2e-6  # (g * 1/(scale k)) vs (g / scale / k): 1 ulp
    after = state(four)
    four.flush()  # empty window
    torch.cuda.synchronize()
    assert four.step_count == 1
    for x, y in zip(after, state(four)):
        assert torch.equal(x, y)
