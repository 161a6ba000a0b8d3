"""Resuming the trainers from a checkpoint (save_checkpoint / load_checkpoint, ctrlora_b200.checkpoint) on the GPU:
the restored state takes the same AdamW step as the state it was saved from (bit for bit, from the same gradient buffer:
the backward itself is not bit-reproducible, see test_grad_accum_gpu.rerun_close), for eager and captured trainers,
accumulation windows, a checkpoint after an overflow-skipped step and a pretrain LoRA set unused at save time; the op
sequence of a step after loading; and the exchange with the reference's torch.optim.AdamW state
(tests/golden/tiny_resume_golden.pt from `tools/make_golden.py --resume`)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu

from golden_io import load_golden  # noqa: E402
from test_grad_accum_gpu import ACCUM_TOL, record_ops, rel, rerun_close  # noqa: E402

# Bounds against the reference (norm-relative, worst tensor; set about 20 % above the errors measured on an H100, like
# tolerances.TOL; the tests print what they measure with `pytest -s`).
RESUME_TOL = {
    "exp_avg": 9e-3,        # m = (1 - b1) g after one step (and its pretrain sums after two): the gradient tensors' error
    #                         (tiny_grad_tensor level; worst of four runs 7.5e-3); a layout or index error is off by ~1
    "exp_avg_sq": 1.3e-2,   # v = (1 - b2) g^2: up to twice the gradient's relative error (worst of four runs 1.08e-2)
    "update": 1.7e-2,       # AdamW update of the sampled tensors in the step after loading (worst of four runs 1.4e-2, a
    #                         LoRA `down`: sign noise of near-zero gradients, as ACCUM_TOL["update"]); a wrong step count
    #                         (bias correction) or moment layout (direction) is off by ~1
}


@pytest.fixture(scope="module")
def gold():
    from ctrlora_b200 import dropin
    dropin.activate()
    return load_golden(os.path.join(GOLD, "tiny_resume_golden.pt"))


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


def micro(gold, i, noise_scale=1.0):
    """(x0, hint, ctx, t, noise) of the golden's micro-batch i"""
    from oracle import synth
    B, H, seed = gold["B"], gold["H"], gold["seed"]
    mk = lambda n, s: synth.synth_input(f"{n}_acc{i}", s, seed).cuda()
    return (mk("x", (B, 4, H, H)), mk("hint", (B, 4, H, H)), mk("ctx", (B, 77, 64)), gold["t"][i].cuda(),
            mk("noise", (B, 4, H, H)) * noise_scale)


def counters(tr):
    return (tr.step_count, dict(tr.seg_steps), tr.loss_scale, tr.skipped_steps)


def bufs(tr):
    return [tr.G.flat_p, tr.G.exp_avg, tr.G.exp_avg_sq]


def same_update(a, b, args, task=None):
    """one AdamW update on a and b from a's gradient buffer: bit-identical results"""
    kw = {} if task is None else {"task": task}
    a.loss_and_grads(*args, **kw)
    b.G.flat_g.copy_(a.G.flat_g)
    b._scale_used = a._scale_used
    segs = a.window_segments([task])
    a._update(segs)
    b._update(segs)
    torch.cuda.synchronize()
    for x, y in zip(bufs(a), bufs(b)):
        assert torch.equal(x, y)
    assert counters(a) == counters(b)


CASES = {  # name: (kind, trainer kwargs, capture, tasks of the steps before saving)
    "finetune": ("finetune", {}, False, [None] * 2),
    "finetune_graphed": ("finetune", {}, True, [None] * 2),
    "finetune_accum2": ("finetune", {"accumulate_grad_batches": 2}, False, [None] * 4),
    "finetune_accum2_graphed": ("finetune", {"accumulate_grad_batches": 2}, True, [None] * 4),
    "pretrain_unused_set": ("pretrain", {}, False, ["canny", "depth"]),
    "pretrain_graphed": ("pretrain", {}, True, ["canny", "depth"]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_same_step_from_the_restored_state(gold, case, tmp_path):
    kind, kw, graphed, tasks = CASES[case]
    a, b = make(gold, kind, **kw), make(gold, kind, **kw)
    tkw = (lambda t: {}) if kind == "finetune" else (lambda t: {"task": t})
    if graphed:  # b's graphs exist before it loads
        for tr in (a, b):
            tr.capture(*micro(gold, 0))
    for i, task in enumerate(tasks):
        a.step(*micro(gold, i % 3), **tkw(task))
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)
    b.load_checkpoint(path)
    torch.cuda.synchronize()
    for x, y in zip(bufs(a), bufs(b)):
        assert torch.equal(x, y)
    assert counters(a) == counters(b)
    if kind == "pretrain":
        assert a.seg_steps == {"base": 2, "canny": 1, "depth": 1}
        off, n = b.layout["lora"]["seg"]
        assert not b.G.exp_avg[off:off + n].any() and "seg" not in b.seg_steps
    next_task = None if kind == "finetune" else "seg"  # pretrain: the set unused at save time
    same_update(a, b, micro(gold, 2), next_task)
    if kind == "pretrain":
        assert a.seg_steps == b.seg_steps == {"base": 3, "canny": 1, "depth": 1, "seg": 1}
    # whole steps after resume: equal up to the run-to-run noise of the backward's float atomics
    p0 = a.G.flat_p.clone()
    k = kw.get("accumulate_grad_batches", 1)
    for i in range(k):
        for tr in (a, b):
            tr.step(*micro(gold, (i + 1) % 3), **tkw("canny"))
    torch.cuda.synchronize()
    rerun_close(a, b, p0)
    assert counters(a) == counters(b)
    if kind == "pretrain":
        assert b.seg_steps == {"base": 4, "canny": 2, "depth": 1, "seg": 1}


def test_checkpoint_after_an_overflow_skipped_step(gold, tmp_path):
    a, b = make(gold, "finetune"), make(gold, "finetune")
    for i in range(2):
        a.step(*micro(gold, i))
    a.step(*micro(gold, 2, noise_scale=1e6))  # the fp16 loss gradient overflows: skipped on the device, not yet polled
    scale = a._scale_used
    assert a.step_count == 3 and a.skipped_steps == 0
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)  # polls: the step is uncounted and the scale halved before anything is written
    assert (a.step_count, a.seg_steps, a.skipped_steps, a.loss_scale) == (2, {"all": 2}, 1, 0.5 * scale)
    b.load_checkpoint(path)
    assert counters(a) == counters(b)
    for x, y in zip(bufs(a), bufs(b)):
        assert torch.equal(x, y)
    same_update(a, b, micro(gold, 0))
    assert b._scale_used == 0.5 * scale and b.step_count == 3


def test_op_sequence_after_load_equals_a_fresh_trainers(gold, tmp_path, monkeypatch):
    a = make(gold, "finetune")
    a.step(*micro(gold, 0))
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)
    fresh, loaded = make(gold, "finetune"), make(gold, "finetune")
    seqs = []
    for tr, load in ((fresh, False), (loaded, True)):
        seq = record_ops(monkeypatch)
        if load:
            tr.load_checkpoint(path)
            assert not seq, "loading launches no kernel of the library"
        tr.step(*micro(gold, 1))
        seqs.append(list(seq))
        monkeypatch.undo()
    assert len(seqs[0]) > 100 and seqs[0] == seqs[1]


def check_moments(ours, ref_state, names, which):
    """moments tensor by tensor against the reference's; returns the worst norm-relative errors"""
    worst = {}
    for k in ("exp_avg", "exp_avg_sq"):
        norms = {i: s[k].norm().item() for i, s in ref_state.items()}
        biggest = max(norms.values())
        errs = {}
        for i, s in ref_state.items():
            if norms[i] < 1e-5 * biggest:  # exactly-cancelled gradients (32 channels / 32 groups, see test_train_gpu.py)
                assert ours[i][k].norm().item() < 1e-3 * biggest, (names[i], k)
                continue
            errs[names[i]] = rel(ours[i][k], s[k])
        worst[k] = max(errs.values())
        print(f"{which} {k}: worst rel err {worst[k]:.2e} ({max(errs, key=errs.get)}) over {len(errs)} tensors")
        assert worst[k] < RESUME_TOL[k], (k, sorted(errs.items(), key=lambda e: -e[1])[:3])
    return worst


def check_update(params, before, after, ref_before, which):
    errs = {n: rel(params[n].detach().float().cpu() - before[n], after[n] - ref_before[n]) for n in after}
    print(f"{which} update rel errs:", {k[-40:]: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < RESUME_TOL["update"], errs


def test_finetune_vs_reference(gold, tmp_path):
    sub = gold["finetune"]
    names = sub["trainable_names"]
    # our state after step 1 against the reference's opt.state_dict()
    a = make(gold, "finetune")
    assert a.G.names == names
    a.step(*micro(gold, 0))
    out = a.state_dict()["optimizer"]
    ref_state = gold["ft_state1"]
    assert sorted(out["state"]) == sorted(ref_state) == list(range(len(names)))
    assert all(int(s["step"]) == int(ref_state[i]["step"]) == 1 for i, s in out["state"].items())
    check_moments(out["state"], ref_state, names, "finetune step 1")
    # the reference's step-1 state (weights + optimizer_states) in a Lightning-layout file, loaded into a fresh trainer:
    # its step 2 reproduces the reference's
    b = make(gold, "finetune")
    sd = {k: v.detach().cpu().clone() for k, v in b.model.state_dict().items()}
    for n in names:
        sd["control_model." + n] = gold["ft_params1"][n]
    sd["cond_stage_model.transformer.text_model.embeddings.position_ids"] = torch.arange(77)[None]  # not shipped
    path = str(tmp_path / "reference.ckpt")
    torch.save({"epoch": 0, "global_step": 1, "pytorch-lightning_version": "1.5.0", "state_dict": sd,
                "optimizer_states": [{"state": ref_state, "param_groups": sub["param_groups1"]}], "lr_schedulers": [],
                "callbacks": {}}, path)
    b.load_checkpoint(path)
    assert b.step_count == 1 and b.seg_steps == {"all": 1} and b.loss_scale is None
    params = dict(zip(b.G.names, b.G.params))
    before = {n: params[n].detach().float().cpu().clone() for n in sub["after2"]}
    assert all(torch.equal(before[n], gold["ft_params1"][n]) for n in before)
    b.step(*micro(gold, 1))
    torch.cuda.synchronize()
    check_update(params, before, sub["after2"], {n: gold["ft_params1"][n] for n in sub["after2"]}, "finetune step 2")


def test_pretrain_vs_reference(gold, tmp_path):
    sub = gold["pretrain"]
    a = make(gold, "pretrain")
    assert a.G.names == sub["index_names"]
    a.step(*micro(gold, 0), task="canny")
    a.step(*micro(gold, 1), task="depth")
    out = a.state_dict()["optimizer"]
    assert {i: int(s["step"]) for i, s in out["state"].items()} == sub["steps"]
    for k in ("lr", "betas", "eps", "weight_decay", "amsgrad", "maximize"):
        assert out["param_groups"][0][k] == sub["param_group"][k], k
    idx = {n: i for i, n in enumerate(sub["index_names"])}
    assert any(v["exp_avg"].dim() == 4 and v["exp_avg"].shape[-1] == 3 for v in sub["moments"].values())
    check_moments({idx[n]: out["state"][idx[n]] for n in sub["moments"]},
                  {idx[n]: m for n, m in sub["moments"].items()}, sub["index_names"], "pretrain [canny],[depth]")
    # through a file into a fresh trainer; the third step trains the set unused so far (seg at step 1, base at step 3)
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)
    b = make(gold, "pretrain")
    b.load_checkpoint(path)
    params = dict(zip(b.G.names, b.G.params))
    before = {n: params[n].detach().float().cpu().clone() for n in sub["after3"]}
    b.step(*micro(gold, 2), task="seg")
    torch.cuda.synchronize()
    assert b.seg_steps == {"base": 3, "canny": 1, "depth": 1, "seg": 1}
    check_update(params, before, sub["after3"], sub["before3"], "pretrain step 3")
