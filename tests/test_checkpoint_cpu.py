"""Trainer checkpoints on CPU (ctrlora_b200.checkpoint): the trainers' flat AdamW state exchanged bit for bit with
torch.optim.AdamW's state_dict() over the reference's parameter list (3x3 conv moments in the reference layout, per-LoRA-set
step counts, fresh sets), the Lightning-layout file round trip, the refusals, and rank-0-only writing under gloo.  The
trainers construct on CPU; no kernel runs here.  The GPU side is tests/test_checkpoint_resume_gpu.py."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

# pretrain: which LoRA sets get a gradient in each torch step (base every step): base 3, canny 2, depth 1, seg none
PRETRAIN_STEPS = [["canny"], ["depth"], ["canny"]]


def make(kind, seed=0, **kw):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ctrlora_b200.train import FinetuneTrainer, PretrainTrainer
    torch.manual_seed(seed)
    model = create_model(os.path.join(GOLD, f"tiny_{kind}.yaml"))
    return (FinetuneTrainer if kind == "finetune" else PretrainTrainer)(model, lr=1e-3, **kw)


def torch_adamw(tr, kind, seed=1):
    """torch.optim.AdamW over the trainer's own (aliased) parameters with synthetic gradients; returns the optimizer"""
    opt = torch.optim.AdamW(tr.G.params, lr=1e-3, weight_decay=0.01)
    gen = torch.Generator().manual_seed(seed)
    steps = [[]] * 3 if kind == "finetune" else PRETRAIN_STEPS
    for tasks in steps:
        opt.zero_grad(set_to_none=True)
        for n, p in zip(tr.G.names, tr.G.params):
            if not n.startswith("loras_dict.") or n.split(".")[1] in tasks:
                p.grad = torch.randn(p.shape, generator=gen) * 1e-2
        opt.step()
    for p in tr.G.params:
        p.grad = None
    return opt


def storage_order(t):
    """a reference-shape tensor flattened in the trainers' storage order (conv weights [Cout, kh, kw, Cin])"""
    return (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(-1)


def assert_same_state(a, b):
    assert sorted(a["state"]) == sorted(b["state"])
    for i, s in a["state"].items():
        t = b["state"][i]
        assert s.keys() == t.keys() and torch.equal(s["step"], t["step"]), i
        for k in ("exp_avg", "exp_avg_sq"):
            assert s[k].shape == t[k].shape and torch.equal(s[k], t[k]), (i, k)
    assert a["param_groups"] == b["param_groups"]


@pytest.mark.parametrize("kind", ["finetune", "pretrain"])
def test_bit_exact_exchange_with_torch_adamw(kind):
    tr = make(kind)
    opt = torch_adamw(tr, kind)
    ref = opt.state_dict()
    G = tr.G
    if kind == "pretrain":  # a set the trainer had stepped but the state has none of must come back fresh
        off, n = tr.layout["lora"]["seg"]
        G.exp_avg[off:off + n] = 1.0
        tr._seg_state("seg")[0].fill_(5)
        tr.seg_steps["seg"] = 5
    tr.load_state_dict(ref)
    n_conv3 = 0
    for i, (name, p) in enumerate(zip(G.names, G.params)):
        off, n = G.offsets[name]
        st = ref["state"].get(i)
        for k, buf in (("exp_avg", G.exp_avg), ("exp_avg_sq", G.exp_avg_sq)):
            want = storage_order(st[k]) if st is not None else torch.zeros(n)
            assert torch.equal(buf[off:off + n], want), (name, k)
        n_conv3 += p.dim() == 4 and p.shape[-1] == 3 and st is not None
    if kind == "pretrain":
        assert n_conv3 > 20, "the 3x3 conv moments are the layout the finetune set cannot check"
        assert tr.seg_steps == {"base": 3, "canny": 2, "depth": 1}
        assert {k: int(v) for k, v in tr._step_dev.items()} == {"base": 3, "canny": 2, "depth": 1, "seg": 0}
        assert len(ref["state"]) == 324 + 2 * 164
    else:
        assert tr.seg_steps == {"all": 3} and int(tr._step_dev["all"]) == 3 and len(ref["state"]) == 246
    assert tr.step_count == 3
    b1, b2 = tr.betas
    key = "all" if kind == "finetune" else "depth"
    step = tr.seg_steps[key]
    assert torch.equal(tr._bc_dev[key], torch.tensor([1 - b1 ** step, 1 - b2 ** step]))
    out = tr.state_dict()["optimizer"]
    assert_same_state(out, ref)
    torch.optim.AdamW(tr.G.params, lr=1e-3).load_state_dict(out)


def test_hyper_parameters_come_from_the_state():
    tr = make("finetune")
    opt = torch_adamw(tr, "finetune")
    for g in opt.param_groups:
        g.update(lr=3e-4, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.1)
    tr.load_state_dict(opt.state_dict())
    assert (tr.lr, tr.betas, tr.eps, tr.wd) == (3e-4, (0.8, 0.99), 1e-6, 0.1)


def extract_lora(ckpt):      # scripts/tool_extract_weights.py:22-33
    return {k: v for k, v in ckpt.items() if 'control_model' in k and 'loras_dict' not in k and (
        'lora_layer' in k or 'zero_convs' in k or 'middle_block_out' in k or 'norm' in k)}


@pytest.mark.parametrize("kind", ["finetune", "pretrain"])
def test_file_round_trip(kind, tmp_path):
    from cldm.model import get_state_dict
    from ctrlora_b200.checkpoint import EXTRA_KEY
    a = make(kind)
    a.load_state_dict(torch_adamw(a, kind).state_dict())
    a.loss_scale, a.skipped_steps = 128.0, 2
    if kind == "pretrain":
        a.cn.switch_lora("depth")  # the file carries depth's set under the lora_layer aliases too
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path, epoch=4)
    ckpt = torch.load(path, weights_only=True)
    assert ckpt["epoch"] == 4 and ckpt["global_step"] == 3
    assert ckpt[EXTRA_KEY] == {"loss_scale": 128.0, "skipped_steps": 2, "accumulate_grad_batches": 1}
    sd = ckpt["state_dict"]
    assert list(sd) == list(a.model.state_dict())
    for k, v in sd.items():
        assert v.is_contiguous() and v.untyped_storage().nbytes() == v.numel() * v.element_size(), k
    assert get_state_dict(ckpt) is sd
    if kind == "finetune":
        assert {"control_model." + n for n in a.G.names} <= set(extract_lora(sd))
    assert len(ckpt["optimizer_states"]) == 1
    torch.optim.AdamW(a.G.params, lr=1e-3).load_state_dict(ckpt["optimizer_states"][0])

    b = make(kind, seed=5)
    if kind == "pretrain":
        b.cn.switch_lora("canny")
    assert not torch.equal(a.G.flat_p, b.G.flat_p)
    meta = b.load_checkpoint(path)
    assert meta == {"epoch": 4, "global_step": 3}
    for x, y in ((a.G.flat_p, b.G.flat_p), (a.G.exp_avg, b.G.exp_avg), (a.G.exp_avg_sq, b.G.exp_avg_sq)):
        assert torch.equal(x, y)
    assert (b.step_count, b.seg_steps, b.loss_scale, b.skipped_steps) == (3, a.seg_steps, 128.0, 2)
    assert {k: int(v) for k, v in b._step_dev.items() if int(v)} == a.seg_steps
    fa, fb = a.model.state_dict(), b.model.state_dict()
    # (pretrain: the lora_layer aliases show the set each model has attached: depth in a, canny in b)
    assert all(torch.equal(fa[k], fb[k]) for k in fa if not b._alias_key(k))


def test_reference_checkpoint_without_extra_key_keeps_the_defaults(tmp_path):
    a = make("finetune")
    opt = torch_adamw(a, "finetune")
    sd = dict(a.model.state_dict())
    sd["cond_stage_model.transformer.text_model.embeddings.position_ids"] = torch.zeros(1, 77)  # CLIP: not shipped
    path = str(tmp_path / "ref.ckpt")
    torch.save({"epoch": 0, "global_step": 3, "pytorch-lightning_version": "1.5.0", "state_dict": sd,
                "optimizer_states": [opt.state_dict()], "lr_schedulers": [], "callbacks": {}}, path)
    b = make("finetune", seed=5)
    b.load_checkpoint(path)
    assert b.loss_scale is None and b.skipped_steps == 0 and b.step_count == 3
    assert torch.equal(a.G.flat_p, b.G.flat_p)


def test_refusals(tmp_path):
    tr = make("finetune", accumulate_grad_batches=2)
    tr.begin_micro_batch()
    with pytest.raises(RuntimeError, match="flush"):
        tr.save_checkpoint(str(tmp_path / "x.ckpt"))
    with pytest.raises(RuntimeError, match="window"):
        tr.state_dict()
    assert not os.path.exists(tmp_path / "x.ckpt")

    tr = make("pretrain")
    ref = torch_adamw(tr, "pretrain").state_dict()
    before = [t.clone() for t in (tr.G.exp_avg, tr.G.exp_avg_sq)]
    first, conv = tr.G.names[0], next(i for i, p in enumerate(tr.G.params) if p.dim() == 4 and p.shape[-1] == 3)

    def bad(edit):
        import copy
        sd = copy.deepcopy(ref)
        edit(sd)
        return sd

    cases = [
        (lambda sd: sd["param_groups"][0].update(amsgrad=True), f"amsgrad.*{first}"),
        (lambda sd: sd["param_groups"][0].update(maximize=True), f"maximize.*{first}"),
        (lambda sd: sd["param_groups"].append(dict(sd["param_groups"][0], params=[])), "parameter groups"),
        (lambda sd: sd["param_groups"][0]["params"].pop(), f"816.*{tr.G.names[-1]}"),
        (lambda sd: sd["state"][conv].update(exp_avg=sd["state"][conv]["exp_avg"].permute(0, 2, 3, 1).contiguous()),
         tr.G.names[conv]),
        (lambda sd: sd["state"][conv].update(step=torch.tensor(7.0)), f"{tr.G.names[conv]}.*step 7"),
    ]
    for edit, msg in cases:
        with pytest.raises(ValueError, match=msg.replace("[", r"\[")):
            tr.load_state_dict(bad(edit))
        assert all(torch.equal(x, y) for x, y in zip(before, (tr.G.exp_avg, tr.G.exp_avg_sq))), msg
    assert tr.seg_steps == {} and tr.step_count == 0


def _ddp_worker(rank, world, port, path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        tr = make("finetune", seed=rank)  # replicas start from rank 0's parameters (construction-time broadcast)
        tr.load_state_dict(torch_adamw(tr, "finetune").state_dict())
        writes = []
        orig = torch.save

        def recording(obj, f, *a, **kw):
            writes.append(str(f))
            return orig(obj, f, *a, **kw)

        torch.save = recording
        try:
            tr.save_checkpoint(path)
        finally:
            torch.save = orig
        exists = os.path.exists(path)  # every rank leaves save_checkpoint after the file is complete
        other = make("finetune", seed=10 + rank)
        other.load_checkpoint(path)
        same = torch.equal(other.G.flat_p, tr.G.flat_p) and torch.equal(other.G.exp_avg, tr.G.exp_avg)
        q.put((rank, writes, exists, same))
    finally:
        dist.destroy_process_group()


def test_only_rank0_writes_world2(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() % 2000)
    path = str(tmp_path / "ddp.ckpt")
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, path, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r[0], r[1:]) for r in (q.get(timeout=300) for _ in procs))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res[0][0] == [path] and res[1][0] == []
    assert all(exists and same for _, exists, same in res.values())
