"""Trainer checkpoints in the reference's PyTorch Lightning layout.

The reference trains through Lightning: `CheckpointEveryNSteps` calls `trainer.save_checkpoint` (cldm/logger.py:113-123),
whose file holds the model's `state_dict`, `optimizer_states` (torch.optim.AdamW.state_dict() over the parameter list
configure_optimizers builds), `global_step` and `epoch`.  FinetuneTrainer / PretrainTrainer keep their AdamW state in flat
device buffers instead (train.GradSink) plus device-side step counters; this module is the exact mapping between the two:

  * parameter i of the optimizer state is GradSink parameter i: the finetune filter in the reference's order
    (cldm_ctrlora_finetune.py:84-108) or `list(control_model.parameters())` (cldm_ctrlora_pretrain.py:174-182);
  * conv weights and their moments are STORED in the kernels' [Cout, kh, kw, Cin] order and exchanged in the reference
    shape [Cout, Cin, kh, kw];
  * torch keeps `step` per parameter and no state for a parameter that never had a gradient; the trainers count steps
    per segment (FinetuneTrainer: "all"; PretrainTrainer: "base" and one per LoRA set).  A segment that has not stepped
    exports no state, and an imported parameter without state is fresh (zero moments, its first step is step 1);
  * what torch has no slot for (the loss scale, skipped steps, accumulate_grad_batches) goes under EXTRA_KEY.

Everything here runs off the step path, on the host after a device-to-host copy (export) or as plain tensor copies into
the existing buffers (import), so captured graphs keep valid pointers.
"""
import numbers

import torch

EXTRA_KEY = "ctrlora_b200"
IGNORED_PREFIXES = ("cond_stage_model.",)  # CLIP, unless the model opted into ctrlora_b200.text_encoder (DESIGN.md §9)
# a buffer transformers 4 persisted in SD1.5 files and transformers 5 does not; the text encoder has no such key
CLIP_POSITION_IDS = "cond_stage_model.transformer.text_model.embeddings.position_ids"


def _host(flat, shape):
    """a flat fp32 slice (storage order) -> a contiguous CPU tensor of the reference shape that owns its storage"""
    if len(shape) == 4:
        co, ci, kh, kw = shape
        return flat.view(co, kh, kw, ci).to("cpu", copy=True).permute(0, 3, 1, 2).contiguous()
    return flat.to("cpu", copy=True).view(shape)


def _store(flat, src, shape):
    """copy a reference-shape tensor into a flat fp32 slice in storage order (host-side permutation for conv weights)"""
    src = src.detach()
    if len(shape) == 4:
        co, ci, kh, kw = shape
        flat.view(co, kh, kw, ci).copy_(src.permute(0, 2, 3, 1))
    else:
        flat.view(shape).copy_(src)


def _param_group(trainer):
    """torch.optim.AdamW's param_groups[0] for the trainer's hyper-parameters (every key the installed torch writes)"""
    probe = torch.optim.AdamW([torch.zeros(1, requires_grad=True)], lr=trainer.lr, betas=tuple(trainer.betas),
                              eps=trainer.eps, weight_decay=trainer.wd)
    group = probe.state_dict()["param_groups"][0]
    group["params"] = list(range(len(trainer.G.params)))
    return group


def optimizer_state_dict(trainer):
    """the trainer's AdamW state as torch.optim.AdamW.state_dict() over the reference's parameter list"""
    G = trainer.G
    state = {}
    for i, (name, p, key) in enumerate(zip(G.names, G.params, trainer.segment_keys())):
        step = trainer.seg_steps.get(key, 0)
        if step == 0:
            continue  # never stepped: torch holds no state for it
        off, n = G.offsets[name]
        state[i] = {"step": torch.tensor(float(step)), "exp_avg": _host(G.exp_avg[off:off + n], p.shape),
                    "exp_avg_sq": _host(G.exp_avg_sq[off:off + n], p.shape)}
    return {"state": state, "param_groups": [_param_group(trainer)]}


def trainer_extra(trainer):
    """trainer state torch's optimizer has no slot for"""
    return {"loss_scale": None if trainer.loss_scale is None else float(trainer.loss_scale),
            "skipped_steps": int(trainer.skipped_steps),
            "accumulate_grad_batches": int(trainer.accumulate_grad_batches)}


def _step_of(entry):
    s = entry["step"]
    s = float(s.item()) if isinstance(s, torch.Tensor) else float(s)
    if s != int(s) or s < 0:
        raise ValueError(f"non-integer AdamW step {s}")
    return int(s)


def check_optimizer_state_dict(trainer, sd):
    """Validate an AdamW state dict against the trainer's parameter list.  Returns ([(index, entry or None)], {segment:
    step}, param_group).  Raises ValueError naming the first offending parameter by its reference name."""
    G = trainer.G
    names = G.names
    if not isinstance(sd, dict) or "state" not in sd or "param_groups" not in sd:
        raise ValueError("not an optimizer state dict: expected the keys 'state' and 'param_groups'")
    groups = sd["param_groups"]
    if len(groups) != 1:
        raise ValueError(f"{len(groups)} parameter groups; the trainers' AdamW has one (first parameter {names[0]!r})")
    group = groups[0]
    for flag in ("amsgrad", "maximize"):
        if group.get(flag, False):
            raise ValueError(f"{flag}=True is not supported by the trainers' AdamW (first parameter {names[0]!r})")
    ids = list(group["params"])
    if len(ids) != len(names):
        first = names[min(len(ids), len(names) - 1)]
        raise ValueError(f"the optimizer state covers {len(ids)} parameters, this trainer trains {len(names)} "
                         f"(first unmatched parameter {first!r})")
    state = sd["state"]
    known = set(ids)
    stray = [k for k in state if k not in known]
    if stray:
        raise ValueError(f"state for parameter id {stray[0]!r}, which is not in the parameter group")
    entries, steps, first_of = [], {}, {}
    for i, (name, p, key, pid) in enumerate(zip(names, G.params, trainer.segment_keys(), ids)):
        entry = state.get(pid)
        step = 0
        if entry is not None:
            if "max_exp_avg_sq" in entry:
                raise ValueError(f"amsgrad state (max_exp_avg_sq) for parameter {name!r} is not supported")
            for k in ("exp_avg", "exp_avg_sq"):
                if k not in entry:
                    raise ValueError(f"parameter {name!r}: no {k} in its state")
                if tuple(entry[k].shape) != tuple(p.shape):
                    raise ValueError(f"parameter {name!r}: {k} has shape {tuple(entry[k].shape)}, the parameter "
                                     f"{tuple(p.shape)}")
            step = _step_of(entry)
        if key not in steps:
            steps[key], first_of[key] = step, name
        elif steps[key] != step:
            raise ValueError(f"parameter {name!r} is at AdamW step {step} but {first_of[key]!r} of the same "
                             f"segment {key!r} is at step {steps[key]}: the trainer keeps one step count per segment")
        entries.append((i, entry))
    return entries, steps, group


def load_optimizer_state_dict(trainer, sd):
    """Copy an AdamW state dict into the trainer's flat moments and step counters, in place (validated first: nothing
    changes when it raises).  The file's hyper-parameters replace the trainer's (torch's and Lightning's resume)."""
    entries, steps, group = check_optimizer_state_dict(trainer, sd)
    G = trainer.G
    with torch.no_grad():
        for i, entry in entries:
            off, n = G.offsets[G.names[i]]
            shape = G.params[i].shape
            for buf, k in ((G.exp_avg, "exp_avg"), (G.exp_avg_sq, "exp_avg_sq")):
                if entry is None:
                    buf[off:off + n].zero_()
                else:
                    _store(buf[off:off + n], entry[k], shape)
    trainer.lr = float(group["lr"])
    trainer.betas = tuple(float(b) for b in group["betas"])
    trainer.eps = float(group["eps"])
    trainer.wd = float(group["weight_decay"])
    b1, b2 = trainer.betas
    seg_steps = {}
    for key, step in steps.items():
        if step:
            seg_steps[key] = step
        if step or key in trainer._step_dev:
            step_dev, bc = trainer._seg_state(key)
            step_dev.fill_(step)
            bc.copy_(torch.tensor([1.0 - b1 ** step, 1.0 - b2 ** step] if step else [1.0, 1.0]))
    trainer.seg_steps = seg_steps
    trainer.step_count = seg_steps.get(trainer.segment_keys()[0], 0)


def parse_extra(trainer, extra):
    """(loss_scale, skipped_steps) from the EXTRA_KEY part; a file without it (a reference checkpoint: precision 32, no
    scaler) keeps the trainer's values"""
    if extra is None:
        return trainer.loss_scale, trainer.skipped_steps
    scale = extra.get("loss_scale")
    if scale is not None and (isinstance(scale, bool) or not isinstance(scale, numbers.Real) or not scale > 0):
        raise ValueError(f"loss_scale must be a positive number or None, got {scale!r}")
    return (None if scale is None else float(scale)), int(extra.get("skipped_steps", 0))


def model_state_dict(model):
    """model.state_dict() with every tensor a contiguous CPU copy of its own (a parameter adopted by a trainer is a
    permuted view of a flat buffer: pickling the view would write the whole buffer behind it)"""
    return {k: v.detach().to("cpu", copy=True).contiguous() for k, v in model.state_dict().items()}


def checkpoint_weights(sd, expected, alias=lambda k: False):
    """The file's weights restricted to what the model holds: keys of modules the drop-in does not ship
    (IGNORED_PREFIXES, unless the model holds such keys itself: a model built with the text encoder loads its CLIP
    weights like any other) and aliases (`alias(key)`) are dropped; any other difference from `expected` (the model's
    state_dict()) in keys or shapes raises before anything is loaded."""
    if any(k.startswith(IGNORED_PREFIXES) for k in expected):
        def dropped(k):
            return k == CLIP_POSITION_IDS or alias(k)
    else:
        def dropped(k):
            return k.startswith(IGNORED_PREFIXES) or alias(k)
    keep = {k: v for k, v in sd.items() if not dropped(k)}
    want = {k for k in expected if not dropped(k)}
    missing = [k for k in expected if k in want and k not in keep]
    unexpected = [k for k in keep if k not in want]
    if missing or unexpected:
        raise ValueError(f"checkpoint weights do not match the model: missing {missing[:5]}, unexpected {unexpected[:5]}")
    for k, v in keep.items():
        if tuple(v.shape) != tuple(expected[k].shape):
            raise ValueError(f"checkpoint weight {k!r} has shape {tuple(v.shape)}, the model {tuple(expected[k].shape)}")
    return keep
