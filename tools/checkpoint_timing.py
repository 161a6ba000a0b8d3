"""Time PretrainTrainer.save_checkpoint / load_checkpoint at SD1.5 size (configs/ctrlora_pretrain_sd15_9tasks_rank128.yaml)
and report the file size.  Every segment is marked as stepped, so the file holds both moments of every parameter, as a
checkpoint late in a run does.  Weights are synthetic (the timing does not depend on them).

    python tools/checkpoint_timing.py [--out results/checkpoint_timing.json] [--dir DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default=os.path.join(ROOT, "configs", "ctrlora_pretrain_sd15_9tasks_rank128.yaml"))
    ap.add_argument("--dir", default=None, help="directory of the checkpoint file (default: a temporary directory)")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ctrlora_b200.train import PretrainTrainer
    model = create_model(a.config, init_weights=False).cuda().eval()
    tr = PretrainTrainer(model)
    for key in set(tr.segment_keys()):
        tr._seg_state(key)[0].fill_(1000)
        tr.seg_steps[key] = 1000
    tr.step_count = 1000
    tr.G.flat_p.normal_()  # (init_weights=False leaves the memory as it was: possibly NaN, which never compares equal)
    tr.G.exp_avg.normal_()
    tr.G.exp_avg_sq.uniform_()
    torch.cuda.synchronize()
    res = {"config": os.path.basename(a.config), "params": tr.G.numel, "tensors": len(tr.G.names),
           "model_tensors": len(model.state_dict()), "save_s": [], "load_s": []}
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        path = os.path.join(d, "pretrain.ckpt")
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            tr.save_checkpoint(path)
            torch.cuda.synchronize()
            res["save_s"].append(time.perf_counter() - t0)
            res["file_bytes"] = os.path.getsize(path)
            ref = [t.clone() for t in (tr.G.flat_p, tr.G.exp_avg, tr.G.exp_avg_sq)]
            tr.G.exp_avg.zero_()
            t0 = time.perf_counter()
            tr.load_checkpoint(path)
            torch.cuda.synchronize()
            res["load_s"].append(time.perf_counter() - t0)
            res["exact"] = all(torch.equal(x, y) for x, y in zip(ref, (tr.G.flat_p, tr.G.exp_avg, tr.G.exp_avg_sq)))
            del ref
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["gpu"] = torch.cuda.get_device_name()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
