"""BASELINE.json configs[4]: LoRA rank sweep 32..512, finetune step at batch 8 on one GPU (the B@A-fusion cost curve).

    python tools/rank_sweep.py > rank_sweep.json
The forward folds B@A into the fp16 weights (cost independent of the rank); the backward uses factored weight
gradients (2 skinny TN GEMMs per LoRA layer), so the rank only shows up there and in the re-fold + AdamW.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
out = []
for r in (32, 64, 128, 256, 512):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "train", "--lora-rank", str(r),
                        "--train-batch", "8", "--steps", "10", "--warmup", "3", "--no-cpu-baseline"],
                       capture_output=True, text=True)
    line = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if not line:
        out.append({"lora_rank": r, "error": p.stderr[-400:]})
        continue
    d = json.loads(line[-1])
    out.append({"lora_rank": r, "batch": 8, "images_per_sec": d["value"], "ms_per_step": d["ms_per_step"],
                "trainable_params": d.get("trainable_params")})
print(json.dumps(out, indent=1))
