"""Times every distinct attention-forward launch of the batch-8 sampling step (ctrlora_attention_f16):

    python tools/attn_bench.py [--root TREE] [--rows-per-cta N] [--reps 50] [--out FILE]

--root is the source tree whose built library is imported, so the same script times another checkout's kernel.
--rows-per-cta is the query rows that share one fetch of K / V^T in that tree's kernel (default: this tree's, 192 at
d <= 48 and 128 above); it only enters the byte count.

Per shape, after warm-up, CUDA events around `reps` back-to-back launches give the time per launch.  Reported with it:
  exp/s and its fraction of the MUFU bound: 16 ex2 per clock per SM at the SM clock sampled while the kernel runs
  tensor TFLOP/s: 4 * Nq * Nk * d per (image, head), the QK^T and PV products at the head dimension (no padding)
  kv_gb, kv_tb_s: K and V^T bytes one launch streams from L2 into shared memory (every CTA work unit of rows-per-cta
    queries reads all Nk keys of its head: 4 * d bytes per key), and that over the launch time
Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (Nq, Nk, d, launches per step) at batch 8 (4 images x CFG), 512 x 512: self-attention and cross-attention to the 77
# context tokens at the 64 / 32 / 16 / 8 levels of the UNet and the ControlNet
SHAPES = [(4096, 4096, 40, 7), (1024, 1024, 80, 7), (256, 256, 160, 7), (64, 64, 160, 2),
          (4096, 77, 40, 7), (1024, 77, 80, 7), (256, 77, 160, 7), (64, 77, 160, 2)]
BATCH, HEADS = 8, 8
MUFU_PER_CLK_SM = 16


def gpu_query(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return [x.strip() for x in out.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--rows-per-cta", type=int, default=0)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from ctrlora_b200 import ops
    assert torch.cuda.is_available(), "attn_bench needs a CUDA device"
    dev = torch.device("cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    name, power_limit = gpu_query("name,power.limit")
    g = torch.Generator(device=dev).manual_seed(7)
    rows, step_us = [], 0.0
    for nq, nk, d, count in SHAPES:
        mk = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.5).half()
        q, k, v = mk(BATCH * nq, HEADS * d), mk(BATCH * nk, HEADS * d), mk(BATCH * nk, HEADS * d)
        nk_pad = (nk + 7) // 8 * 8
        vt = torch.zeros(BATCH, HEADS, d, nk_pad, device=dev, dtype=torch.float16)
        vt[..., :nk] = v.view(BATCH, nk, HEADS, d).permute(0, 2, 3, 1)
        out = torch.empty_like(q)
        run = lambda: ops.attention(q, k, vt, BATCH, HEADS, nq, nk, d, out=out)
        for _ in range(5):
            run()
        torch.cuda.synchronize()
        # sample the SM clock while about half a second of launches is queued
        t0 = time.perf_counter()
        run()
        torch.cuda.synchronize()
        n_busy = max(20, int(0.5 / max(time.perf_counter() - t0, 1e-6)))
        for _ in range(n_busy):
            run()
        clk_mhz = float(gpu_query("clocks.sm")[0])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / args.reps
        exps = float(BATCH) * HEADS * nq * nk
        rows_per_cta = args.rows_per_cta or (192 if d <= 48 else 128)
        units = math.ceil(nq / rows_per_cta) * HEADS * BATCH
        kv_bytes = float(units) * nk * 4 * d
        mufu_bound = MUFU_PER_CLK_SM * sms * clk_mhz * 1e6
        rows.append({"nq": nq, "nk": nk, "d": d, "per_step": count, "rows_per_cta": rows_per_cta, "us": round(us, 1),
                     "exp_per_s": exps / (us * 1e-6), "mufu_frac": round(exps / (us * 1e-6) / mufu_bound, 3),
                     "tflops": round(4.0 * exps * d / (us * 1e-6) / 1e12, 1), "kv_gb": round(kv_bytes / 1e9, 3),
                     "kv_tb_s": round(kv_bytes / (us * 1e-6) / 1e12, 2), "sm_clock_mhz": clk_mhz})
        step_us += count * us
        del q, k, v, vt, out
    for r in rows:
        print(f"Nq {r['nq']:5d} Nk {r['nk']:5d} d {r['d']:3d} x{r['per_step']}: {r['us']:8.1f} us  "
              f"MUFU {r['mufu_frac']:.2f} @ {r['sm_clock_mhz']:.0f} MHz  {r['tflops']:6.1f} TFLOP/s  "
              f"K/V {r['kv_gb']:.3f} GB = {r['kv_tb_s']:.2f} TB/s", file=sys.stderr)
    res = {"gpu": name, "power_limit_w": power_limit, "root": os.path.abspath(args.root),
           "attention_us_per_step": round(step_us, 1), "shapes": rows}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
