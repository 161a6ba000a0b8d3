"""Per-class device time of the sampling step's GEMMs, next to the tile model's prediction.

One DDIM step of the bench workload (batched CFG at batch 4, i.e. one batch-8 pass) runs un-graphed while every
ctrlora_gemm_f16 argument block is recorded.  The launches are grouped by class (level, Cin, N, ksize, epilogue kind);
each class's launches, with their multiplicity, are captured into one CUDA graph and replayed back to back between
two CUDA events, as ops.replay_gemms does for the whole step.

    python tools/gemm_classes.py [--reps 20] [--json out.json] [--sm-scaling]

--sm-scaling also times two representative launches (64x64 3x3 conv 320->320, 16x16 3x3 conv 1280->1280) with the
persistent grid limited to 132 / 66 / 33 SMs.  A kernel bound inside each SM (MMA issue, latency) takes ~2x as long on
half the SMs; one bound by a shared resource (L2 -> SM bandwidth) takes less than 2x.
"""
import argparse
import ctypes as C
import json
import math
import os
import sys
from collections import OrderedDict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

# tile model of gemm_sm90.cu (ctrlora_gemm_f16), in SM cycles; keep in step with the constants there
MODEL = dict(l2_bpc=40.0, epi_fixed=600.0, epi_per_col=12.0, split_per_col=12.0)


def model_cycles(a, sms, widths, m=MODEL):
    """Cycles the model predicts for the plan it picks for one launch with argument block `a`."""
    bw = 1 << int(math.log2(min(a.a_w, 128)))
    bh = 1 << int(math.log2(min(a.a_h, 128 // bw)))
    nb = 128 // (bw * bh)
    m_tiles = -(-a.a_w // bw) * -(-a.a_h // bh) * -(-a.a_b // nb)
    k_iters = a.kh * a.kw * -(-a.a_c // 64) + (-(-a.a2_c // 64) if a.a2 else 0)
    # ping-pong plans: whole tiles that all take the TMA epilogue, K loop under GEMM_PP_MAX_KITERS (40)
    pp_launch = (not a.out_f32 and not any(a.transposed) and not (a.residual and a.residual_f32) and k_iters < 40
                 and a.split_k <= 1)
    best = None
    for cand in ([w // 2 for w in widths if w >= 64 and w != 160] if a.geglu else widths):  # no 80 + 80 GEGLU tile
        if a.seg_width and a.seg_width % cand:
            continue
        if (2 * cand if a.geglu else cand) > 256 and k_iters < 40:  # GEMM_WIDE_MIN_KITERS
            continue
        if not a.geglu and cand == 160 and k_iters >= 40:  # 160 only where 320 is excluded
            continue
        bnt = 2 * cand if a.geglu else cand
        tiles = m_tiles * -(-a.n // cand)
        step = max(4.0 * bnt, (16384 + bnt * 128) / m["l2_bpc"])
        if pp_launch and (cand == 64 if a.geglu else 64 <= cand <= 160):
            epi = m["epi_fixed"] + 2 * m["epi_per_col"] * cand  # one warpgroup runs the tile's epilogue
            cost = -(-tiles // sms) * max(k_iters * step, epi) + epi
            if best is None or cost < best:
                best = cost
        for S in range(1, 9):
            kps = -(-k_iters // S)
            s_eff = -(-k_iters // kps)
            w = tiles if s_eff == 1 else (tiles // sms) * sms
            tail = tiles - w
            if s_eff > 1 and tail == 0:
                continue
            epi = m["epi_fixed"] + m["epi_per_col"] * cand
            t_whole = k_iters * step + epi
            t_split = kps * step + epi + m["split_per_col"] * bnt * (1 + s_eff)
            cost = -(-w // sms) * t_whole + -(-(tail * s_eff) // sms) * t_split
            if best is None or cost < best:
                best = cost
    return best


def klass(a):
    kind = "geglu" if a.geglu else "qkv" if a.seg_width else f"skip{a.a2_c}" if a.a2 else "res" if a.residual else ""
    level = f"{a.a_h}x{a.a_w}" if a.a_h > 1 else f"lin M={a.a_w}"
    return (level, a.a_c, a.n * (2 if a.geglu else 1), a.kh, kind)


def time_graph(lib, recs, reps):
    def launch_all():
        sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for args in recs:
            rc = lib.ctrlora_gemm_f16(C.addressof(args), sp)
            assert rc == 0, rc

    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        launch_all()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            launch_all()
        for _ in range(3):
            graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            graph.replay()
        e1.record()
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--sm-scaling", action="store_true")
    ap.add_argument("--widths", default="320,256,160,128,64,32", help="tile widths the model chooses among")
    ap.add_argument("--clock-mhz", type=float, default=1980.0, help="SM clock the model's cycles are converted at")
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    from ctrlora_b200 import _lib, dropin, ops
    dropin.activate()
    from cldm.ddim_hacked import DDIMSampler
    model = bench.build_model(device)
    sampler = DDIMSampler(model, batched_cfg=True, use_cuda_graph=False)
    sampler.make_schedule(50, ddim_eta=0.0, verbose=False)
    B = bench.BATCH
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 4, 64, 64, generator=g).to(device)
    hint = torch.randn(B, 4, 64, 64, generator=g).to(device)
    ctx = torch.randn(B, 77, 768, generator=g).to(device)
    uc = torch.randn(B, 77, 768, generator=g).to(device)
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    ts = torch.full((B,), 981, device=device, dtype=torch.long)

    def step():
        with sampler.run_mode():
            sampler.p_sample_ddim(x, cond, ts, index=49, unconditional_guidance_scale=7.5, unconditional_conditioning=ucond)

    step()
    torch.cuda.synchronize()
    ops._GEMM_RECORD = []
    step()
    torch.cuda.synchronize()
    recs, ops._GEMM_RECORD = ops._GEMM_RECORD, None
    lib = _lib.load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    widths = [int(w) for w in args.widths.split(",")]
    classes = OrderedDict()
    for args_, flops, _keep in recs:
        classes.setdefault(klass(args_), []).append((args_, flops))
    name = torch.cuda.get_device_name(0)
    print(f"{name}, {sms} SMs, {len(recs)} GEMM launches in {len(classes)} classes")
    print(f"{'level':>12} {'Cin':>6} {'N':>5} {'k':>2} {'epi':>8} {'n':>3} {'GFLOP':>8} {'ms':>7} {'TFLOP/s':>8} {'model ms':>8}")
    rows, tot_ms, tot_fl, tot_model = [], 0.0, 0.0, 0.0
    for key, items in sorted(classes.items(), key=lambda kv: -sum(f for _, f in kv[1])):
        ms = time_graph(lib, [a for a, _ in items], args.reps)
        fl = sum(f for _, f in items)
        mod = sum(model_cycles(a, sms, widths) for a, _ in items) / (args.clock_mhz * 1e3)
        tot_ms, tot_fl, tot_model = tot_ms + ms, tot_fl + fl, tot_model + mod
        rows.append(dict(level=key[0], cin=key[1], n=key[2], ksize=key[3], epi=key[4], count=len(items), gflop=fl / 1e9,
                         ms=ms, tflops=fl / ms / 1e9, model_ms=mod))
        print(f"{key[0]:>12} {key[1]:>6} {key[2]:>5} {key[3]:>2} {key[4]:>8} {len(items):>3} {fl / 1e9:8.1f} {ms:7.3f} "
              f"{fl / ms / 1e9:8.1f} {mod:8.3f}")
    whole = time_graph(lib, [a for a, _, _ in recs], args.reps)
    print(f"sum of classes {tot_ms:.2f} ms ({tot_fl / tot_ms / 1e9:.0f} TFLOP/s), model {tot_model:.2f} ms; "
          f"whole step replayed {whole:.2f} ms ({tot_fl / whole / 1e9:.0f} TFLOP/s)")
    out = {"device": name, "classes": rows, "sum_ms": tot_ms, "step_ms": whole, "tflop": tot_fl / 1e12}
    if args.sm_scaling:
        out["sm_scaling"] = sm_scaling(ops, lib, args.reps)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


def sm_scaling(ops, lib, reps):
    res = []
    for (b, h, w, c, n) in ((8, 64, 64, 320, 320), (8, 16, 16, 1280, 1280)):
        a = (torch.randn(b, h, w, c, device="cuda") * 0.5).half()
        wt = (torch.randn(n, 9, c, device="cuda") * (9 * c) ** -0.5).half()
        fl = 2.0 * b * h * w * n * 9 * c
        for limit in (0, 66, 33):
            ops.set_sm_limit(limit)
            try:
                ops.gemm(a, wt, ksize=3)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    ops.gemm(a, wt, ksize=3)
                e1.record()
                torch.cuda.synchronize()
            finally:
                ops.set_sm_limit(0)
            us = e0.elapsed_time(e1) / reps * 1e3
            sms = limit or torch.cuda.get_device_properties(0).multi_processor_count
            print(f"  3x3 {h}x{w} {c}->{n} on {sms:3d} SMs: {us:8.1f} us, {fl / us / 1e6:6.1f} TFLOP/s, "
                  f"{fl / us / 1e6 / sms:5.2f} TFLOP/s per SM")
            res.append(dict(shape=[b, h, w, c, n], sms=sms, us=us, tflops=fl / us / 1e6))
    return res


if __name__ == "__main__":
    main()
