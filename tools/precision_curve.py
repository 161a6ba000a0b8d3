"""Error-vs-cost curve for closing the fp16 parity gap with a selective two-term (hi + lo) operand split.

Input: precision_attribution.json (tools/precision_attribution.py: err_g = end-to-end error when ONLY block g
rounds to fp16; the squares add up to the measured end-to-end error^2 within 13 %).  A block whose GEMM operands are split
(A_hi W_hi + A_lo W_hi + A_hi W_lo, three GEMM passes instead of one) stops contributing its operand-rounding error;
its cost is 2 extra passes over its GEMM flops at the measured GEMM-family rate of the bench line.  Blocks are taken in
order of error^2 removed per extra flop.  (Attention-internal roundings inside a block are not removed by the split, so
the curve is optimistic by the attention share of each block.)
"""
import json, sys
src = sys.argv[1] if len(sys.argv) > 1 else "precision_attribution.json"
rate_tflops = float(sys.argv[2]) if len(sys.argv) > 2 else 829.0    # measured GEMM-family TFLOP/s of the DDIM step
passes_per_step = 8                                                  # batch 4 x (cond, uncond)
step_ms = 15.36
d = json.load(open(src))
groups = d["groups"]; flops = d["flops"]
tot_var = sum(v * v for v in groups.values())
scale = (d["all"] ** 2) / tot_var          # calibrate the additive model to the measured all-roundings figure
items = sorted(groups, key=lambda g: -(groups[g] ** 2) / max(flops[g], 1e6))
rows, removed, extra = [], 0.0, 0.0
print(f"{'protected blocks':>4s} {'last block added':40s} {'err':>9s} {'extra GF/img':>12s} {'extra ms/step':>13s} {'step x':>7s}")
for i, gname in enumerate(items, 1):
    removed += groups[gname] ** 2
    extra += 2.0 * flops[gname]
    err = (max(tot_var - removed, 0.0) * scale) ** 0.5
    ms = extra * passes_per_step / (rate_tflops * 1e12) * 1e3
    rows.append({"n_blocks": i, "block": gname, "err": err, "extra_gflop_per_image": extra / 1e9, "extra_ms_per_step": ms,
                 "step_factor": (step_ms + ms) / step_ms})
    if i <= 12 or err < 1.05e-3 and rows[-2]["err"] >= 0.9e-3 or i % 6 == 0:
        print(f"{i:4d} {gname:40s} {err:9.2e} {extra / 1e9:12.1f} {ms:13.2f} {(step_ms + ms) / step_ms:7.2f}")
first = next(r for r in rows if r["err"] <= 1.0e-3)
print("first point at or below 1e-3:", first)
json.dump({"source": src, "gemm_rate_tflops": rate_tflops, "baseline_err": d["all"], "curve": rows, "first_below_1e-3": first},
          open("precision_curve.json", "w"), indent=1)
