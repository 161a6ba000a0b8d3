"""Sweep (block_n, split_k) of ctrlora_gemm_f16 on the step's tile-starved shapes; prints a table per shape."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ctrlora_b200 import ops  # noqa: E402


def rnd(*s, scale=1.0):
    return (torch.randn(*s, device="cuda") * scale).half()


def timeit(fn, n=10):
    """Mean seconds per call over n calls after 3 warm-up calls (CUDA events)."""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e-3


import os as _os
SHAPES_SMALL = [(8, 8, 8, 1280, 1280, 3), (8, 8, 8, 2560, 1280, 3), (8, 8, 8, 1280, 1280, 1), (8, 16, 16, 1280, 1280, 3), (8, 16, 16, 1280, 1280, 1)]
SHAPES = [  # B, H, W, C, N, ksize
    (8, 8, 8, 1280, 1280, 3), (8, 16, 16, 1280, 1280, 3), (8, 16, 16, 1280, 1280, 1), (8, 32, 32, 640, 640, 1),
    (8, 64, 64, 320, 320, 1), (8, 8, 8, 1280, 1280, 1), (8, 16, 16, 2560, 1280, 3), (8, 32, 32, 640, 640, 3),
    (8, 64, 64, 320, 320, 3), (8, 32, 32, 1920, 640, 3), (8, 64, 64, 960, 320, 3), (8, 64, 64, 640, 320, 3),
]
if __name__ == "__main__":
    for (b, h, w, c, n, ks) in (SHAPES_SMALL if _os.environ.get('SWEEP_SMALL') else SHAPES):
        a, wt = rnd(b, h, w, c), rnd(n, ks * ks, c, scale=(ks * ks * c) ** -0.5)
        bias, res = torch.randn(n, device="cuda"), rnd(b * h * w, n)
        out = torch.empty(b, h, w, n, device="cuda", dtype=torch.float16)
        fl = 2.0 * b * h * w * n * c * ks * ks
        print(f"--- {ks}x{ks} {h}x{w} {c}->{n} (M={b * h * w}), {fl / 1e9:.0f} GF")
        auto = timeit(lambda: ops.gemm(a, wt, ksize=ks, bias=bias, residual=res, out=out))
        print(f"  auto: {auto * 1e3:7.1f} us {fl / auto / 1e9:6.0f} TF/s")
        for bn in (320, 256, 128, 64, 32):  # the wgmma tile widths of ctrlora_gemm_f16
            row = []
            for s in (1, 2, 4, 6, 8, 12):
                try:
                    ms = timeit(lambda: ops.gemm(a, wt, ksize=ks, bias=bias, residual=res, out=out, block_n=bn, split_k=s), n=5)
                    row.append(f"S{s}:{ms * 1e3:6.1f}")
                except Exception:
                    row.append(f"S{s}:   n/a")
            print(f"  bn={bn:3d} " + " ".join(row))
