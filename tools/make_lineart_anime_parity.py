"""Record what the line-art kernels' existing calls return, for tests/test_lineart_anime_gpu.py to hold later builds
to bit for bit: the 64 / 128 / 256-channel ctrlora_instance_norm_f16 calls (plain and phase-interleaved) and
ctrlora_tap_gather_f16 calls of tests/lineart_anime_golden.py's PARITY_* cases.

    python tools/make_lineart_anime_parity.py LIB OUT

LIB is a libctrlora_b200.so built from a commit before the 512-channel instance norm (only those two entry points are
declared, so an older library loads); needs an H100.  Writes OUT (a .pt file, split into part files by golden_io).
"""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from ctrlora_b200 import _lib, ops  # noqa: E402
from golden_io import save_golden  # noqa: E402
import lineart_anime_golden as lg  # noqa: E402


def main():
    lib_path, out = sys.argv[1], sys.argv[2]
    lib = C.CDLL(lib_path)
    for name in ("ctrlora_tap_gather_f16", "ctrlora_instance_norm_f16", "ctrlora_last_cuda_error"):
        fn = getattr(lib, name)
        if name == "ctrlora_last_cuda_error":
            fn.restype = C.c_char_p
        else:
            fn.restype, fn.argtypes = C.c_int, _lib._ARGTYPES[name]
    _lib._lib = lib
    res = lg.parity_calls(ops, torch.device("cuda"))
    torch.cuda.synchronize()
    save_golden(res, out)
    print(f"wrote {out}: {sorted(res)}")


if __name__ == "__main__":
    main()
