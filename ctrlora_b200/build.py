"""Builds ctrlora_b200/lib/libctrlora_b200.so (sm_90a only) with nvcc; no torch headers are involved.

The library is in-tree so that it travels to the GPU box with the repo snapshot.  `build()` is idempotent: it
recompiles only when a source is newer than the library.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
INCLUDE = os.path.join(os.path.dirname(ROOT), "include")
LIB_DIR = os.path.join(ROOT, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libctrlora_b200.so")
OBJ_DIR = os.path.join(ROOT, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-I", CSRC, "-I", INCLUDE,
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return hs


def build(force=False, verbose=False):
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    hdr_m = max(os.path.getmtime(h) for h in _headers())
    objs, procs = [], []
    for src in _sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) >= os.path.getmtime(src)
                and os.path.getmtime(obj) >= hdr_m):
            continue
        cmd = [nvcc] + NVCC_FLAGS + os.environ.get("CTRLORA_NVCC_EXTRA", "").split() + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    rebuilt = bool(procs)
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
        if verbose:
            sys.stderr.write(out)
    if rebuilt or not os.path.exists(LIB_PATH):
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-cudart", "static",
               "-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
