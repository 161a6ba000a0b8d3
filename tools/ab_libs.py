"""Run one command under several builds of libctrlora_b200.so, alternating, each run in a subprocess of its own.

    python tools/ab_libs.py --lib old=/path/old.so --lib new=/path/new.so --runs 3 --out DIR -- \
        python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline

For run r and library L the library file is copied over ctrlora_b200/lib/libctrlora_b200.so, the command runs, and its
stdout goes to DIR/<L>.<r>.txt ("{tag}" in the command is replaced by "<L>.<r>", e.g. for a --json path).  The card's
name, power limit and SM clock (sampled by nvidia-smi while nothing runs) head the log; the library that was in place
at the start is put back at the end.
"""
import argparse
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ctrlora_b200", "lib", "libctrlora_b200.so")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="name=path, in the order they alternate")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", required=True)
    ap.add_argument("cmd", nargs=argparse.REMAINDER)
    args = ap.parse_args()
    cmd = args.cmd[1:] if args.cmd[:1] == ["--"] else args.cmd
    libs = [tuple(s.split("=", 1)) for s in args.lib]
    os.makedirs(args.out, exist_ok=True)
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    print("card:", r.stdout.strip(), flush=True)
    keep = LIB + ".kept"
    shutil.copyfile(LIB, keep)
    try:
        for run in range(args.runs):
            for name, path in libs:
                shutil.copyfile(path, LIB)
                tag = f"{name}.{run}"
                out = subprocess.run([c.replace("{tag}", tag) for c in cmd], cwd=ROOT, stdout=subprocess.PIPE,
                                     stderr=subprocess.STDOUT, text=True)
                with open(os.path.join(args.out, tag + ".txt"), "w") as f:
                    f.write(out.stdout)
                last = out.stdout.strip().splitlines()[-1:] or [""]
                print(f"[{tag}] exit {out.returncode}: {last[0][:600]}", flush=True)
    finally:
        shutil.move(keep, LIB)


if __name__ == "__main__":
    sys.exit(main())
