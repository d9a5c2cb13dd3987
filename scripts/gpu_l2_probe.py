"""L2 ceilings for the f-k column passes' intermediate V: compile and run scripts/l2_probe.cu.

    python scripts/gpu_l2_probe.py [--out DIR]

Compiles the probe for sm_90a into a temporary directory (nothing is written to the tree), runs it, and prints the card
(name, power limit, maximum SM clock) together with the SM clock sampled while the probe runs.  With --out, the probe's
output and the card lines also go to DIR/l2_probe.txt."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={query}", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as exc:       # noqa: BLE001
        return f"nvidia-smi unavailable: {exc!r}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "l2_probe")
        subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(HERE, "l2_probe.cu")], check=True)
        card = smi("name,power.limit,clocks.max.sm")
        clocks, done = [], threading.Event()

        def sample():
            while not done.wait(0.25):
                s = smi("clocks.sm").split()
                if s and s[0].isdigit():
                    clocks.append(int(s[0]))

        th = threading.Thread(target=sample)
        th.start()
        try:
            r = subprocess.run([exe], capture_output=True, text=True)
        finally:
            done.set()
            th.join()
    lines = [f"card: {card}",
             f"SM clock while probing (MHz): min {min(clocks, default=0)}, max {max(clocks, default=0)}, "
             f"samples {len(clocks)}",
             r.stdout.rstrip()]
    text = "\n".join(lines)
    print(text)
    if r.returncode:
        print(r.stderr, file=sys.stderr)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "l2_probe.txt"), "w") as f:
            f.write(text + "\n")
    return r.returncode


if __name__ == "__main__":
    sys.exit(main())
