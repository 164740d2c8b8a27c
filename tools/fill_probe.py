"""Zero-fill rate of the S1 dense gradient (268 MB fp32, 134 MB half) against the fill's CTA count, on the GPU.

Builds tools/fill_probe.cu with nvcc into a temporary directory, runs it, and writes the curve together with the card's
name, power limit and maximum SM clock (read in the same run) to <out>/fill_probe.json.

    python tools/fill_probe.py [--out DIR (default fill_probe_out)] [--reps N (launches timed per point)]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="fill_probe_out")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "fill_probe")
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        os.path.join(HERE, "fill_probe.cu"), "-o", exe], check=True)
        out = subprocess.run([exe, str(a.reps)], capture_output=True, text=True, check=True).stdout
    rows = [json.loads(l) for l in out.splitlines() if l.startswith("{")]
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "fill_probe.json"), "w") as f:
        json.dump({"card": card, "rows": rows}, f, indent=1)
    print(card)
    for r in rows:
        print(json.dumps(r))
    return 0


if __name__ == "__main__":
    sys.exit(main())
