"""Timing and peak memory of the fused RMI seg loss (csrc/pcl_segce.cu) vs the reference's torch op sequence on the GPU
(oracle/rmi_port.py with the reference's precisions: fp32 up-sampling / sigmoid / pooling, float64 moments) at the
Cityscapes shape: B=8, 19x128x256 logits -> 512x1024 labels, radius 3, max pool 3/3, lambda 0.5.

    python tools/rmi_bench.py [--rounds 3] [--iters 10] [--out rmi_bench.json]

Reports min-max over alternating rounds, CUDA events; torch.cuda.max_memory_allocated per path; the card's name and
power limit.  Also checks that both paths give the same loss."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import contrastiveseg_b200 as cs  # noqa: E402
from contrastiveseg_b200.synth import make_contrast_batch  # noqa: E402
from oracle.rmi_port import rmi_loss  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rmi_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    data = make_contrast_batch(B=8, D=8, h=128, w=256, num_classes=19, img_stride=4, block=32, seed=304)
    seg, tgt = data["seg"].to(dev), data["target"].to(dev)
    x = seg.clone().requires_grad_(True)
    K = seg.shape[1]
    paths = {
        "fused": lambda: cs.upsample_rmi_loss(x, tgt, num_classes=K),
        "torch": lambda: rmi_loss(x, tgt, num_classes=K, front=torch.float32),
    }

    def fwd(f):
        with torch.no_grad():
            f()

    def fwd_bwd(f):
        x.grad = None
        f().backward()

    def timeit(fn, f):
        for _ in range(2):
            fn(f)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn(f)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.iters

    res = {k: {"fwd_ms": [], "fwd_bwd_ms": []} for k in paths}
    for _ in range(args.rounds):
        for name, f in paths.items():                # alternating
            res[name]["fwd_ms"].append(timeit(fwd, f))
            res[name]["fwd_bwd_ms"].append(timeit(fwd_bwd, f))
    for name, f in paths.items():
        x.grad = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        f().backward()
        torch.cuda.synchronize()
        res[name]["peak_mb"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        res[name]["loss"] = f().item()
    out = {"shape": "B=8 19x128x256 -> 512x1024, r=3, max pool 3/3",
           "rounds": args.rounds, "iters": args.iters}
    for name in paths:
        out[name] = {k: ([round(min(v), 3), round(max(v), 3)] if isinstance(v, list) else v)
                     for k, v in res[name].items()}
    try:
        out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    capture_output=True, text=True).stdout.strip()
    except OSError:
        out["gpu"] = torch.cuda.get_device_name(0)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
