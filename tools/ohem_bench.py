"""Timing and peak memory of the fused OHEM cross-entropy (csrc/pcl_segce.cu, fourth part) vs the reference's torch op
sequence on the GPU (oracle/ohem_port.py with the reference's precision: fp32 up-sampled logits, a full softmax, a
gather, a boolean-mask copy, a sort of every labelled pixel, a CE with reduction='none', two fancy-index copies) at two
shapes, Cityscapes S1 (B=8, 19x128x256 logits -> 512x1024 labels) and an ADE20K-sized one (B=2, 150x130x130 ->
520x520), each at two confidences of make_contrast_batch, boost 2 and boost 8, with thresh 0.9 and min_kept 100000 as
the contrast configs set them.  Both take the threshold branch (fp32(thresh) decides): the bilinear blend across the
synthetic label blocks leaves more than min_kept pixels below 0.9 even at boost 8.  A third workload, boost 8 with
min_kept 1000000 (above the count below 0.9), makes the exact select run.

    python tools/ohem_bench.py [--rounds 3] [--iters 5] [--out ohem_bench.json]

Reports min-max over alternating rounds, CUDA events; peak memory above the inputs (torch.cuda.max_memory_allocated)
per path; the branch the fused path took, read from its scratch; the card's name and power limit, read in the same
call.  Also reports both paths' losses."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import contrastiveseg_b200 as cs  # noqa: E402
from contrastiveseg_b200.functional import ohem_selection  # noqa: E402
from contrastiveseg_b200.synth import make_contrast_batch  # noqa: E402
from oracle.ohem_port import ohem_loss  # noqa: E402

SHAPES = {"S1 B=8 19x128x256 -> 512x1024": dict(B=8, h=128, w=256, num_classes=19, block=32),
          "ADE B=2 150x130x130 -> 520x520": dict(B=2, h=130, w=130, num_classes=150, block=10)}
WORKLOADS = ((2.0, 100000), (8.0, 100000), (8.0, 1000000))     # (boost, min_kept)
THRESH = 0.9


def bench_shape(dev, args, B, h, w, num_classes, block, boost, min_kept):
    data = make_contrast_batch(B=B, D=8, h=h, w=w, num_classes=num_classes, img_stride=4, block=block, boost=boost,
                               seed=304)
    seg, tgt = data["seg"].to(dev), data["target"].to(dev)
    x = seg.clone().requires_grad_(True)
    paths = {
        "fused": lambda: cs.upsample_ohem_cross_entropy(x, tgt, thresh=THRESH, min_kept=min_kept),
        "torch": lambda: ohem_loss(x, tgt, thresh=THRESH, min_kept=min_kept, front=torch.float32),
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
        res[name]["peak_mb"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        res[name]["loss"] = f().item()
    out = {name: {k: ([round(min(v), 3), round(max(v), 3)] if isinstance(v, list) else v) for k, v in r.items()}
           for name, r in res.items()}
    sel = ohem_selection(x.detach(), tgt, thresh=THRESH, min_kept=min_kept)
    out["fused"].update(branch=sel["branch"], n=sel["n"], selected=sel["count"], threshold=sel["threshold"])
    n = cs._abi.load().pcl_ohem_ce_scratch_bytes(B, num_classes, h, w, tgt.shape[1], tgt.shape[2])
    out["fused"]["scratch_mb"] = round(n / 2 ** 20, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ohem_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"rounds": args.rounds, "iters": args.iters, "thresh": THRESH}
    for name, kw in SHAPES.items():
        for boost, min_kept in WORKLOADS:
            out[f"{name} boost {boost:g} min_kept {min_kept}"] = bench_shape(dev, args, boost=boost, min_kept=min_kept,
                                                                             **kw)
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
