"""ProjectionHead(fused=True, fuse_bn_relu=True[, fuse_conv1=True]) + ContrastCELoss's contrast term, forward +
backward at S1 (x (8, 720, 128, 256), max_samples 1024), with sparse_grad=False (the loss writes the dense embedding
gradient, the head runs its dense backward) against sparse_grad=True (the loss hands the head its anchor columns), in
fp32 and under torch.autocast(bfloat16).

    python tools/sparse_head_bench.py [--iters 20] [--rounds 3]

CUDA events around `iters` iterations after a warm-up; three rounds that alternate the sparse and dense arms (min and
max of the per-iteration time printed), and the peak memory of one loss + backward.  The card's name and power limit
are read in the same run."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import contrastiveseg_b200 as cs  # noqa: E402
from contrastiveseg_b200 import functional as Fn  # noqa: E402
from contrastiveseg_b200.synth import make_contrast_batch  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                       # noqa: BLE001
        return f"unknown ({e})"


def setup(conv1, sparse, B=8, C=720, h=128, w=256, K=19):
    torch.manual_seed(0)
    head = cs.ProjectionHead(C, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True, fuse_conv1=conv1,
                             sparse_grad=sparse).cuda().train()
    cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": 4},
                       "loss": {"params": {"ce_ignore_index": -1}},
                       "contrast": {"temperature": 0.1, "base_temperature": 0.07, "max_samples": 1024,
                                    "max_views": 100, "loss_weight": 0.1}})
    crit = cs.PixelContrastLoss(cfg)
    data = make_contrast_batch(B=B, D=8, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=5)
    x = torch.randn(B, C, h, w, device="cuda").requires_grad_(True)
    return head, crit, x, data["target"].cuda(), data["seg"].cuda()


def step(head, crit, x, target, seg, bf16):
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
        zn = head(x)
        loss = crit(zn, target, seg=seg)
    loss.backward()


def time_arm(arm, bf16, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        step(*arm, bf16)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def peak(arm, bf16):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step(*arm, bf16)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print(f"card: {card()}")
    print("S1 head + contrast loss, forward + backward, ms per iteration (min-max over rounds); peak MiB over one step")
    for conv1 in (False, True):
        for bf16 in (False, True):
            arms = {name: setup(conv1, name == "sparse") for name in ("dense", "sparse")}
            for arm in arms.values():                    # warm-up: modules, workspaces, allocator
                for _ in range(3):
                    step(*arm, bf16)
            times = {name: [] for name in arms}
            for _ in range(a.rounds):
                for name, arm in arms.items():
                    times[name].append(time_arm(arm, bf16, a.iters))
            mem = {name: peak(arm, bf16) for name, arm in arms.items()}
            label = f"{'fuse_conv1' if conv1 else 'fuse_bn_relu'} {'bf16 autocast' if bf16 else 'fp32'}"
            row = "  ".join(f"{n} {min(t):.3f}-{max(t):.3f} ms ({mem[n]:.0f} MiB)" for n, t in times.items())
            print(f"{label:28s} {row}  speed-up {min(times['dense']) / min(times['sparse']):.2f}x", flush=True)
            del arms
            Fn.clear_workspaces()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
