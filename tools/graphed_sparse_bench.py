"""The sparse projection head (ProjectionHead(fused=True, fuse_bn_relu=True[, fuse_conv1=True], sparse_grad=True)) behind
the captured contrast step, forward + backward at S1 (x (8, 720, 128, 256), max_samples 1024, the fused small-anchor
step: precision bf16, device RNG), in fp32 and under torch.autocast(bfloat16).  Three arms:

    dense   GraphedContrastStep(grad="dense") + the head without sparse_grad (zn written into the step's embed)
    cols    GraphedContrastStep(grad="cols") + the sparse_grad head (the columns handed over by apply())
    eager   pixel_contrast_loss + the sparse_grad head (no graph)

and the captured step alone (one replay, no head) in both modes.

    python tools/graphed_sparse_bench.py [--iters 20] [--step-iters 1000] [--rounds 3] [--out FILE]

CUDA events around `iters` iterations after a warm-up (`step-iters` replays for the step alone, about 0.1 s of GPU
time per window); `rounds` rounds that alternate the arms (min and max of the per-iteration time printed).  The card's
name, power limit and clocks are read in the same run."""
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
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                       # noqa: BLE001
        return f"unknown ({e})"


def setup(conv1, bf16, B=8, C=720, h=128, w=256, K=19):
    torch.manual_seed(0)
    heads = {}
    for sparse in (False, True):
        torch.manual_seed(0)
        heads[sparse] = cs.ProjectionHead(C, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                                          fuse_conv1=conv1, sparse_grad=sparse).cuda().train()
    data = make_contrast_batch(B=B, D=8, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=5)
    target, seg = data["target"].cuda(), data["seg"].cuda()
    x = torch.randn(B, C, h, w, device="cuda").requires_grad_(True)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=1024, max_views=100,
                              precision="bf16", rng="device", seed=3)
    zdt = torch.bfloat16 if bf16 else torch.float32
    steps = {g: cs.GraphedContrastStep(torch.zeros(B, 256, h, w, dtype=zdt, device="cuda"), target, seg=seg,
                                       options=opts, grad=g) for g in ("dense", "cols")}
    assert all(s.fused for s in steps.values())

    def captured(g, head):
        def run():
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                zn = head(x, out=steps[g].embed)
                loss = steps[g].apply(zn)
            loss.backward()
        return run

    def eager():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
            zn = heads[True](x)
            loss = Fn.pixel_contrast_loss(zn, target, seg=seg, options=opts)
        loss.backward()

    arms = {"dense": captured("dense", heads[False]), "cols": captured("cols", heads[True]), "eager": eager}
    alone = {f"step {g}": s.replay for g, s in steps.items()}
    return arms, alone, steps


def time_fn(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def rounds(fns, iters, n):
    for fn in fns.values():                          # warm-up: modules, workspaces, allocator
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in fns}
    for _ in range(n):
        for name, fn in fns.items():
            times[name].append(time_fn(fn, iters))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--step-iters", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graphed_sparse_bench needs a CUDA device")
    lines = [f"card (name, power limit, SM clock, max SM clock, memory clock): {card()}",
             "S1 head + captured contrast step, forward + backward, ms per iteration (min-max over rounds)"]
    print("\n".join(lines), flush=True)
    for conv1 in (False, True):
        for bf16 in (False, True):
            arms, alone, steps = setup(conv1, bf16)
            t = rounds(arms, a.iters, a.rounds)
            ta = rounds(alone, a.step_iters, a.rounds)
            label = f"{'fuse_conv1' if conv1 else 'fuse_bn_relu'} {'bf16 autocast' if bf16 else 'fp32'}"
            row = "  ".join(f"{n} {min(v):.3f}-{max(v):.3f}" for n, v in list(t.items()) + list(ta.items()))
            line = (f"{label:26s} {row}  cols vs dense {min(t['dense']) / min(t['cols']):.2f}x  "
                    f"step alone {min(ta['step dense']) / min(ta['step cols']):.2f}x")
            print(line, flush=True)
            lines.append(line)
            del arms, alone, steps
            Fn.clear_workspaces()
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
