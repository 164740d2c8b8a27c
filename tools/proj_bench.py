"""Projection head's last 1x1 conv + L2 normalise: cuDNN Conv2d + cs.l2_normalize vs the fused wgmma GEMM
(cs.project_normalize), forward alone and forward + backward, at S1 (8, 720, 128, 256) and DeepLab C4 (2, 2048, 66, 66);
then one stand-in training iteration (the structure of bench.py's train_iter) with ProjectionHead(fused=False / True).

    python tools/proj_bench.py [--iters 20] [--rounds 3]

CUDA events around `iters` calls after a warm-up, three alternating A/B rounds (min and max printed).  The byte floor
of each variant is its algorithmic HBM traffic computed from tensor sizes (fp32 activations, bf16 gz workspace) over
the H100 SXM data-sheet bandwidth of 3.35 TB/s; it is a floor, not a measurement."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import contrastiveseg_b200 as cs  # noqa: E402

HBM = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                       # noqa: BLE001
        return f"unknown ({e})"


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def floors(B, Cin, HW):
    """bytes: (unfused fwd, unfused fwd+bwd, fused fwd, fused fwd+bwd)."""
    X, Z = 4 * B * Cin * HW, 4 * B * 256 * HW
    uf = X + Z + 2 * Z                                     # conv: x -> z; normalise: z -> zn
    ub = 3 * Z + (Z + X) + (Z + X)                         # l2 bwd: z, gzn -> gz; dgrad: gz -> gx; wgrad: gz, x
    ff = X + Z                                             # x -> zn (+ inv_norm, B*HW floats)
    fb = 2 * Z + X + Z // 2 + (Z // 2 + X)                 # dgrad: zn, gzn -> gx, gz (bf16); wgrad: gz, x
    return uf, uf + ub, ff, ff + fb


def head_pair(shape, iters, rounds):
    B, Cin, H, W = shape
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(shape, device=dev, generator=g).requires_grad_(True)
    conv = nn.Conv2d(Cin, 256, 1).to(dev)
    gzn = torch.randn((B, 256, H, W), device=dev, generator=g)

    def unfused():
        return cs.l2_normalize(conv(x))

    def fused():
        return cs.project_normalize(x, conv.weight, conv.bias)

    def fb(fn):
        def run():
            x.grad = None
            conv.weight.grad = conv.bias.grad = None
            fn().backward(gzn)
        return run

    with torch.no_grad():
        a, b = unfused(), fused()
        dz = (a - b).abs().max().item()
    fb(unfused)()
    ga = (x.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone())
    fb(fused)()
    gb = (x.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone())
    dg = [((p - q).abs().max() / p.abs().max()).item() for p, q in zip(ga, gb)]
    del a, b, ga, gb
    res = {"unfused fwd": [], "fused fwd": [], "unfused fwd+bwd": [], "fused fwd+bwd": []}
    for _ in range(rounds):
        with torch.no_grad():
            res["unfused fwd"].append(timeit(unfused, iters))
            res["fused fwd"].append(timeit(fused, iters))
        res["unfused fwd+bwd"].append(timeit(fb(unfused), iters))
        res["fused fwd+bwd"].append(timeit(fb(fused), iters))
    fl = dict(zip(("unfused fwd", "unfused fwd+bwd", "fused fwd", "fused fwd+bwd"), floors(B, Cin, H * W)))
    print(f"shape {shape}:  max |zn_unfused - zn_fused| = {dz:.3e};  max |g_unfused - g_fused| / max |g_unfused| "
          f"gx {dg[0]:.3e}  gW {dg[1]:.3e}  gb {dg[2]:.3e}")
    for k, v in res.items():
        print(f"  {k:16s} {min(v):8.3f} - {max(v):8.3f} ms   byte floor {fl[k] / 1e9:6.3f} GB = {fl[k] / HBM * 1e3:6.3f} ms")


def train_iter_pair(iters, rounds):
    """Stand-in iteration: conv body (720-channel stride-4 features) -> 19-class head + convmlp projection head ->
    ContrastCELoss (fused seg CE + pixel contrast) -> backward -> SGD step, as in bench.py's train_iter."""
    from contrastiveseg_b200.synth import make_contrast_batch
    dev = torch.device("cuda:0")
    B, K, D, C, Hi, Wi = 8, 19, 256, 720, 512, 1024
    data = make_contrast_batch(B=B, D=8, h=Hi // 4, w=Wi // 4, num_classes=K, img_stride=4, block=32, seed=304)
    target = data["target"].to(dev)

    class StandIn(nn.Module):
        def __init__(self, fused):
            super().__init__()
            self.body = nn.Sequential(nn.Conv2d(3, 64, 3, 2, 1), nn.BatchNorm2d(64), nn.ReLU(inplace=True),
                                      nn.Conv2d(64, C, 3, 2, 1), nn.BatchNorm2d(C), nn.ReLU(inplace=True))
            self.cls = nn.Conv2d(C, K, 1)
            self.proj = cs.ProjectionHead(C, D, proj="convmlp", bn_type="torchbn", fused=fused)

        def forward(self, x):
            f = self.body(x)
            return {"seg": self.cls(f), "embed": self.proj(f)}

    x = torch.randn(B, 3, Hi, Wi, device=dev)
    runs = {}
    for fused in (False, True):
        torch.manual_seed(304)
        net = StandIn(fused).to(dev)
        opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
        crit = cs.ContrastCELoss(cs.Configer(cs.cityscapes_contrast_config())).to(dev)

        def it(net=net, opt=opt, crit=crit):
            loss = crit(net(x), target, with_embed=True)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
        runs[fused] = it
    res = {False: [], True: []}
    for _ in range(rounds):
        for fused in (False, True):
            res[fused].append(timeit(runs[fused], iters))
    for fused in (False, True):
        print(f"  train iter, ProjectionHead(fused={fused!s:5s}) {min(res[fused]):8.3f} - {max(res[fused]):8.3f} ms")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("proj_bench: needs a CUDA device")
    print(f"card: {card()}   torch.backends.cudnn.allow_tf32 = {torch.backends.cudnn.allow_tf32}")
    for shape in ((8, 720, 128, 256), (2, 2048, 66, 66)):
        head_pair(shape, args.iters, args.rounds)
    train_iter_pair(max(3, args.iters // 4), args.rounds)


if __name__ == "__main__":
    main()
