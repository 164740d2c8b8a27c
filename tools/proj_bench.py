"""Projection head's last 1x1 conv + L2 normalise: cuDNN Conv2d + cs.l2_normalize vs the fused wgmma GEMM
(cs.project_normalize), forward alone and forward + backward, at S1 (8, 720, 128, 256) and DeepLab C4 (2, 2048, 66, 66),
with fp32 activations and with bf16 activations (the fused GEMM on bf16 x against the autocast baseline: cuDNN bf16
conv + cs.l2_normalize); then one stand-in training iteration (the structure of bench.py's train_iter) with
ProjectionHead(fused=False / True), in fp32 and under torch.autocast(bfloat16).

    python tools/proj_bench.py [--iters 20] [--rounds 3]

CUDA events around `iters` calls after a warm-up, three rounds that alternate the variants (min and max printed).  The
byte floor of each variant is its algorithmic HBM traffic computed from tensor sizes (fp32 or bf16 activations, bf16 gz
workspace) over the H100 SXM data-sheet bandwidth of 3.35 TB/s; it is a floor, not a measurement."""
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
    """bytes: (unfused fwd, unfused fwd+bwd, fused fwd, fused fwd+bwd) with fp32 activations."""
    X, Z = 4 * B * Cin * HW, 4 * B * 256 * HW
    uf = X + Z + 2 * Z                                     # conv: x -> z; normalise: z -> zn
    ub = 3 * Z + (Z + X) + (Z + X)                         # l2 bwd: z, gzn -> gz; dgrad: gz -> gx; wgrad: gz, x
    ff = X + Z                                             # x -> zn (+ inv_norm, B*HW floats)
    fb = 2 * Z + X + Z // 2 + (Z // 2 + X)                 # dgrad: zn, gzn -> gx, gz (bf16); wgrad: gz, x
    return uf, uf + ub, ff, ff + fb


def floors_bf16(B, Cin, HW):
    """bytes: (autocast fwd, autocast fwd+bwd, fused fwd, fused fwd+bwd) with bf16 activations.  The autocast baseline:
    cuDNN bf16 conv, then cs.l2_normalize, which copies its bf16 input to fp32 and returns fp32 (autograd casts the fp32
    gradient back to bf16 for the conv).  The fused path: fp32 floors with x, zn, gzn and gx halved; the gz workspace
    is bf16 in both."""
    X, Z = 2 * B * Cin * HW, 2 * B * 256 * HW              # bf16 sizes
    uf = X + Z + (Z + 2 * Z) + 2 * 2 * Z                   # conv: x -> z; z -> fp32 copy; normalise: z -> zn (fp32)
    ub = 3 * 2 * Z + (2 * Z + Z) + (Z + X) + (Z + X)       # l2 bwd (fp32); cast gz to bf16; dgrad; wgrad
    ff = X + Z
    fb = 2 * Z + X + Z + (Z + X)                           # dgrad: zn, gzn -> gx, gz (bf16); wgrad: gz, x
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

    x16 = x.detach().to(torch.bfloat16).requires_grad_(True)
    gzn16 = gzn.to(torch.bfloat16)

    def autocast_bf16():                                     # what an autocast user gets without the fused head
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return cs.l2_normalize(conv(x16))

    def fused_bf16():
        return cs.project_normalize(x16, conv.weight, conv.bias)

    def fb(fn, xin, g):
        def run():
            xin.grad = None
            conv.weight.grad = conv.bias.grad = None
            y = fn()
            y.backward(g.to(y.dtype))
        return run

    def grads(xin):
        return (xin.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone())

    def rel(ga, gb):
        return [((p.float() - q.float()).abs().max() / p.float().abs().max()).item() for p, q in zip(ga, gb)]

    with torch.no_grad():
        a, b = unfused(), fused()
        dz = (a - b).abs().max().item()
        a16, b16 = autocast_bf16(), fused_bf16()
        dz16 = (a16.float() - b16.float()).abs().max().item()
    fb(unfused, x, gzn)()
    ga = grads(x)
    fb(fused, x, gzn)()
    dg = rel(ga, grads(x))
    fb(autocast_bf16, x16, gzn16)()
    ga16 = grads(x16)
    fb(fused_bf16, x16, gzn16)()
    dg16 = rel(ga16, grads(x16))
    del a, b, a16, b16, ga, ga16
    variants = {"fp32": {"unfused": (unfused, x, gzn), "fused": (fused, x, gzn)},
                "bf16": {"autocast": (autocast_bf16, x16, gzn16), "fused": (fused_bf16, x16, gzn16)}}
    res = {(act, name, ph): [] for act, v in variants.items() for name in v for ph in ("fwd", "fwd+bwd")}
    for _ in range(rounds):
        for act, v in variants.items():                      # fp32 and bf16 arms alternate within each round
            for name, (fn, xin, g) in v.items():
                with torch.no_grad():
                    res[(act, name, "fwd")].append(timeit(fn, iters))
                res[(act, name, "fwd+bwd")].append(timeit(fb(fn, xin, g), iters))
    HW = H * W
    fl = {}
    for act, f in (("fp32", floors(B, Cin, HW)), ("bf16", floors_bf16(B, Cin, HW))):
        base = "unfused" if act == "fp32" else "autocast"
        fl.update({(act, base, "fwd"): f[0], (act, base, "fwd+bwd"): f[1], (act, "fused", "fwd"): f[2],
                   (act, "fused", "fwd+bwd"): f[3]})
    print(f"shape {shape}:  max |zn_unfused - zn_fused| = {dz:.3e};  max |g_unfused - g_fused| / max |g_unfused| "
          f"gx {dg[0]:.3e}  gW {dg[1]:.3e}  gb {dg[2]:.3e}")
    print(f"  bf16 x:  max |zn_autocast - zn_fused| = {dz16:.3e};  max |g_autocast - g_fused| / max |g_autocast| "
          f"gx {dg16[0]:.3e}  gW {dg16[1]:.3e}  gb {dg16[2]:.3e}")
    for k, v in res.items():
        name = f"{k[0]} {k[1]} {k[2]}"
        print(f"  {name:26s} {min(v):8.3f} - {max(v):8.3f} ms   byte floor {fl[k] / 1e9:6.3f} GB = "
              f"{fl[k] / HBM * 1e3:6.3f} ms")


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
    for amp in (False, True):
        for fused in (False, True):
            torch.manual_seed(304)
            net = StandIn(fused).to(dev)
            opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
            crit = cs.ContrastCELoss(cs.Configer(cs.cityscapes_contrast_config())).to(dev)

            def it(net=net, opt=opt, crit=crit, amp=amp):
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                    loss = crit(net(x), target, with_embed=True)
                opt.zero_grad(set_to_none=True)
                loss.backward()
                opt.step()
            runs[(amp, fused)] = it
    res = {k: [] for k in runs}
    for _ in range(rounds):
        for k in runs:
            res[k].append(timeit(runs[k], iters))
    for (amp, fused), v in res.items():
        mode = "autocast(bf16)" if amp else "fp32          "
        print(f"  train iter {mode}, ProjectionHead(fused={fused!s:5s}) {min(v):8.3f} - {max(v):8.3f} ms")


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
