"""Timing of the contrast criterion, eager against replayed as one CUDA graph, and of the seg CE's two-call form
(pcl_seg_ce_fwd + pcl_seg_ce_bwd) against its one-pass form (pcl_seg_ce_fwd_bwd).

    python tools/criterion_bench.py [--rounds 3] [--iters 20] [--out criterion_bench.json]

Workloads:
  * criterion: S1 ContrastCELoss (B=8, 19x128x256 logits and D=256 embeddings -> 512x1024 labels), S1
    ContrastAuxCELoss (two logit heads), and the S2 bank step (MemContrastCELoss + enqueue, bank 19 x (5000+5000) x
    256); eager forward + backward() against GraphedContrastCriterion.replay()
  * seg CE alone: at S1 and at the ADE20K shape (B=2, 150x130x130 -> 520x520), the kernels called directly with
    pre-allocated buffers, so the arms differ only in the kernels they launch
Method: CUDA events around `iters` calls after a warm-up, the arms alternated, min-max over `rounds` rounds; the outputs
of the arms compared on the same seeded inputs; the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch  # noqa: E402

import contrastiveseg_b200 as cs  # noqa: E402
from contrastiveseg_b200 import _abi  # noqa: E402
from contrastiveseg_b200.synth import make_bank, make_contrast_batch  # noqa: E402

CE_SHAPES = {"S1 B=8 19x128x256 -> 512x1024": dict(B=8, h=128, w=256, num_classes=19, block=32),
             "ADE B=2 150x130x130 -> 520x520": dict(B=2, h=130, w=130, num_classes=150, block=10)}


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


def alternate(arms, rounds, iters):
    """{name: [min, max] ms} over `rounds` rounds, the arms alternated within each round."""
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timeit(fn, iters))
    return {k: [round(min(v), 4), round(max(v), 4)] for k, v in res.items()}


def bench_seg_ce(dev, args, B, h, w, num_classes, block):
    data = make_contrast_batch(B=B, D=8, h=h, w=w, num_classes=num_classes, img_stride=4, block=block, seed=304)
    seg, tgt = data["seg"].to(dev).contiguous(), data["target"].to(dev).contiguous()
    K, H, W = num_classes, tgt.shape[1], tgt.shape[2]
    lib = _abi.load()
    st = torch.cuda.current_stream(dev).cuda_stream
    grad = torch.ones(1, dtype=torch.float32, device=dev)
    sc2 = torch.empty(lib.pcl_seg_ce_scratch_floats(B, H, W), dtype=torch.float32, device=dev)
    sc1 = torch.empty(lib.pcl_seg_ce_fwd_bwd_scratch_floats(B, K, H, W), dtype=torch.float32, device=dev)
    loss2, loss1 = (torch.empty((), dtype=torch.float32, device=dev) for _ in range(2))
    d2, d1 = torch.empty_like(seg), torch.empty_like(seg)
    args_ = (seg.data_ptr(), tgt.data_ptr(), None, B, K, h, w, H, W, -1)

    def pair():
        _abi.check(lib.pcl_seg_ce_fwd(*args_, sc2.data_ptr(), loss2.data_ptr(), st), "pcl_seg_ce_fwd")
        _abi.check(lib.pcl_seg_ce_bwd(*args_, sc2.data_ptr(), grad.data_ptr(), d2.data_ptr(), st), "pcl_seg_ce_bwd")

    def one_pass():
        _abi.check(lib.pcl_seg_ce_fwd_bwd(*args_, sc1.data_ptr(), grad.data_ptr(), loss1.data_ptr(), d1.data_ptr(), st),
                   "pcl_seg_ce_fwd_bwd")

    out = alternate({"fwd+bwd (two calls)": pair, "fwd_bwd (one pass)": one_pass}, args.rounds, args.iters)
    pair()
    one_pass()
    torch.cuda.synchronize()
    out["loss_bit_equal"] = bool(torch.equal(loss1, loss2))
    out["dseg_max_err_over_max_g"] = float(((d1 - d2).abs().max() / d2.abs().max()).item())
    return out


def bench_criterion(dev, args, wrapper):
    """S1 ContrastCELoss / ContrastAuxCELoss, or the S2 bank step (MemContrastCELoss + enqueue) when wrapper is
    MemContrastCELoss: eager forward + backward() (+ the bank enqueue) against one replay."""
    mem = wrapper is cs.MemContrastCELoss
    cfg = cs.Configer(cs.cityscapes_contrast_config(with_memory=mem))
    cfg.add(["network", "loss_weights"], {"seg_loss": 1.0, "aux_loss": 0.4})
    crit = wrapper(cfg).to(dev)
    data = make_contrast_batch(B=8, D=256, h=128, w=256, num_classes=19, img_stride=4, block=32, seed=304)
    target = data["target"].to(dev)
    preds = {"seg": data["seg"].to(dev), "embed": data["embed"].to(dev)}
    if wrapper is cs.ContrastAuxCELoss:
        preds["seg_aux"] = (data["seg"] * 0.5).to(dev)
    enq = [None, None]
    banks = []
    if mem:
        for i in range(2):                   # the eager arm's bank and the graph's
            b = cs.MemoryBank(19, 5000, 256).to(dev)
            init = make_bank(19, 5000, 256)
            b.segment_queue.copy_(init["segment_queue"])
            b.pixel_queue.copy_(init["pixel_queue"])
            banks.append(b)
        enq[1] = dict(bank=banks[1], network_stride=4, pixel_update_freq=10)
    leaves = {k: v.clone().requires_grad_(True) for k, v in preds.items()}

    def eager():
        p = dict(leaves)
        if mem:
            p.update(segment_queue=banks[0].segment_queue, pixel_queue=banks[0].pixel_queue)
        for v in leaves.values():
            v.grad = None
        crit(p, target, with_embed=True).backward()
        if mem:
            banks[0].enqueue(leaves["embed"].detach(), target, network_stride=4, pixel_update_freq=10)

    gp = dict(preds)
    if mem:
        gp.update(segment_queue=banks[1].segment_queue, pixel_queue=banks[1].pixel_queue)
    gc = cs.GraphedContrastCriterion(crit, gp, target, enqueue=enq[1])
    out = alternate({"eager forward + backward": eager, "graph replay": gc.replay}, args.rounds, args.iters)
    # the seg half of the same inputs, eager against the replay (the contrast half draws its own anchors in each arm)
    e = {k: preds[k].clone().requires_grad_(True) for k in gc.heads}
    seg_loss = crit._seg_loss(e, target)
    seg_loss.backward()
    gc.replay()
    torch.cuda.synchronize()
    out["seg_grad_max_err_over_max_g"] = max(float(((gc.grads[k] - e[k].grad).abs().max() / e[k].grad.abs().max()).item())
                                             for k in gc.heads)
    return out


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("criterion_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"rounds": args.rounds, "iters": args.iters, "gpu": gpu_info()}
    for wrapper in (cs.ContrastCELoss, cs.ContrastAuxCELoss, cs.MemContrastCELoss):
        key = "S2 bank step MemContrastCELoss + enqueue" if wrapper is cs.MemContrastCELoss else f"S1 {wrapper.__name__}"
        out[key] = bench_criterion(dev, args, wrapper)
        print(key, out[key], flush=True)
    for name, kw in CE_SHAPES.items():
        out[f"seg CE {name}"] = bench_seg_ce(dev, args, **kw)
        print(name, out[f"seg CE {name}"], flush=True)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
