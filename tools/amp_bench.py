"""Half-precision inputs against fp32 inputs on the seeded S1 / S2 inputs of bench.py (one GPU).

Alternates fp32 and bf16 inputs for --rounds rounds and reports min-max per case over the rounds (CUDA events after
warm-up):
  s1_fused_fill     S1 captured step, fused path, dense gradient zero-filled every replay
  s1_sparse_reset   S1 captured step, fused path, sparse reset of the persistent gradient
  s2_bank_enqueue   S2 captured bank step with the enqueue (keys = embed)
  eager_contrast_ce eager ContrastCELoss forward + backward (fused seg CE), embed and seg in the input dtype
  workaround        bf16 embed/seg -> .float() -> eager ContrastCELoss -> autograd's cast back (bf16 rows only)
Checks the bit-identity contract at these sizes (loss bit-equal, gradient == fp32 gradient rounded, bank bit-equal)
and reports the in-graph kernel timeline of the S1 fused step per dtype.  Prints the card name and power limit
(nvidia-smi query).  Writes nothing unless --out is given.

    python tools/amp_bench.py [--rounds 3] [--steps 50] [--warmup 10] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import contrastiveseg_b200 as cs  # noqa: E402
from contrastiveseg_b200 import functional as Fn  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:                                   # noqa: BLE001
        return f"unknown ({exc})"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def opts(cfg, **kw):
    return cs.ContrastOptions(temperature=cfg["T"], base_temperature=cfg["bT"], max_samples=cfg["max_samples"],
                              max_views=cfg["max_views"], num_classes=cfg["K"], seed=5, precision="bf16", **kw)


def s1_step(inp, dtype, sparse_reset):
    return cs.GraphedContrastStep(inp["embed"].to(dtype), inp["target"], seg=inp["seg"].to(dtype), options=opts(bench.S1),
                                  sparse_reset=sparse_reset)


def s2_step(inp, dtype):
    cfg = bench.S2
    bank = cs.MemoryBank(cfg["K"], cfg["M"], cfg["D"], with_shadow=True).cuda()
    bank.segment_queue.copy_(inp["segment_queue"]); bank.pixel_queue.copy_(inp["pixel_queue"])
    bank.sync_shadow()
    step = cs.GraphedContrastStep(inp["embed"].to(dtype), inp["target"], seg=inp["seg"].to(dtype),
                                  segment_queue=bank.segment_queue, pixel_queue=bank.pixel_queue, bank_shadow=bank.shadow,
                                  options=opts(cfg),
                                  enqueue=dict(bank=bank, network_stride=cfg["net_stride"], pixel_update_freq=cfg["F"], seed=3))
    return step, bank


def eager_fn(inp, dtype, workaround=False):
    crit = cs.ContrastCELoss(bench.engine_configer(bench.S1, False, "bf16")).cuda()
    # leaves of their own: `.to(torch.float32)` of an fp32 tensor returns the shared input itself, and marking that as
    # requiring grad would make every later copy of it a non-leaf that accumulates into a gradient of the shared input
    embed = inp["embed"].detach().to(dtype).requires_grad_(True)
    seg = inp["seg"].detach().to(dtype).requires_grad_(True)

    def run():
        embed.grad = None; seg.grad = None
        e, s = (embed.float(), seg.float()) if workaround else (embed, seg)
        crit({"seg": s, "embed": e}, inp["target"], with_embed=True).backward()
    return run


def check_identity(inp1, inp2):
    """The contract at the timed sizes, bf16 against the same call on the fp32 copies."""
    out = {}
    dt = torch.bfloat16
    h = {k: (v.to(dt) if k in ("embed", "seg") else v) for k, v in inp1.items()}
    f = {k: (v.float() if k in ("embed", "seg") else v) for k, v in h.items()}
    for name, sr in (("s1_fused_fill", False), ("s1_sparse_reset", True)):
        a, b = s1_step(h, dt, sr), s1_step(f, torch.float32, sr)
        ok = True
        for _ in range(3):
            la, ga = a.replay(); lb, gb = b.replay()
            torch.cuda.synchronize()
            ok &= torch.equal(la, lb) and torch.equal(ga, gb.to(dt)) and torch.equal(a.ws.anchor_meta, b.ws.anchor_meta)
        out[name] = bool(ok)
    h2 = {k: (v.to(dt) if k in ("embed", "seg") else v) for k, v in inp2.items()}
    f2 = {k: (v.float() if k in ("embed", "seg") else v) for k, v in h2.items()}
    (a, ba), (b, bb) = s2_step(h2, dt), s2_step(f2, torch.float32)
    ok = True
    for _ in range(3):
        la, ga = a.replay(); lb, gb = b.replay()
        torch.cuda.synchronize()
        ok &= torch.equal(la, lb) and torch.equal(ga, gb.to(dt))
        for n in ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr", "shadow"):
            ok &= torch.equal(getattr(ba, n), getattr(bb, n))
    out["s2_bank_enqueue"] = bool(ok)
    res = []
    for e, s in ((h["embed"], h["seg"]), (f["embed"], f["seg"])):
        g = torch.Generator().manual_seed(7)
        o = opts(bench.S1, perm_fn=lambda n, g=g: torch.randperm(n, generator=g))
        e = e.detach().clone().requires_grad_(True)
        loss = cs.pixel_contrast_loss(e, h["target"], seg=s, options=o)
        loss.backward()
        res.append((loss.detach(), e.grad))
    out["eager_loss"] = bool(torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1].to(dt)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    inp1 = bench.make_inputs(bench.S1, 304, dev)
    inp2 = bench.make_inputs(bench.S2, 304, dev, bank=True)
    result = {"card": card(), "torch": torch.__version__, "rounds": args.rounds, "steps": args.steps,
              "warmup": args.warmup, "identity": check_identity(inp1, inp2)}
    cases = {}
    dtypes = {"fp32": torch.float32, "bf16": torch.bfloat16}
    timelines = {}
    for r in range(args.rounds):
        for dn, dt in dtypes.items():
            runs = {}
            st = s1_step(inp1, dt, False)
            runs["s1_fused_fill"] = timed(st.replay, args.steps, args.warmup)
            if r == 0:
                timelines[dn] = bench.Workload.graph_timeline(types.SimpleNamespace(steps=[st], dev=dev))
            del st
            st = s1_step(inp1, dt, True)
            runs["s1_sparse_reset"] = timed(st.replay, args.steps, args.warmup)
            del st
            st, bank = s2_step(inp2, dt)
            runs["s2_bank_enqueue"] = timed(st.replay, args.steps, args.warmup)
            del st, bank
            runs["eager_contrast_ce"] = timed(eager_fn(inp1, dt), max(10, args.steps // 5), 3)
            if dt != torch.float32:
                runs["workaround"] = timed(eager_fn(inp1, dt, workaround=True), max(10, args.steps // 5), 3)
            Fn.clear_workspaces()
            torch.cuda.empty_cache()
            for k, v in runs.items():
                cases.setdefault(k, {}).setdefault(dn, []).append(round(v, 4))
    result["ms"] = {k: {dn: {"min": min(v), "max": max(v), "rounds": v} for dn, v in d.items()} for k, d in cases.items()}
    result["s1_fused_timeline_us"] = timelines
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
