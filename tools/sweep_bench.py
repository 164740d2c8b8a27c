"""S4 sweep (BASELINE configs[4]): tensor-core (wgmma) InfoNCE forward / backward throughput at anchor x bank sizes.
Prints one JSON line per point: ms (CUDA events, median of iters after warm-up), algorithmic TFLOP/s
(fwd 2*A*N*D; bwd 2*A*N*D, recompute not counted) and the fraction of the measured bf16 peak.

    python tools/sweep_bench.py [AxN ...] [--neg-only]     # --neg-only: similarity + negative-sum sweep, no backward"""
import json
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
import torch
torch.set_num_threads(min(16, __import__("os").cpu_count() or 1))

from contrastiveseg_b200 import functional as Fn
from contrastiveseg_b200.synth import make_sweep_point

dev = torch.device("cuda:0")
peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) if os.path.exists(
    os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {"bf16_tflops": 1590.0}
points = [(1024, 190000), (4096, 32768), (16384, 65536), (65536, 131072)]
args = [x for x in sys.argv[1:] if "x" in x]
if args:
    points = [tuple(int(x) for x in p.split("x")) for p in args]
neg_only = "--neg-only" in sys.argv[1:]
iters = 5


def timed(fn):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


for A, N in points:
    g = torch.Generator(device="cpu").manual_seed(A + N)
    K = 19
    a = torch.nn.functional.normalize(torch.randn(A, 256, generator=g), dim=1).to(dev)
    c = torch.nn.functional.normalize(torch.randn(N, 256, generator=g), dim=1).to(dev)
    ya = torch.sort(torch.randint(0, K, (A,), generator=g)).values.to(dev)     # class-sorted anchors (like the engine)
    yc = torch.sort(torch.randint(0, K, (N,), generator=g)).values.to(dev)
    c16 = Fn.to_bf16_rows(c, -(-N // 256) * 256)
    diag = torch.arange(A, device=dev) % N
    state_box = {}

    def fwd():
        loss, st, state = Fn.infonce_tc_forward(a, ya, contrast_bf16=c16, contrast_cls=yc, n_cols=N, diag_col=diag,
                                                temperature=0.07, base_temperature=0.07, neg_only=neg_only)
        state_box["s"] = (loss, st, state)

    def bwd():
        loss, st, state = state_box["s"]
        Fn.infonce_tc_backward(state, st)

    t_f = timed(fwd)
    t_b = float("nan") if neg_only else timed(bwd)
    fl = 2.0 * A * N * 256
    out = {"A": A, "N": N, "fwd_ms": t_f, "bwd_ms": t_b, "fwd_tflops": fl / t_f / 1e9, "bwd_tflops": fl / t_b / 1e9,
           "fwd_frac_of_measured_peak": fl / t_f / 1e9 / peaks["bf16_tflops"],
           "bwd_frac_of_measured_peak": fl / t_b / 1e9 / peaks["bf16_tflops"], "loss": state_box["s"][0].item(), "neg_only": neg_only}
    print(json.dumps(out), flush=True)
