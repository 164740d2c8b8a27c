"""a10 (per-anchor top-k hard negatives, csrc/pcl_topk.cuh) at the bank shape of BASELINE configs[2] for ncu: three
histogram sweeps + scans + weighted NEG sweep + POS + finalize (forward) and the top-k backward, exact fp32 path."""
import hashlib
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from contrastiveseg_b200 import functional as Fn
from contrastiveseg_b200.synth import make_bank

dev = torch.device("cuda:0")
A, K, M, D, k = int(os.environ.get("PROBE_A", "1024")), 19, int(os.environ.get("PROBE_M", "5000")), 256, int(os.environ.get("PROBE_K", "1024"))
g = torch.Generator().manual_seed(3)
a = torch.nn.functional.normalize(torch.randn(A, D, generator=g), dim=1).to(dev)
ya = torch.randint(0, K, (A,), generator=g)
ya = ya[torch.argsort(torch.where(ya == 0, torch.full_like(ya, K), ya), stable=True)].to(dev)   # engine row order: class rank 1..K-1, 0
bank = make_bank(K, M, D, 5)
sq, pq = bank["segment_queue"].to(dev), bank["pixel_queue"].to(dev)
diag = torch.arange(A, device=dev)
path = os.environ.get("PROBE_PATH", "simt")
if path == "tc":
    from contrastiveseg_b200 import _abi
    import ctypes as C
    from contrastiveseg_b200.bank import shadow_rows
    shadow = torch.empty((shadow_rows(K, M), D), dtype=torch.bfloat16, device=dev)
    _abi.check(_abi.load().pcl_bank_shadow_rebuild(sq.data_ptr(), pq.data_ptr(), K, M, D, shadow.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
for it in range(3):
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    if path == "tc":
        loss, st, state = Fn.infonce_tc_forward(a, ya, bank=(shadow, K, 2 * M), diag_col=diag, temperature=0.07,
                                                base_temperature=0.07, topk=k)
    else:
        loss, st, state = Fn.infonce_forward(a, ya, queues=(sq, pq), diag_col=diag, temperature=0.07, base_temperature=0.07, topk=k)
    e1.record()
    dA = Fn.infonce_tc_backward(state, st) if path == "tc" else Fn.infonce_backward(state, st)
    e2.record()
    torch.cuda.synchronize()
print(json.dumps({"path": path, "A": A, "N": (K - 1) * 2 * M, "k": k, "fwd_ms": e0.elapsed_time(e1), "bwd_ms": e1.elapsed_time(e2),
                  "loss": float(loss.item()), "dA_sha256": hashlib.sha256(dA.cpu().numpy().tobytes()).hexdigest()}))
