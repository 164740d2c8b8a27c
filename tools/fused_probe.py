"""Timing probe at the S1 shape: ms per graph replay of the fused, the sparse-reset and the unfused step."""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import contrastiveseg_b200 as cs
import bench

dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
cfg = dict(bench.S1)
B = int(os.environ.get("PROBE_B", cfg["B"]))
cfg["B"] = B
inp = {k: v.to(dev) for k, v in bench.make_inputs(cfg, 304, None, False).items()}
crit = cs.PixelContrastLoss(bench.engine_configer(cfg, False, "bf16"))
opts = crit.options(); opts.num_classes = cfg["K"]
steps = int(os.environ.get("PROBE_STEPS", "200"))
for fused in (True, "sparse", False):
    st = cs.GraphedContrastStep(inp["embed"], inp["target"], seg=inp["seg"], options=opts, fused=bool(fused),
                                sparse_reset=(fused == "sparse"))
    for _ in range(10):
        st.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        st.replay()
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({"B": B, "fused": fused, "ms_per_step": e0.elapsed_time(e1) / steps, "loss": float(st.loss.item())}),
          flush=True)
    del st
