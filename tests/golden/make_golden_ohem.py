"""Generate the OHEM CE golden vectors (tests/golden/ohem_*.npz) by running the UNMODIFIED reference on CPU.

    python tests/golden/make_golden_ohem.py

FSOhemCELoss (lib/loss/loss_helper.py:215-261) on logits at label resolution (its own call) in the threshold branch, the
min_kept branch, with ohem_minkeep >= n, with ce_weight, with 'sum' and with ignore_index 255; one bilinear case
(F.interpolate, then the module); and FSAuxOhemCELoss (lib/loss/loss_helper.py:264-281) on a bilinear pair.  The labels
of pixels whose p_t lies within a few fp32 ulps of the threshold are set to ignore (oracle/ohem_port.gap_labels), so
fp32 and float64 select the same pixels and the goldens pin the gradient as well as the loss.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle.ohem_port import gap_labels  # noqa: E402
from oracle.ref_loader import DictConfiger, load_reference  # noqa: E402

# name, B, K, h, w, H, W, params (loss.params), ignore_index, logit scale
CASES = [
    ("ohem_thresh_branch", 2, 5, 16, 18, 16, 18, {"ohem_thresh": 0.7, "ohem_minkeep": 50}, -1, 3.0),
    ("ohem_minkept_branch", 2, 5, 16, 18, 16, 18, {"ohem_thresh": 0.05, "ohem_minkeep": 300}, -1, 3.0),
    ("ohem_minkeep_ge_n", 1, 4, 12, 13, 12, 13, {"ohem_thresh": 0.5, "ohem_minkeep": 100000}, -1, 3.0),
    ("ohem_weight", 2, 6, 14, 15, 14, 15,
     {"ohem_thresh": 0.6, "ohem_minkeep": 200, "ce_weight": [0.5, 1.0, 1.5, 2.0, 0.75, 1.25]}, -1, 3.0),
    ("ohem_sum", 2, 5, 13, 17, 13, 17, {"ohem_thresh": 0.3, "ohem_minkeep": 250, "ce_reduction": "sum"}, -1, 3.0),
    ("ohem_ignore255", 2, 5, 15, 16, 15, 16, {"ohem_thresh": 0.7, "ohem_minkeep": 100, "ce_ignore_index": 255}, 255,
     3.0),
    ("ohem_bilinear", 2, 7, 9, 11, 33, 41, {"ohem_thresh": 0.4, "ohem_minkeep": 1500}, -1, 4.0),
]


def _params(p, ignore_index):
    d = {"ce_ignore_index": ignore_index, "ce_reduction": "elementwise_mean"}
    d.update(p)
    return d


def _inputs(B, K, h, w, H, W, seed, ignore_index, scale, params):
    g = torch.Generator().manual_seed(seed)
    seg = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * scale
    target = torch.randint(0, K, (B, H, W), generator=g)
    target[torch.rand(B, H, W, generator=g) < 0.15] = ignore_index
    wt = torch.tensor(params["ce_weight"], dtype=torch.float32) if "ce_weight" in params else None
    red = params.get("ce_reduction", "mean")
    target = gap_labels(seg, target, ignore_index=ignore_index, weight=wt, thresh=params["ohem_thresh"],
                        min_kept=params["ohem_minkeep"], reduction=red)
    return seg, target


def loss_case(name, B, K, h, w, H, W, p, ignore_index, scale, seed):
    load_reference()
    import lib.loss.loss_helper as lh
    params = _params(p, ignore_index)
    seg, target = _inputs(B, K, h, w, H, W, seed, ignore_index, scale, params)
    cfg = DictConfiger({"loss": {"params": params}})
    x = seg.clone().requires_grad_(True)
    up = x if (h, w) == (H, W) else F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)
    loss = lh.FSOhemCELoss(cfg)(up, target.clone())
    loss.backward()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), seg=seg.numpy(), target=target.numpy(),
                        thresh=np.float64(params["ohem_thresh"]), min_kept=np.int64(params["ohem_minkeep"]),
                        weight=np.array(params.get("ce_weight", []), np.float32),
                        reduction=np.array(params["ce_reduction"]), ignore_index=np.int64(ignore_index),
                        loss=np.float32(loss.item()), grad_seg=x.grad.numpy())
    print(f"{name}: loss={loss.item():.7f}")


def aux_case(name, seed):
    load_reference()
    import lib.loss.loss_helper as lh
    B, K, h, w, H, W = 2, 6, 10, 12, 37, 45
    params = _params({"ohem_thresh": 0.5, "ohem_minkeep": 800}, -1)
    seg, target = _inputs(B, K, h, w, H, W, seed, -1, 4.0, params)
    g = torch.Generator().manual_seed(seed + 1)
    aux = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * 2.0
    cfg = DictConfiger({"loss": {"loss_type": "fs_auxohemce_loss", "params": params},
                        "network": {"loss_weights": {"seg_loss": 1.0, "aux_loss": 0.4}}})
    xs, xa = seg.clone().requires_grad_(True), aux.clone().requires_grad_(True)
    up = [F.interpolate(v, size=(H, W), mode="bilinear", align_corners=True) for v in (xa, xs)]
    loss = lh.FSAuxOhemCELoss(cfg)(up, target.clone())
    loss.backward()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), seg=seg.numpy(), aux=aux.numpy(), target=target.numpy(),
                        thresh=np.float64(0.5), min_kept=np.int64(800), seg_w=np.float64(1.0), aux_w=np.float64(0.4),
                        loss=np.float32(loss.item()), grad_seg=xs.grad.numpy(), grad_aux=xa.grad.numpy())
    print(f"{name}: loss={loss.item():.7f}")


if __name__ == "__main__":
    for i, c in enumerate(CASES):
        loss_case(*c, seed=90 + i)
    aux_case("ohem_aux_bilinear", seed=99)
