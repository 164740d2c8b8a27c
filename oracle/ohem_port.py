"""Float64 restatement of FSOhemCELoss.forward (lib/loss/loss_helper.py:237-261), written from its definition, in plain
torch ops so autograd gives the reference gradient.

Over the counted pixels (label not ignore_index and inside [0, K)) of the whole batch, p_t is the softmax of the target
class.  kth is the m-th smallest p_t, 0-based, m = min(max(1, min_kept), n - 1); threshold = max(kth, fp32(thresh)) and
the selected pixels are those with p_t < threshold.  loss_i = w[t_i] * nll_i; 'mean' (or 'elementwise_mean') divides the
selected sum by the selected count, 'sum' does not.  No counted pixel gives 0; an empty selection gives NaN for 'mean'
and 0 for 'sum'; both with a zero gradient.

``front`` is the dtype of the up-sampling, softmax, sort and CE: float64 for the exact value, float32 for the
reference's own precision, which is also the torch op sequence the fused kernels replace (up-sampled logits, a full
softmax, a gather, a boolean-mask copy, a sort of every counted pixel, a CE with reduction='none' and two fancy-index
copies).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def ohem_loss(seg: torch.Tensor, target: torch.Tensor, weight=None, ignore_index: int = -1, thresh: float = 0.9,
              min_kept: int = 100000, reduction: str = "mean", front: torch.dtype = torch.float64,
              near_ulps: float = 0.0, details: bool = False):
    """The loss (0-dim tensor of dtype ``front``).  With details=True, a dict instead: loss, threshold, selected
    ((B,Himg,Wimg) bool), n, count and, with near_ulps > 0, near: the counted pixels other than those equal to the
    threshold whose p_t lies within near_ulps fp32 ulps of it, where fp32 may select differently from float64."""
    if reduction not in ("mean", "elementwise_mean", "sum"):
        raise NotImplementedError("Reduction Error!")
    B, K = seg.shape[:2]
    H, W = target.shape[1:]
    z = seg.to(front)
    if tuple(z.shape[2:]) != (H, W):
        z = F.interpolate(z, size=(H, W), mode="bilinear", align_corners=True)
    t = target.to(z.device)
    valid = (t != ignore_index) & (t >= 0) & (t < K)
    tc = torch.where(valid, t, torch.zeros_like(t))
    p = torch.softmax(z, dim=1).gather(1, tc.unsqueeze(1)).squeeze(1).detach()
    w = None if weight is None else weight.to(device=z.device, dtype=front)
    nll = F.cross_entropy(z, tc, weight=w, reduction="none")             # w_t * nll_t
    n = int(valid.sum())
    thr32 = float(np.float32(thresh))
    if n == 0:
        loss = z.sum() * 0.0
        thr = torch.tensor(thr32, dtype=front)
        sel = torch.zeros_like(valid)
    else:
        sort_p = p[valid].sort().values
        kth = sort_p[min(max(1, int(min_kept)), n - 1)]
        thr = torch.maximum(kth, torch.tensor(thr32, dtype=front, device=kth.device))
        sel = valid & (p < thr)
        count = int(sel.sum())
        total = nll[sel].sum()
        if reduction == "sum":
            loss = total
        elif count == 0:
            loss = z.sum() * 0.0 + float("nan")
        else:
            loss = total / count
    if not details:
        return loss
    out = {"loss": loss, "threshold": float(thr), "selected": sel, "n": n, "count": int(sel.sum()), "p": p}
    if near_ulps > 0:
        pd, td = p.double(), float(thr)
        tol = near_ulps * 2.0 ** -23 * max(abs(td), 1e-30)
        out["near"] = valid & ((pd - td).abs() <= tol) & (pd != td)
    return out


def ohem_loss_and_grad(seg: torch.Tensor, target: torch.Tensor, grad_out: float = 1.0, **kw):
    """(details dict, d loss / d seg) in float64."""
    s = seg.detach().double().requires_grad_(True)
    d = ohem_loss(s, target, details=True, **kw)
    (d["loss"] * grad_out).backward()
    d["loss"] = d["loss"].detach()
    return d, s.grad


def gap_labels(seg: torch.Tensor, target: torch.Tensor, ignore_index: int = -1, near_ulps: float = 64, **kw):
    """A copy of target with the near-threshold pixels (ohem_loss's near mask) ignored, repeated until none is left:
    inputs on which fp32 and float64 select the same pixels."""
    t = target.clone()
    for _ in range(20):
        near = ohem_loss(seg, t, ignore_index=ignore_index, near_ulps=near_ulps, details=True, **kw)["near"]
        if not bool(near.any()):
            return t
        t[near.to(t.device)] = ignore_index
    raise RuntimeError("near-threshold pixels remain")
