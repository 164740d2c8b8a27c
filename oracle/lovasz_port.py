"""Float64 restatement of the Lovasz-softmax term of FSCELOVASZLoss (lovasz_softmax_flat(*flatten_probas(softmax(pred),
target, ignore_index), only_present=True), lib/loss/lovasz_loss.py:216-267), written from its definition, in plain
torch ops so autograd gives the reference gradient.

Pixels are pooled over the batch; a pixel counts when its label is not ignore_index and lies in [0, K).  Per present
class c, the errors e = |fg - p_c| are sorted descending with ties in ascending pixel index (a stable sort), and
loss_c = sum_i e_(i) g_i with the closed form of the Lovasz gradient: g = 1/U for a fg step, I/(U(U+1)) for a bg step,
I = gts - cumfg, U = gts + cumbg counted before the step.  The loss is the mean over the present classes, 0 when none.

``front`` is the dtype of the up-sampling and the softmax: float64 for the exact value, float32 for the reference's
own precision, which is also the torch op sequence the fused kernels replace.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _probas(seg, H, W, front):
    z = seg.to(front)
    if tuple(z.shape[2:]) != (H, W):
        z = F.interpolate(z, size=(H, W), mode="bilinear", align_corners=True)
    return torch.softmax(z, dim=1)


def lovasz_loss(seg: torch.Tensor, target: torch.Tensor, ignore_index: int = -1, front: torch.dtype = torch.float64,
                near_tie_ulps: float = 0.0):
    """The loss (0-dim float64 tensor).  With near_tie_ulps > 0, also a (B, Himg, Wimg) bool mask of the near-tie
    pixels: counted pixels whose error lies within near_tie_ulps fp32 ulps (of max(e, p_c)) of the error of a pixel of
    the same class with the opposite fg flag, where fp32 may order the pair differently from float64."""
    B, K = seg.shape[:2]
    H, W = target.shape[1:]
    p = _probas(seg, H, W, front).permute(0, 2, 3, 1).reshape(-1, K)
    t = target.reshape(-1).to(p.device)
    valid = (t != ignore_index) & (t >= 0) & (t < K)
    pv, tv = p[valid], t[valid]
    idx = torch.nonzero(valid).squeeze(1)
    near = torch.zeros(t.numel(), dtype=torch.bool, device=p.device) if near_tie_ulps > 0 else None
    losses = []
    for c in range(K):
        fg = tv == c
        gts = int(fg.sum())
        if gts == 0:
            continue
        e = (fg.to(p.dtype) - pv[:, c]).abs()
        order = torch.sort(e.detach(), descending=True, stable=True).indices
        fgs = fg[order].to(torch.float64)
        F_before = torch.cumsum(fgs, 0) - fgs
        Bg_before = torch.cumsum(1.0 - fgs, 0) - (1.0 - fgs)
        I, U = gts - F_before, gts + Bg_before
        g = torch.where(fgs > 0, 1.0 / U, I / (U * (U + 1.0)))
        losses.append((e[order].to(torch.float64) * g).sum())
        if near is not None:
            ed = e.detach().double()
            tol = near_tie_ulps * 2.0 ** -24 * torch.maximum(ed, pv[:, c].detach().double())
            asc, perm = torch.sort(ed)
            fga = fg[perm].to(torch.int64)
            cum = torch.cat([torch.zeros(1, dtype=torch.int64, device=ed.device), torch.cumsum(fga, 0)])
            lo = torch.searchsorted(asc, asc - tol[perm], right=False)
            hi = torch.searchsorted(asc, asc + tol[perm], right=True)
            nfg = cum[hi] - cum[lo]
            nbg = (hi - lo) - nfg
            hit = torch.where(fga > 0, nbg > 0, nfg > 0)
            near[idx[perm[hit]]] = True
    loss = torch.stack(losses).mean() if losses else torch.zeros((), dtype=torch.float64, device=p.device)
    if near is not None:
        return loss, near.view(target.shape)
    return loss


def lovasz_loss_and_grad(seg: torch.Tensor, target: torch.Tensor, grad_out: float = 1.0, **kw):
    """(loss, d loss / d seg) in float64 (with near_tie_ulps > 0: and the near-tie mask)."""
    s = seg.detach().double().requires_grad_(True)
    out = lovasz_loss(s, target, **kw)
    loss = out[0] if isinstance(out, tuple) else out
    if loss.requires_grad:
        (loss * grad_out).backward()
    grad = s.grad if s.grad is not None else torch.zeros_like(s)
    if isinstance(out, tuple):
        return loss.detach(), grad, out[1]
    return loss.detach(), grad


def footprint_mask(near: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """(B, h, w) bool: the low-resolution logits whose bilinear footprint holds a near-tie pixel (every class plane)."""
    B, H, W = near.shape
    if (H, W) == (h, w):
        return near.clone()
    x = torch.zeros(B, 1, h, w, dtype=torch.float64, device=near.device, requires_grad=True)
    up = F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)
    (up[:, 0] * near.to(torch.float64)).sum().backward()
    return x.grad[:, 0] != 0
