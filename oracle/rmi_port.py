"""Float64 restatement of the RMI segmentation loss (sigmoid path) that the contrast wrappers use with
contrast.use_rmi: RMILoss.forward -> forward_sigmoid -> rmi_lower_bound (lib/loss/rmi_loss.py:200-402), written from
its definition, in plain torch ops so autograd gives the reference gradient.

``front`` is the dtype of the up-sampling, sigmoid, BCE and pooling: float64 for the exact value, float32 for the
reference's own precisions (fp32 front end, float64 moments), which is also the torch op sequence the fused kernels
replace.  The caller's ``target`` is not modified.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

POS_ALPHA = 1e-3
CLIP_MIN = 1e-6


def rmi_loss(seg: torch.Tensor, target: torch.Tensor, *, num_classes: int, radius: int = 3, pool_way: int = 0,
             pool_stride: int = 3, weight_lambda: float = 0.5, lambda_way: int = 1, loss_weight: float = 1.0,
             front: torch.dtype = torch.float64, parts: bool = False):
    B, K = seg.shape[:2]
    H, W = target.shape[1:]
    z = seg.to(front)
    if tuple(z.shape[2:]) != (H, W):
        z = F.interpolate(z, size=(H, W), mode="bilinear", align_corners=True)
    t = torch.where(target < 0, torch.full_like(target, 255), target)
    valid = t < num_classes
    vm = valid.unsqueeze(1).to(front)
    y = F.one_hot(torch.where(valid, t, torch.zeros_like(t)), num_classes).permute(0, 3, 1, 2).to(front) * vm
    bce = (F.binary_cross_entropy_with_logits(z, y, reduction="none") * vm).sum() / (valid.sum().to(front) + 1.0)
    p = torch.sigmoid(z) * vm + CLIP_MIN
    s = pool_stride
    if s > 1:
        if pool_way == 0:
            y, p = F.max_pool2d(y, s, s, s // 2), F.max_pool2d(p, s, s, s // 2)
        elif pool_way == 1:
            y, p = F.avg_pool2d(y, s, s, s // 2), F.avg_pool2d(p, s, s, s // 2)
        else:
            raise NotImplementedError(pool_way)
    r, D = radius, radius * radius
    nY, nX = y.shape[2] - r + 1, y.shape[3] - r + 1

    def vectors(m):
        v = torch.stack([m[:, :, dy:dy + nY, dx:dx + nX] for dy in range(r) for dx in range(r)], dim=2)
        v = v.reshape(B, K, D, -1).double()
        return v - v.mean(dim=3, keepdim=True)

    xv, pv = vectors(y), vectors(p)
    eye = torch.eye(D, dtype=torch.float64, device=seg.device)
    X = xv @ xv.transpose(2, 3)
    P = pv @ pv.transpose(2, 3) + POS_ALPHA * eye
    Q = xv @ pv.transpose(2, 3)
    M = X - Q @ torch.inverse(P) @ Q.transpose(2, 3) + POS_ALPHA * eye
    chol = torch.linalg.cholesky(M)
    rmi_bc = torch.log(torch.diagonal(chol, dim1=-2, dim2=-1) + 1e-8).sum(-1)      # 0.5 * log det
    rmi = (rmi_bc.mean(dim=0) / D).sum()
    if lambda_way:
        loss = loss_weight * (weight_lambda * bce.double() + (1.0 - weight_lambda) * rmi)
    else:
        loss = loss_weight * (bce.double() + weight_lambda * rmi)
    if parts:                     # the per-(image, class) 0.5 log det M and the BCE term as well
        return loss, rmi_bc, bce
    return loss


def rmi_loss_and_grad(seg: torch.Tensor, target: torch.Tensor, grad_out: float = 1.0, **kw):
    """(loss, d loss / d seg) in float64."""
    s = seg.detach().double().requires_grad_(True)
    loss = rmi_loss(s, target, **kw)
    (loss * grad_out).backward()
    return loss.detach(), s.grad
