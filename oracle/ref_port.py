"""CPU port of the reference pixel-contrast hot path (TEST INFRASTRUCTURE — see oracle/__init__).

Each function restates one reference function and cites it (paths relative to the
tfzhou/ContrastiveSeg tree).  The arithmetic lives in torch/ATen (reference pins
``torch>=1.7.0``, requirements.txt:16); this port runs the same ATen ops on CPU in a selectable
dtype: float64 when used as the parity checker, float32 when timed as the CPU baseline.

Parity: pinned against the imported reference modules and against golden vectors they produced
(tests/test_oracle_vs_reference.py, tests/test_golden.py).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

PermFn = Callable[[int], torch.Tensor]
_torch_randperm = torch.randperm      # bound at import: tests patch torch.randperm to route it here


class PermRecorder:
    """perm_fn that draws torch.randperm (CPU generator) and remembers every draw."""

    def __init__(self, generator: Optional[torch.Generator] = None):
        self.generator = generator
        self.draws: List[torch.Tensor] = []

    def __call__(self, n: int) -> torch.Tensor:
        p = _torch_randperm(n, generator=self.generator) if self.generator is not None else _torch_randperm(n)
        self.draws.append(p.clone())
        return p


class PermReplay:
    """perm_fn that replays recorded permutations in call order."""

    def __init__(self, draws: Sequence[torch.Tensor]):
        self.draws = [torch.as_tensor(d, dtype=torch.long) for d in draws]
        self.pos = 0

    def __call__(self, n: int) -> torch.Tensor:
        p = self.draws[self.pos]
        self.pos += 1
        if p.numel() != n:
            raise ValueError(f"replayed permutation #{self.pos - 1} has length {p.numel()}, expected {n}")
        return p


# --------------------------------------------------------------------------------------------
# a3: label down-sampling — lib/loss/loss_contrast.py:131-134
# --------------------------------------------------------------------------------------------
def downsample_labels(target: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """(B,Himg,Wimg) int64 -> (B,h,w) int64 through float nearest interpolation."""
    t = target.unsqueeze(1).to(torch.float32)
    t = F.interpolate(t, size=(h, w), mode="nearest")
    return t.squeeze(1).long()


# --------------------------------------------------------------------------------------------
# a4: hard-anchor sampling — lib/loss/loss_contrast.py:30-89
# --------------------------------------------------------------------------------------------
def kept_classes(lab_row: torch.Tensor, ignore_label: int, max_views: int) -> List[int]:
    """Classes of one image that take part: not ignore, strictly more than max_views pixels
    (loss_contrast.py:37-39)."""
    ids, cnt = torch.unique(lab_row, return_counts=True)
    return [int(c) for c, n in zip(ids.tolist(), cnt.tolist()) if c != ignore_label and n > max_views]


def split_hard_easy(num_hard: int, num_easy: int, n_view: int) -> Tuple[int, int]:
    """How many hard / easy pixels one (image, class) contributes (loss_contrast.py:66-77)."""
    half = n_view / 2
    if num_hard >= half and num_easy >= half:
        keep_hard = n_view // 2
        keep_easy = n_view - keep_hard
    elif num_hard >= half:
        keep_easy = num_easy
        keep_hard = n_view - keep_easy
    elif num_easy >= half:
        keep_hard = num_hard
        keep_easy = n_view - keep_hard
    else:  # unreachable when count > max_views >= n_view (loss_contrast.py:75-77 raises)
        raise RuntimeError(f"hard/easy split impossible: {num_hard} {num_easy} {n_view}")
    return keep_hard, keep_easy


def sample_anchor_indices(lab: torch.Tensor, prd: torch.Tensor, max_samples: int, max_views: int,
                          ignore_label: int, perm_fn: PermFn):
    """lab, prd: (B,HW) int64 (GT at embedding resolution, argmax prediction).

    Returns (idx (TC,V) int64 pixel indices, cls (TC,) int64, img (TC,) int64, n_view) or None
    when no class qualifies (the reference returns (None, None) and then crashes, Q8).
    RNG call order: image ascending, class ascending, randperm(num_hard) then randperm(num_easy)
    (loss_contrast.py:79-82)."""
    B = lab.shape[0]
    per_image = [kept_classes(lab[b], ignore_label, max_views) for b in range(B)]
    total = sum(len(c) for c in per_image)
    if total == 0:
        return None
    n_view = min(max_samples // total, max_views)
    rows, cls, img = [], [], []
    for b in range(B):
        for c in per_image[b]:
            is_c = lab[b] == c
            hard = (is_c & (prd[b] != c)).nonzero()[:, 0]
            easy = (is_c & (prd[b] == c)).nonzero()[:, 0]
            kh, ke = split_hard_easy(hard.numel(), easy.numel(), n_view)
            ph = perm_fn(hard.numel())
            pe = perm_fn(easy.numel())
            rows.append(torch.cat([hard[ph[:kh]], easy[pe[:ke]]]))
            cls.append(c)
            img.append(b)
    if n_view == 0:
        idx = torch.zeros((total, 0), dtype=torch.long)
    else:
        idx = torch.stack(rows)
    return idx, torch.tensor(cls, dtype=torch.long), torch.tensor(img, dtype=torch.long), n_view


# --------------------------------------------------------------------------------------------
# a5: bank flattening — lib/loss/loss_contrast_mem.py:91-105   (quirks Q2, Q3)
# --------------------------------------------------------------------------------------------
def flatten_queue(queue: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(K,R,D) -> rows (K*R,D), labels (K*R,).  Class 0 is skipped, so classes 1..K-1 fill the
    first (K-1)*R rows and the last R rows stay zero with label 0."""
    K, R, D = queue.shape
    rows = torch.zeros((K * R, D), dtype=queue.dtype, device=queue.device)
    labels = torch.zeros((K * R,), dtype=queue.dtype, device=queue.device)
    at = 0
    for c in range(1, K):
        rows[at:at + R] = queue[c]
        labels[at:at + R] = c
        at += R
    return rows, labels


# --------------------------------------------------------------------------------------------
# a6: InfoNCE — lib/loss/loss_contrast.py:91-128, lib/loss/loss_contrast_mem.py:107-152
# --------------------------------------------------------------------------------------------
def infonce_dense(anchors: torch.Tensor, ya: torch.Tensor, contrast: torch.Tensor, yc: torch.Tensor,
                  temperature: float, base_temperature: float) -> torch.Tensor:
    """Dense formulation with the same tensor temporaries as the reference (autograd-capable).
    anchors (A,D) in the reference's view-major row order; the (i,i) entry is removed from the
    positives in both modes (Q1); all negatives are used (no top-k)."""
    A = anchors.shape[0]
    same = torch.eq(ya.view(-1, 1), yc.view(1, -1)).to(anchors.dtype)
    logits = torch.matmul(anchors, contrast.t()) / temperature
    logits = logits - logits.max(dim=1, keepdim=True).values.detach()
    diff = 1 - same
    keep = torch.ones_like(same)
    keep[torch.arange(A), torch.arange(A)] = 0
    pos = same * keep
    e = torch.exp(logits)
    neg_sum = (e * diff).sum(1, keepdim=True)
    log_prob = logits - torch.log(e + neg_sum)
    mean_log_prob_pos = (pos * log_prob).sum(1) / pos.sum(1)
    return (-(temperature / base_temperature) * mean_log_prob_pos).mean()


def infonce_closed_form(anchors: torch.Tensor, ya: torch.Tensor, contrast: torch.Tensor, yc: torch.Tensor,
                        temperature: float, base_temperature: float, self_contrast: bool,
                        diag_cols: Optional[torch.Tensor] = None):
    """Loss, analytic gradient and the per-row statistics the kernels keep (SURVEY appendix A).

    diag_cols[i] = the contrast column removed from anchor i's positives (default i, Q1).
    Returns dict(loss, dA, row_loss, m, neg, s, npos)."""
    A = anchors.shape[0]
    if diag_cols is None:
        diag_cols = torch.arange(A)
    l = (anchors @ contrast.t()) / temperature
    m = l.max(1, keepdim=True).values
    e = torch.exp(l - m)
    same = ya.view(-1, 1) == yc.view(1, -1)
    neg = (e * (~same)).sum(1, keepdim=True)
    pos = same.clone()
    pos[torch.arange(A), diag_cols] = False
    npos = pos.sum(1, keepdim=True).to(anchors.dtype)
    logp = (l - m) - torch.log(e + neg)
    row_loss = -(temperature / base_temperature) * (logp * pos).sum(1, keepdim=True) / npos
    loss = row_loss.mean()
    c = (temperature / base_temperature) / (A * npos)
    inv = 1.0 / (e + neg)
    s = (pos * inv).sum(1, keepdim=True)
    G = torch.where(pos, -c * (1 - e * inv), torch.zeros_like(e)) + torch.where(~same, c * e * s, torch.zeros_like(e))
    dA = (G @ contrast) / temperature
    if self_contrast:
        dA = dA + (G.t() @ anchors) / temperature
    return dict(loss=loss, dA=dA, row_loss=row_loss[:, 0], m=m[:, 0], neg=neg[:, 0], s=s[:, 0], npos=npos[:, 0], G=G)


def topk_negative_weights(l: torch.Tensor, neg_mask: torch.Tensor, k: Optional[int]):
    """a10 selection weights (EXTENSION — the reference has no top-k code; semantics defined by SURVEY §8 a10 and
    contrastiveseg_b200/csrc/pcl_topk.cuh).  l (A,N) logits, neg_mask (A,N) bool.  Per row: tau = k-th largest
    negative logit, weight 1 above tau, (k - G)/E on the E ties at tau, 0 below; rows with <= k negatives keep all.
    Returns (w, tau, G, E) with tau = -inf / E = 0 for rows that keep everything."""
    A, N = l.shape
    w = neg_mask.to(l.dtype)
    n_neg = neg_mask.sum(1)
    tau = torch.full((A,), float("-inf"), dtype=l.dtype)
    G = n_neg.clone()
    E = torch.zeros_like(n_neg)
    if k is None:
        return w, tau, G, E
    lneg = torch.where(neg_mask, l, torch.full_like(l, float("-inf")))
    srt = torch.sort(lneg, dim=1, descending=True).values
    for i in range(A):
        if int(n_neg[i]) <= k:
            continue
        t = srt[i, k - 1]
        gt = neg_mask[i] & (l[i] > t)
        eq = neg_mask[i] & (l[i] == t)
        g, e = int(gt.sum()), int(eq.sum())
        w[i] = gt.to(l.dtype) + eq.to(l.dtype) * ((k - g) / e)
        tau[i], G[i], E[i] = t, g, e
    return w, tau, G, E


def infonce_dense_topk(anchors: torch.Tensor, ya: torch.Tensor, contrast: torch.Tensor, yc: torch.Tensor,
                       temperature: float, base_temperature: float, k: Optional[int]) -> torch.Tensor:
    """infonce_dense (autograd-capable, (i,i) removed from the positives) with the a10 selection weights on the
    negatives; the weights are computed from the detached logits (piecewise-constant selection)."""
    A = anchors.shape[0]
    same = torch.eq(ya.view(-1, 1), yc.view(1, -1))
    logits = torch.matmul(anchors, contrast.t()) / temperature
    w, _, _, _ = topk_negative_weights(logits.detach(), ~same, k)
    logits = logits - logits.max(dim=1, keepdim=True).values.detach()
    keep = torch.ones_like(logits)
    keep[torch.arange(A), torch.arange(A)] = 0
    pos = same.to(anchors.dtype) * keep
    e = torch.exp(logits)
    neg_sum = (e * w).sum(1, keepdim=True)
    log_prob = logits - torch.log(e + neg_sum)
    mean_log_prob_pos = (pos * log_prob).sum(1) / pos.sum(1)
    return (-(temperature / base_temperature) * mean_log_prob_pos).mean()


def infonce_topk(anchors: torch.Tensor, ya: torch.Tensor, contrast: torch.Tensor, yc: torch.Tensor,
                 temperature: float, base_temperature: float, k: Optional[int], self_contrast: bool,
                 diag_cols: Optional[torch.Tensor] = None):
    """infonce_closed_form with the a10 top-k hard-negative selection on Neg_i (k=None == the reference).
    The selection is piecewise constant: the gradient treats the weights as constants."""
    A = anchors.shape[0]
    if diag_cols is None:
        diag_cols = torch.arange(A)
    l = (anchors @ contrast.t()) / temperature
    m = l.max(1, keepdim=True).values
    e = torch.exp(l - m)
    same = ya.view(-1, 1) == yc.view(1, -1)
    w, tau, Gc, Ec = topk_negative_weights(l, ~same, k)
    neg = (e * w).sum(1, keepdim=True)
    pos = same.clone()
    pos[torch.arange(A), diag_cols] = False
    npos = pos.sum(1, keepdim=True).to(anchors.dtype)
    logp = (l - m) - torch.log(e + neg)
    row_loss = -(temperature / base_temperature) * (logp * pos).sum(1, keepdim=True) / npos
    loss = row_loss.mean()
    c = (temperature / base_temperature) / (A * npos)
    inv = 1.0 / (e + neg)
    s = (pos * inv).sum(1, keepdim=True)
    G = torch.where(pos, -c * (1 - e * inv), torch.zeros_like(e)) + w * c * e * s
    dA = (G @ contrast) / temperature
    if self_contrast:
        dA = dA + (G.t() @ anchors) / temperature
    return dict(loss=loss, dA=dA, row_loss=row_loss[:, 0], m=m[:, 0], neg=neg[:, 0], s=s[:, 0], npos=npos[:, 0],
                tau=tau, n_above=Gc, n_ties=Ec, w=w)


# --------------------------------------------------------------------------------------------
# a3+a4+a6: PixelContrastLoss.forward — loss_contrast.py:130-147, loss_contrast_mem.py:154-171
# --------------------------------------------------------------------------------------------
def pixel_contrast_loss(feats: torch.Tensor, labels: torch.Tensor, predict: torch.Tensor, *,
                        temperature: float, base_temperature: float, max_samples: int, max_views: int,
                        ignore_label: int = -1, queue: Optional[torch.Tensor] = None,
                        perm_fn: Optional[PermFn] = None, per_pair_gather: bool = True,
                        return_details: bool = False):
    """feats (B,D,h,w) L2-normalised embedding (requires_grad allowed), labels (B,Himg,Wimg) int64,
    predict (B,h,w) int64, queue (K,R,D) or None.

    per_pair_gather=True indexes the (B,HW,D) tensor once per (image, class) like the reference
    (loss_contrast.py:83-85), which is what makes the reference backward expensive (one
    SelectBackward per pair); False uses one batched gather (same values)."""
    perm_fn = perm_fn or (lambda n: torch.randperm(n))
    B, D, h, w = feats.shape
    lab = downsample_labels(labels, h, w).reshape(B, -1)
    prd = predict.reshape(B, -1)
    X = feats.permute(0, 2, 3, 1).contiguous().view(B, h * w, D)

    plan = sample_anchor_indices(lab, prd, max_samples, max_views, ignore_label, perm_fn)
    if plan is None:
        raise RuntimeError("no class qualifies for anchor sampling (reference crashes here, Q8)")
    idx, cls, img, n_view = plan
    TC = idx.shape[0]
    if per_pair_gather:
        X_ = torch.zeros((TC, n_view, D), dtype=feats.dtype, device=feats.device)   # loss_contrast.py:51 (.cuda())
        for t in range(TC):
            X_[t] = X[int(img[t]), idx[t], :]
    else:
        X_ = X[img.view(-1, 1).to(idx.device), idx]
    y_ = cls.to(device=feats.device, dtype=feats.dtype)                              # loss_contrast.py:52 (.cuda())

    # view-major reordering: row r = v*TC + t (loss_contrast.py:98)
    anchors = torch.cat(torch.unbind(X_, dim=1), dim=0)
    ya = y_.repeat(n_view)
    if queue is not None:
        contrast, yc = flatten_queue(queue.to(feats.dtype))
    else:
        contrast, yc = anchors, ya
    loss = infonce_dense(anchors, ya, contrast, yc, temperature, base_temperature)
    if return_details:
        return loss, dict(idx=idx, cls=cls, img=img, n_view=n_view, anchors=anchors, ya=ya,
                          contrast=contrast, yc=yc, lab=lab, prd=prd)
    return loss


# --------------------------------------------------------------------------------------------
# a8: memory-bank update — segmentor/trainer_contrastive.py:102-138   (quirks Q2, Q4, Q5, Q6)
# --------------------------------------------------------------------------------------------
def dequeue_and_enqueue(keys: torch.Tensor, labels: torch.Tensor, segment_queue: torch.Tensor,
                        segment_queue_ptr: torch.Tensor, pixel_queue: torch.Tensor,
                        pixel_queue_ptr: torch.Tensor, *, network_stride: int, memory_size: int,
                        pixel_update_freq: int, perm_fn: Optional[PermFn] = None) -> None:
    """In place on the four buffers.  keys (B,D,h,w), labels (B,Himg,Wimg) int64."""
    perm_fn = perm_fn or (lambda n: torch.randperm(n))
    B, D = keys.shape[0], keys.shape[1]
    sub = labels[:, ::network_stride, ::network_stride]
    for b in range(B):
        feat = keys[b].contiguous().view(D, -1)
        lb = sub[b].contiguous().view(-1)
        for c in [int(x) for x in torch.unique(lb).tolist() if x > 0]:
            where = (lb == c).nonzero()[:, 0]              # flat index in the sub-sampled map (Q6)
            seg = feat[:, where].mean(dim=1)
            sp = int(segment_queue_ptr[c])
            segment_queue[c, sp, :] = F.normalize(seg, p=2, dim=0)
            segment_queue_ptr[c] = (sp + 1) % memory_size
            n = where.numel()
            perm = perm_fn(n)
            k = min(n, pixel_update_freq)
            rows = F.normalize(feat[:, perm[:k]].t(), p=2, dim=1)   # perm indexes columns directly (Q5)
            pp = int(pixel_queue_ptr[c])
            if pp + k >= memory_size:
                pixel_queue[c, memory_size - k:, :] = rows
                pixel_queue_ptr[c] = 0
            else:
                pixel_queue[c, pp:pp + k, :] = rows
                pixel_queue_ptr[c] = (pp + 1) % memory_size       # +1, not +k (Q4)


# --------------------------------------------------------------------------------------------
# a1: projection-head normalise — lib/models/modules/projection.py:24
# --------------------------------------------------------------------------------------------
def l2_normalize(x: torch.Tensor) -> torch.Tensor:
    return F.normalize(x, p=2, dim=1)


# --------------------------------------------------------------------------------------------
# a2: ContrastCELoss.forward — loss_contrast.py:171-189, loss_contrast_mem.py:198-231
# --------------------------------------------------------------------------------------------
def seg_cross_entropy(seg: torch.Tensor, target: torch.Tensor, ignore_index: int = -1,
                      weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """FSCELoss on bilinearly up-sampled logits (loss_contrast.py:180-181, loss_helper.py:169-212)."""
    h, w = target.shape[1], target.shape[2]
    up = F.interpolate(seg, size=(h, w), mode="bilinear", align_corners=True)
    return F.cross_entropy(up, target, weight=weight, ignore_index=ignore_index, reduction="mean")


def contrast_ce_loss(preds: dict, target: torch.Tensor, *, with_embed: bool, loss_weight: float,
                     temperature: float, base_temperature: float, max_samples: int, max_views: int,
                     ignore_label: int = -1, with_memory: bool = False, ce_weight=None,
                     perm_fn: Optional[PermFn] = None, per_pair_gather: bool = True) -> torch.Tensor:
    seg, embed = preds["seg"], preds["embed"]
    loss = seg_cross_entropy(seg, target, ignore_label, ce_weight)
    predict = seg.argmax(dim=1)
    queue = None
    if with_memory:
        if "segment_queue" in preds and "pixel_queue" in preds:
            queue = torch.cat((preds["segment_queue"], preds["pixel_queue"]), dim=1)   # mem:221
        else:
            return loss                                                                 # mem:225-226
    lc = pixel_contrast_loss(embed, target, predict, temperature=temperature,
                             base_temperature=base_temperature, max_samples=max_samples,
                             max_views=max_views, ignore_label=ignore_label, queue=queue,
                             perm_fn=perm_fn, per_pair_gather=per_pair_gather)
    if with_embed:
        return loss + loss_weight * lc
    return loss + 0 * lc


def contrast_auxce_loss(preds: dict, target: torch.Tensor, *, with_embed: bool, loss_weight: float,
                        seg_loss_weight: float, aux_loss_weight: float, temperature: float, base_temperature: float,
                        max_samples: int, max_views: int, ignore_label: int = -1, ce_weight=None,
                        perm_fn: Optional[PermFn] = None, per_pair_gather: bool = True) -> torch.Tensor:
    """ContrastAuxCELoss.forward — lib/loss/loss_contrast.py:213-234: FSAuxCELoss (lib/loss/loss_helper.py:301-313:
    seg_loss * CE(up(seg)) + aux_loss * CE(up(seg_aux)), both bilinear align_corners=True, :223-225) + the no-bank
    pixel-contrast term on predict = argmax(seg) (:227-228); `loss + loss_weight * lc` or `loss + 0 * lc` (:230-234)."""
    seg, seg_aux, embed = preds["seg"], preds["seg_aux"], preds["embed"]
    loss = (seg_loss_weight * seg_cross_entropy(seg, target, ignore_label, ce_weight) +
            aux_loss_weight * seg_cross_entropy(seg_aux, target, ignore_label, ce_weight))
    predict = seg.argmax(dim=1)
    lc = pixel_contrast_loss(embed, target, predict, temperature=temperature, base_temperature=base_temperature,
                             max_samples=max_samples, max_views=max_views, ignore_label=ignore_label, queue=None,
                             perm_fn=perm_fn, per_pair_gather=per_pair_gather)
    if with_embed:
        return loss + loss_weight * lc
    return loss + 0 * lc
