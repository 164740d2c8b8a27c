"""Drop-in loss modules: same class names, constructor ``(configer)``, forward signatures and registry keys
as the reference (lib/loss/loss_contrast.py, lib/loss/loss_contrast_mem.py, lib/loss/loss_manager.py:36-41).

The contrast term runs on the H100 engine (functional.pixel_contrast_loss); the plain segmentation CE runs on
the fused up-sample + CE kernels (``contrast.fused_seg_ce``, default on).  Engine-only knobs are read from
optional config keys under ``contrast``: ``rng`` ("device" | "torch_cpu"), ``nan_safe``, ``precision``
("fp32" | "bf16"), ``skip_warmup_contrast``, ``topk_negatives`` (a10 extension, default off).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .functional import ContrastOptions, pixel_contrast_loss, upsample_cross_entropy
from .loss_helper import FSAuxCELoss, FSCELoss


def _opt(configer, key, default):
    return configer.get("contrast", key) if configer.exists("contrast", key) else default


def _ignore_index(configer) -> int:
    if configer.exists("loss", "params") and "ce_ignore_index" in configer.get("loss", "params"):
        return configer.get("loss", "params")["ce_ignore_index"]
    return -1


class PixelContrastLoss(nn.Module):
    """lib/loss/loss_contrast.py:15-147 and lib/loss/loss_contrast_mem.py:15-171 (one class serves both:
    pass ``queue`` for the memory-bank variant)."""

    def __init__(self, configer):
        super().__init__()
        self.configer = configer
        self.temperature = configer.get("contrast", "temperature")
        self.base_temperature = configer.get("contrast", "base_temperature")
        self.ignore_label = _ignore_index(configer)
        self.max_samples = configer.get("contrast", "max_samples")
        self.max_views = configer.get("contrast", "max_views")
        self.num_classes = configer.get("data", "num_classes") if configer.exists("data", "num_classes") else None
        self.rng = _opt(configer, "rng", "device")
        self.nan_safe = bool(_opt(configer, "nan_safe", False))
        self.precision = _opt(configer, "precision", "fp32")
        self.seed = int(_opt(configer, "seed", 304))
        self.topk_negatives = _opt(configer, "topk_negatives", None)    # a10 extension, None = all negatives (reference)
        self.perm_fn = None            # tests inject recorded permutations here

    def options(self, normalize: bool = False) -> ContrastOptions:
        return ContrastOptions(temperature=self.temperature, base_temperature=self.base_temperature,
                               max_samples=self.max_samples, max_views=self.max_views,
                               ignore_label=self.ignore_label, num_classes=self.num_classes, normalize=normalize,
                               nan_safe=self.nan_safe, rng=self.rng, perm_fn=self.perm_fn, seed=self.seed,
                               precision=self.precision, topk_negatives=self.topk_negatives)

    def forward(self, feats, labels=None, predict=None, queue=None, seg=None, normalize: bool = False,
                bank_shadow=None):
        """feats (B,D,h,w); labels (B,Himg,Wimg) int64; predict (B,h,w) int64 (or pass the logits as ``seg`` and
        the argmax is fused into the first kernel); queue: None, a (K,R,D) tensor (the reference's
        cat(segment_queue, pixel_queue, dim=1)) or the pair (segment_queue, pixel_queue) read in place."""
        segq = pixq = None
        if queue is not None:
            if isinstance(queue, (tuple, list)):
                segq, pixq = queue
            else:
                segq = queue
        opts = self.options(normalize)
        if seg is not None:
            opts.num_classes = seg.shape[1]
        elif segq is not None and opts.num_classes is None:
            opts.num_classes = segq.shape[0]
        return pixel_contrast_loss(feats, labels, seg=seg, predict=predict if seg is None else None,
                                   segment_queue=segq, pixel_queue=pixq, bank_shadow=bank_shadow, options=opts)


class _ZeroWithGraph(torch.autograd.Function):
    """0 * contrast without running it: keeps `embed` in the autograd graph (DDP find_unused_parameters) and
    returns a zero gradient (the reference runs the whole contrast fwd+bwd during warm-up and scales it by 0,
    lib/loss/loss_contrast.py:189)."""

    @staticmethod
    def forward(ctx, embed):
        ctx.shape, ctx.dev = embed.shape, embed.device
        return embed.new_zeros(())

    @staticmethod
    def backward(ctx, g):
        return torch.zeros(ctx.shape, dtype=torch.float32, device=ctx.dev)


class ContrastCELoss(nn.Module):
    """lib/loss/loss_contrast.py:150-189 ('contrast_ce_loss')."""

    with_memory = False

    def __init__(self, configer=None, seg_criterion: Optional[nn.Module] = None):
        super().__init__()
        self.configer = configer
        self.loss_weight = configer.get("contrast", "loss_weight")
        self.use_rmi = _opt(configer, "use_rmi", False)
        self.use_lovasz = _opt(configer, "use_lovasz", False)
        if seg_criterion is None:
            if self.use_rmi or self.use_lovasz:
                raise NotImplementedError("RMI / Lovasz seg losses are outside the hot path; pass the reference "
                                          "module via seg_criterion=")
            seg_criterion = self._default_seg_criterion(configer)
        self.seg_criterion = seg_criterion
        self.contrast_criterion = PixelContrastLoss(configer)
        self.skip_warmup_contrast = bool(_opt(configer, "skip_warmup_contrast", False))
        # §8f row 1: bilinear up-sampling + CE fused in one kernel pair (no (B,K,Himg,Wimg) intermediate); applies when
        # the seg criterion is the plain mean-reduced CE of the reference configs
        self.fused_seg_ce = bool(_opt(configer, "fused_seg_ce", True))

    def _fused_ce(self, seg, target, ce_module):
        ce = ce_module.ce_loss
        return upsample_cross_entropy(seg, target, ce.weight, ce.ignore_index)

    def _can_fuse(self, ce_module, seg):
        return (self.fused_seg_ce and isinstance(ce_module, FSCELoss) and seg.is_cuda and
                ce_module.ce_loss.reduction == "mean" and getattr(ce_module.ce_loss, "label_smoothing", 0.0) == 0.0)

    @staticmethod
    def _default_seg_criterion(configer):
        return FSCELoss(configer)

    def _seg_loss(self, preds, target):
        if self._can_fuse(self.seg_criterion, preds["seg"]):
            return self._fused_ce(preds["seg"], target, self.seg_criterion)
        h, w = target.size(1), target.size(2)
        pred = F.interpolate(input=preds["seg"], size=(h, w), mode="bilinear", align_corners=True)
        return self.seg_criterion(pred, target)

    def _queues(self, preds):
        return None

    def forward(self, preds, target, with_embed=False):
        assert "seg" in preds and "embed" in preds
        seg, embedding = preds["seg"], preds["embed"]
        loss = self._seg_loss(preds, target)
        queue = self._queues(preds)
        if self.with_memory and queue is None:
            loss_contrast = 0                                   # loss_contrast_mem.py:225-226
        elif with_embed is not True and self.skip_warmup_contrast:
            loss_contrast = _ZeroWithGraph.apply(embedding)
        else:
            loss_contrast = self.contrast_criterion(embedding, target, seg=seg, queue=queue,
                                                    bank_shadow=preds.get("bank_shadow"))
        if with_embed is True:
            return loss + self.loss_weight * loss_contrast
        return loss + 0 * loss_contrast      # keeps the projection head in the DDP graph (loss_contrast.py:189)


class ContrastAuxCELoss(ContrastCELoss):
    """lib/loss/loss_contrast.py:192-234 ('contrast_auxce_loss')."""

    @staticmethod
    def _default_seg_criterion(configer):
        return FSAuxCELoss(configer)

    def _seg_loss(self, preds, target):
        assert "seg_aux" in preds
        crit = self.seg_criterion
        if isinstance(crit, FSAuxCELoss) and self._can_fuse(crit.ce_loss, preds["seg"]):
            lw = crit.configer.get("network", "loss_weights")
            return (lw["seg_loss"] * self._fused_ce(preds["seg"], target, crit.ce_loss) +
                    lw["aux_loss"] * self._fused_ce(preds["seg_aux"], target, crit.ce_loss))
        h, w = target.size(1), target.size(2)
        pred = F.interpolate(input=preds["seg"], size=(h, w), mode="bilinear", align_corners=True)
        pred_aux = F.interpolate(input=preds["seg_aux"], size=(h, w), mode="bilinear", align_corners=True)
        return self.seg_criterion([pred_aux, pred], target)


class MemContrastCELoss(ContrastCELoss):
    """lib/loss/loss_contrast_mem.py:174-231 ('mem_contrast_ce_loss'): the contrast set is the memory bank.
    The two queues are read in place (no 194.6 MB torch.cat per step)."""

    with_memory = True

    def _queues(self, preds):
        sq, pq = preds.get("segment_queue"), preds.get("pixel_queue")
        if sq is None or pq is None:
            return None
        return (sq, pq)


# registry with the reference's keys (lib/loss/loss_manager.py:36-41)
SEG_LOSS_DICT = {
    "contrast_ce_loss": ContrastCELoss,
    "contrast_auxce_loss": ContrastAuxCELoss,
    "mem_contrast_ce_loss": MemContrastCELoss,
}


def get_seg_loss(configer, loss_type: Optional[str] = None) -> nn.Module:
    """LossManager.get_seg_loss (lib/loss/loss_manager.py:61-68) for the contrast keys."""
    key = loss_type or configer.get("loss", "loss_type")
    if key not in SEG_LOSS_DICT:
        raise KeyError(f"loss type {key!r} is not a contrast loss (engine scope: {sorted(SEG_LOSS_DICT)})")
    return SEG_LOSS_DICT[key](configer)
