"""Segmentation losses used inside the contrast wrappers (lib/loss/loss_helper.py:169-212, :215-280, :316-369).

The CE modules are plain PyTorch ops so the wrappers are drop-in (the wrappers run the fused up-sample + CE kernels
instead when they can, SURVEY §8f row 1).  The RMI modules (contrast.use_rmi) run the fused RMI kernels
(functional.upsample_rmi_loss, §8f row f5).  FSCELOVASZLoss adds the Lovasz-softmax term of the fused up-sample +
Lovasz kernels (functional.upsample_lovasz_softmax, §8f row f6) to the CE.  FSOhemCELoss and the seg term of
FSAuxOhemCELoss run the fused up-sample + OHEM CE kernels (functional.upsample_ohem_cross_entropy, §8f row f7).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from .functional import upsample_lovasz_softmax, upsample_ohem_cross_entropy, upsample_rmi_loss


def _ce_params(configer):
    weight, reduction, ignore_index = None, "mean", -1
    if configer is not None and configer.exists("loss", "params"):
        p = configer.get("loss", "params")
        if "ce_weight" in p:
            weight = torch.tensor(p["ce_weight"], dtype=torch.float32)
        if "ce_reduction" in p:
            reduction = {"elementwise_mean": "mean"}.get(p["ce_reduction"], p["ce_reduction"])
        if "ce_ignore_index" in p:
            ignore_index = p["ce_ignore_index"]
    return weight, reduction, ignore_index


def _scale_target(target: torch.Tensor, size) -> torch.Tensor:
    t = target.clone().unsqueeze(1).float()
    return F.interpolate(t, size=size, mode="nearest").squeeze(1).long()


class FSCELoss(nn.Module):
    def __init__(self, configer=None):
        super().__init__()
        weight, reduction, ignore_index = _ce_params(configer)
        self.ce_loss = nn.CrossEntropyLoss(weight=weight, ignore_index=ignore_index, reduction=reduction)

    def forward(self, inputs, *targets, weights=None, **kwargs):
        if isinstance(inputs, (tuple, list)):
            weights = weights or [1.0] * len(inputs)
            loss = 0.0
            for i, x in enumerate(inputs):
                tgt = targets[i] if len(targets) > 1 else targets[0]
                loss = loss + weights[i] * self.ce_loss(x, _scale_target(tgt, (x.size(2), x.size(3))))
            return loss
        return self.ce_loss(inputs, _scale_target(targets[0], (inputs.size(2), inputs.size(3))))


class FSAuxCELoss(nn.Module):
    """seg_loss_weight * CE(seg) + aux_loss_weight * CE(aux)  (lib/loss/loss_helper.py:301-313)."""

    def __init__(self, configer=None):
        super().__init__()
        self.configer = configer
        self.ce_loss = FSCELoss(configer)

    def forward(self, inputs, targets, **kwargs):
        aux_out, seg_out = inputs
        w = self.configer.get("network", "loss_weights")
        return w["seg_loss"] * self.ce_loss(seg_out, targets) + w["aux_loss"] * self.ce_loss(aux_out, targets)


class RMILoss(nn.Module):
    """lib/loss/rmi_loss.py:200-402 (sigmoid path, ``forward``) on the engine.  Reads the reference's ``loss.params``
    keys: num_classes, rmi_radius, rmi_pool_way, rmi_pool_size (== rmi_pool_stride), rmi_pool_stride,
    loss_weight_lambda, loss_weight, lambda_way; use_sigmoid is read and ignored, as the reference's forward always
    takes the sigmoid path.  ``cls_score`` may be the logits at label resolution (the reference's call) or below it:
    the bilinear up-sampling (align_corners=True) is fused.  Unlike the reference, ``label`` is left unchanged."""

    def __init__(self, configer=None):
        super().__init__()
        p = configer.get("loss", "params")
        self.use_sigmoid = p["use_sigmoid"]
        self.num_classes = p["num_classes"]
        self.rmi_radius = p["rmi_radius"]
        assert self.rmi_radius in range(1, 11)
        self.rmi_pool_way = p["rmi_pool_way"]
        assert self.rmi_pool_way in (0, 1, 2, 3)
        self.rmi_pool_size = p["rmi_pool_size"]
        self.rmi_pool_stride = p["rmi_pool_stride"]
        assert self.rmi_pool_size == self.rmi_pool_stride
        self.weight_lambda = p["loss_weight_lambda"]
        self.loss_weight = p["loss_weight"]
        self.lambda_way = p["lambda_way"]

    def forward(self, cls_score, label, weight=None, **kwargs):
        return upsample_rmi_loss(cls_score, label, num_classes=self.num_classes, radius=self.rmi_radius,
                                 pool_way=self.rmi_pool_way, pool_stride=self.rmi_pool_stride,
                                 weight_lambda=self.weight_lambda, lambda_way=self.lambda_way,
                                 loss_weight=self.loss_weight)


class FSRMILoss(nn.Module):
    """RMI(seg)  (lib/loss/loss_helper.py:359-369)."""

    def __init__(self, configer=None):
        super().__init__()
        self.configer = configer
        self.rmi_loss = RMILoss(configer)

    def forward(self, inputs, targets, **kwargs):
        return self.rmi_loss(inputs, targets)


class FSAuxRMILoss(nn.Module):
    """seg_loss_weight * RMI(seg) + aux_loss_weight * CE(aux)  (lib/loss/loss_helper.py:316-330)."""

    def __init__(self, configer=None):
        super().__init__()
        self.configer = configer
        self.ce_loss = FSCELoss(configer)
        self.rmi_loss = RMILoss(configer)

    def forward(self, inputs, targets, **kwargs):
        aux_out, seg_out = inputs
        w = self.configer.get("network", "loss_weights")
        return w["seg_loss"] * self.rmi_loss(seg_out, targets) + w["aux_loss"] * self.ce_loss(aux_out, targets)


class FSCELOVASZLoss(nn.Module):
    """CE + Lovasz-softmax  (lib/loss/loss_helper.py:77-124).  Reads ce_weight, ce_reduction and ce_ignore_index.  A
    single tensor gives CE + Lovasz at the input's resolution (the target nearest-scaled to it); a list or tuple gives
    the weighted CE sum of the reference's list branch, without the Lovasz term.  The Lovasz term runs on the engine
    (upsample_lovasz_softmax with the identity geometry); the contrast wrappers hand it the low-resolution logits
    instead, with the up-sampling fused."""

    def __init__(self, configer=None):
        super().__init__()
        self.configer = configer
        weight, reduction, ignore_index = _ce_params(configer)
        self.ignore_index = ignore_index
        self.ce_loss = nn.CrossEntropyLoss(weight=weight, ignore_index=ignore_index, reduction=reduction)

    def forward(self, inputs, *targets, weights=None, **kwargs):
        if isinstance(inputs, dict) and "seg" in inputs:
            inputs = inputs["seg"]
        if isinstance(inputs, (tuple, list)):
            weights = weights or [1.0] * len(inputs)
            loss = 0.0
            for i, x in enumerate(inputs):
                tgt = targets[i] if len(targets) > 1 else targets[0]
                loss = loss + weights[i] * self.ce_loss(x, _scale_target(tgt, (x.size(2), x.size(3))))
            return loss
        target = _scale_target(targets[0], (inputs.size(2), inputs.size(3)))
        return self.ce_loss(inputs, target) + upsample_lovasz_softmax(inputs, target, self.ignore_index)


class FSOhemCELoss(nn.Module):
    """OHEM cross-entropy  (lib/loss/loss_helper.py:215-261) on the engine (upsample_ohem_cross_entropy).  Reads
    ohem_thresh, ohem_minkeep (min_kept = max(1, ohem_minkeep)), ce_weight, ce_reduction ('elementwise_mean' by default,
    'mean' accepted as its alias, 'sum'; anything else raises NotImplementedError in forward) and ce_ignore_index.
    ``predict`` may be the logits at label resolution (the reference's call) or below it: the bilinear up-sampling
    (align_corners=True) is fused.  Labels outside [0, K) count as ignored; no labelled pixel gives 0."""

    def __init__(self, configer=None):
        super().__init__()
        self.configer = configer
        p = configer.get("loss", "params")
        self.thresh = p["ohem_thresh"]
        self.min_kept = max(1, p["ohem_minkeep"])
        weight, reduction, ignore_index = _ce_params(configer)
        self.register_buffer("weight", weight, persistent=False)
        self.reduction = reduction
        self.ignore_label = ignore_index

    def forward(self, predict, target, **kwargs):
        return upsample_ohem_cross_entropy(predict, target, self.weight, self.ignore_label, self.thresh, self.min_kept,
                                           self.reduction)


class FSAuxOhemCELoss(nn.Module):
    """seg_loss_weight * OHEM CE(seg) + aux_loss_weight * CE(aux)  (lib/loss/loss_helper.py:264-281).  Always the OHEM
    CE: unlike the reference, loss.loss_type is not asserted, so the module can be built from a contrast config."""

    def __init__(self, configer=None):
        super().__init__()
        self.configer = configer
        self.ce_loss = FSCELoss(configer)
        self.ohem_ce_loss = FSOhemCELoss(configer)

    def forward(self, inputs, targets, **kwargs):
        aux_out, seg_out = inputs
        w = self.configer.get("network", "loss_weights")
        return w["seg_loss"] * self.ohem_ce_loss(seg_out, targets) + w["aux_loss"] * self.ce_loss(aux_out, targets)
