"""H100-native pixel-contrast loss engine: drop-in for the loss path of tfzhou/ContrastiveSeg.

Public surface mirrors the reference (SURVEY §8b): ``PixelContrastLoss``, ``ContrastCELoss``,
``ContrastAuxCELoss``, ``MemContrastCELoss`` (registry keys in ``SEG_LOSS_DICT``), ``MemoryBank`` /
``dequeue_and_enqueue``, ``ProjectionHead`` / ``l2_normalize`` and the trainer hook.  All arithmetic runs in
hand-written sm_90a kernels (csrc/) behind the C ABI of include/pcl.h; there is no CPU or PyTorch fallback.
"""
from .configer import Configer, cityscapes_contrast_config            # noqa: F401
from .functional import ContrastOptions, l2_normalize, pixel_contrast_loss, project_normalize, upsample_cross_entropy  # noqa: F401,E501
from .functional import bn_relu_project_normalize                     # noqa: F401
from .functional import conv_bn_relu_project_normalize                # noqa: F401
from .loss import (ContrastAuxCELoss, ContrastCELoss, MemContrastCELoss, PixelContrastLoss, SEG_LOSS_DICT,  # noqa: F401
                   get_seg_loss)
from .bank import MemoryBank, dequeue_and_enqueue, gather_packets      # noqa: F401
from .projection import ProjectionHead                                  # noqa: F401
from .trainer_hook import ContrastTrainerHook, LossStepTimer            # noqa: F401
from .graph_step import GraphedContrastStep                             # noqa: F401

__version__ = "0.1.0"
