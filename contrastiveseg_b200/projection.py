"""ProjectionHead with the engine's L2-normalise (lib/models/modules/projection.py:8-24).

By default the 1x1 convolutions / BatchNorm stay cuDNN / PyTorch and only the final F.normalize(p=2, dim=1) runs on
the engine kernel.  ``fused=True`` runs the last Conv2d (Cin -> 256) and the normalise as one wgmma GEMM with the
normalise in its epilogue (functional.project_normalize, bf16 operands, fp32 accumulate); the 720 -> 720 conv, BN and
ReLU of ``convmlp`` still run in torch.  The fused head takes a float32 or bfloat16 input; the dtype of the tensor
reaching the last conv decides the output's (under ``torch.autocast(dtype=torch.bfloat16)`` the ``convmlp`` prefix
hands it bf16, so zn is bf16).  The module tree and state_dict keys are the same either way.
``fuse_bn_relu=True`` (with ``fused=True``, ``convmlp`` only) runs everything after the 720 -> 720 conv on the engine:
its output y goes through functional.bn_relu_project_normalize, which applies the BatchNorm (batch statistics in
training, running ones in eval; SyncBatchNorm reduces over its process group) and the ReLU inside the fused GEMM.
``fuse_conv1=True`` (with ``fuse_bn_relu=True``) runs the 720 -> 720 conv on the engine too
(functional.conv_bn_relu_project_normalize): a bf16 wgmma GEMM that also sums the BatchNorm statistics of its output,
so the whole head is one autograd node with no cuDNN call.  Under ``torch.autocast(dtype=torch.bfloat16)`` a float32
input is cast to bfloat16 as autocast's conv would cast it (y and zn are then bf16); fp16 autocast is refused.
``sparse_grad=True`` (with ``fuse_bn_relu=True``) lets an engine contrast loss that reads zn hand the head's backward
its anchor columns instead of a dense gradient: the last conv's gradients and the BN backward's sums run over those
columns, and zn itself receives a zero placeholder (INTEGRATION §1).
``normalize=False`` returns the raw projection for the fused loss path (PixelContrastLoss(..., normalize=True) then
normalises only the sampled columns)."""
from __future__ import annotations

import torch
import torch.nn as nn

from . import functional as _fn
from ._abi import PclError
from .functional import bn_relu_project_normalize, conv_bn_relu_project_normalize, l2_normalize, project_normalize


def _autocast_input(x):
    """x as autocast's conv would take it: cast to bfloat16 under a bfloat16 autocast of x's device type; any other
    autocast dtype is refused (the engine's activations are fp32 or bf16)."""
    if not torch.is_autocast_enabled(x.device.type):
        return x
    dtype = torch.get_autocast_dtype(x.device.type)
    if dtype != torch.bfloat16:
        raise PclError(f"ProjectionHead(fuse_conv1=True) under autocast needs dtype=torch.bfloat16, got {dtype}")
    return x.to(torch.bfloat16)


class ProjectionHead(nn.Module):
    def __init__(self, dim_in, proj_dim=256, proj="convmlp", bn_type="torchsyncbn", normalize=True, fused=False,
                 fuse_bn_relu=False, fuse_conv1=False, sparse_grad=False):
        super().__init__()
        if sparse_grad and not fuse_bn_relu:
            # without the BN inside the node the input gradient would be a dense zero tensor of Cin channels
            raise PclError("ProjectionHead(sparse_grad=True) needs fused=True, fuse_bn_relu=True and proj='convmlp'")
        if fuse_conv1 and not fuse_bn_relu:
            raise PclError("ProjectionHead(fuse_conv1=True) needs fuse_bn_relu=True")
        if fuse_bn_relu and not fused:
            raise PclError("ProjectionHead(fuse_bn_relu=True) needs fused=True")
        if fuse_bn_relu and proj != "convmlp":
            raise PclError(f"ProjectionHead(fuse_bn_relu=True) needs proj='convmlp', got {proj!r}")
        if fused and proj_dim != _fn.PROJ_DIM:
            raise PclError(f"ProjectionHead(fused=True) needs proj_dim == {_fn.PROJ_DIM}, got {proj_dim}")
        if fused and not normalize:
            raise PclError("ProjectionHead(fused=True) fuses the normalise: normalize=False is not supported")
        if proj == "linear":
            self.proj = nn.Conv2d(dim_in, proj_dim, kernel_size=1)
        elif proj == "convmlp":
            bn = nn.SyncBatchNorm(dim_in) if bn_type == "torchsyncbn" else nn.BatchNorm2d(dim_in)
            self.proj = nn.Sequential(nn.Conv2d(dim_in, dim_in, kernel_size=1), nn.Sequential(bn, nn.ReLU()),
                                      nn.Conv2d(dim_in, proj_dim, kernel_size=1))
        else:
            raise ValueError(f"unknown projection type {proj!r}")
        self.normalize = normalize
        self.fused = fused
        self.fuse_bn_relu = fuse_bn_relu
        self.fuse_conv1 = fuse_conv1
        self.sparse_grad = sparse_grad

    def forward(self, x, out=None):
        """out (fuse_bn_relu heads): a (B, proj_dim, H, W) tensor of zn's dtype that zn is written into, e.g. the static
        embed of a GraphedContrastStep (bn_relu_project_normalize)."""
        if out is not None and not self.fuse_bn_relu:
            raise PclError("ProjectionHead.forward(out=...) needs fuse_bn_relu=True (the fused BN heads write zn in place)")
        if self.fused:
            _fn._require_cuda(x, "x")
            _fn.proj_dtype_code(x.dtype, "ProjectionHead(fused=True)")
            if self.fuse_conv1:
                conv1, conv2 = self.proj[0], self.proj[2]
                return conv_bn_relu_project_normalize(_autocast_input(x), conv1.weight, conv1.bias, self.proj[1][0],
                                                      conv2.weight, conv2.bias, sparse_grad=self.sparse_grad, out=out)
            if self.fuse_bn_relu:
                return bn_relu_project_normalize(self.proj[0](x), self.proj[1][0], self.proj[2].weight,
                                                 self.proj[2].bias, sparse_grad=self.sparse_grad, out=out)
            if isinstance(self.proj, nn.Conv2d):
                last, y = self.proj, x
            else:
                last, y = self.proj[-1], self.proj[:-1](x)
            # the tensor reaching the fused conv decides zn's dtype (bf16 under autocast for convmlp), and
            # project_normalize refuses any other than float32 / bfloat16
            return project_normalize(y, last.weight, last.bias)
        y = self.proj(x)
        return l2_normalize(y) if self.normalize else y
