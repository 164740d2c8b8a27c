"""ProjectionHead with the engine's L2-normalise (lib/models/modules/projection.py:8-24).

By default the 1x1 convolutions / BatchNorm stay cuDNN / PyTorch and only the final F.normalize(p=2, dim=1) runs on
the engine kernel.  ``fused=True`` runs the last Conv2d (Cin -> 256) and the normalise as one wgmma GEMM with the
normalise in its epilogue (functional.project_normalize, bf16 operands, fp32 accumulate); the 720 -> 720 conv, BN and
ReLU of ``convmlp`` still run in torch.  The fused head takes a float32 or bfloat16 input; the dtype of the tensor
reaching the last conv decides the output's (under ``torch.autocast(dtype=torch.bfloat16)`` the ``convmlp`` prefix
hands it bf16, so zn is bf16).  The module tree and state_dict keys are the same either way.
``normalize=False`` returns the raw projection for the fused loss path (PixelContrastLoss(..., normalize=True) then
normalises only the sampled columns)."""
from __future__ import annotations

import torch.nn as nn

from . import functional as _fn
from ._abi import PclError
from .functional import l2_normalize, project_normalize


class ProjectionHead(nn.Module):
    def __init__(self, dim_in, proj_dim=256, proj="convmlp", bn_type="torchsyncbn", normalize=True, fused=False):
        super().__init__()
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

    def forward(self, x):
        if self.fused:
            _fn._require_cuda(x, "x")
            _fn.proj_dtype_code(x.dtype, "ProjectionHead(fused=True)")
            if isinstance(self.proj, nn.Conv2d):
                last, y = self.proj, x
            else:
                last, y = self.proj[-1], self.proj[:-1](x)
            # the tensor reaching the fused conv decides zn's dtype: bf16 under autocast for convmlp
            _fn.proj_dtype_code(y.dtype, "ProjectionHead(fused=True)")
            return project_normalize(y, last.weight, last.bias)
        y = self.proj(x)
        return l2_normalize(y) if self.normalize else y
