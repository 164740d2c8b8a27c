"""The fused step's gradient scatter writes whole 32-byte sectors (csrc/pcl_select.cu, k_scatter_reduce): with nearly
every pixel sampled, most sectors hold several anchors, and each anchor's gradient must still land, with +0 everywhere
else, whatever the sign of the scale."""
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import functional as Fn
from contrastiveseg_b200.synth import make_contrast_batch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda:0"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_dense_sampling_shares_sectors_and_every_anchor_lands(dtype):
    B, D, h, w, K = 2, 256, 16, 16, 2
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=8, seed=41)
    embed, tgt, seg = data["embed"].to(DEV).to(dtype), data["target"].to(DEV), data["seg"].to(DEV)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=1024, max_views=64, seed=9,
                              precision="bf16", num_classes=K)
    step = cs.GraphedContrastStep(embed, tgt, seg=seg, options=opts, grad_scale=-0.5)
    assert step.fused
    loss, grad = step.replay()
    torch.cuda.synchronize()
    A = int(step.ws.plan[2].item())
    meta = step.ws.anchor_meta.view(4, 1024)[:, :A].long()
    pix, img = meta[0], meta[1]
    E = 32 // grad.element_size()
    sectors = torch.unique(img * (h * w) + pix // E)
    assert A >= 256 and sectors.numel() < A // 2             # most sectors hold several anchors
    sampled = torch.zeros(B, h * w, dtype=torch.bool, device=DEV)
    sampled[img, pix] = True
    g = grad.float().permute(0, 2, 3, 1).reshape(B, h * w, D)
    assert bool((g[sampled] != 0).any(dim=1).all())            # every anchor's row landed
    assert bool((g[~sampled] == 0).all())
    assert not bool(torch.signbit(g[~sampled]).any())           # +0, not -0 from a negative scale
    # the same gradient as the eager autograd path (its own scatter), up to the tensor path's summation order
    Fn._step_counter[0] = 0
    e = embed.clone().requires_grad_(True)
    cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts).backward()
    torch.cuda.synchronize()
    ref = -0.5 * e.grad.float()
    assert (ref - grad.float()).abs().max().item() <= 2e-2 * ref.abs().max().item()
