"""Fused RMI seg loss (csrc/pcl_segce.cu, functional.upsample_rmi_loss, contrast.use_rmi) against the float64 restatement
in oracle/rmi_port.py: up-sampling geometries, class chunks, ignored labels, pooling ways and strides, radii, the
ill-conditioned regime, the full Cityscapes shape through both wrappers, bf16 logits, reproducibility and CUDA-graph
capture.  tests/test_emu_rmi.py runs the small cases on the emulated kernels."""
import os

import numpy as np
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi
from oracle.rmi_port import rmi_loss, rmi_loss_and_grad

DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _inputs(B, K, h, w, H, W, seed, ignored=0.15, scale=6.0):
    g = torch.Generator().manual_seed(seed)
    seg = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * scale          # logits in [-6, 6]: no max-pool ties
    target = torch.randint(0, K, (B, H, W), generator=g)
    drop = torch.rand(B, H, W, generator=g) < ignored
    kinds = torch.tensor([-1, 255, K, K + 3])
    target[drop] = kinds[torch.randint(0, 4, (int(drop.sum()),), generator=g)]
    return seg, target


def check_rmi(B, K, h, w, H, W, radius=3, way=0, stride=3, lambda_way=1, seed=0, target=None, seg=None, grad_out=0.7,
              loss_rel=1e-5, grad_rel=1e-4):
    s0, t0 = _inputs(B, K, h, w, H, W, seed)
    seg = s0 if seg is None else seg
    target = t0 if target is None else target
    kw = dict(num_classes=K, radius=radius, pool_way=way, pool_stride=stride, weight_lambda=0.5, lambda_way=lambda_way,
              loss_weight=1.3)
    ref, gref = rmi_loss_and_grad(seg, target, grad_out, **kw)
    _, g32 = rmi_loss_and_grad(seg, target, grad_out, front=torch.float32, **kw)
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    t_before = t.clone()
    loss = cs.upsample_rmi_loss(x, t, **kw)
    (loss * grad_out).backward()
    torch.cuda.synchronize()
    assert torch.equal(t, t_before), "target must not be modified"
    assert torch.isfinite(loss).item()
    assert abs(loss.item() - ref.item()) <= loss_rel * max(abs(ref.item()), 1e-3), (loss.item(), ref.item())
    assert_grad_close(x.grad, gref, g32, grad_rel)
    return loss, x.grad


def assert_grad_close(g, gref, g32, grad_rel=1e-4):
    """max |g - gref| within grad_rel of max |gref|, or within 4x the reference's own spread (its fp32 front end vs a
    float64 one, g32 vs gref): where P is nearly singular (smooth probabilities, few pixels per class) the fp32 rounding
    of the pooled probabilities reaches the gradient through P^-1, in the reference as in the engine."""
    gref = gref.to(g.device)
    err = (g.double() - gref).abs().max().item()
    spread = (g32.to(g.device) - gref).abs().max().item()
    assert err <= max(grad_rel * gref.abs().max().item(), 4 * spread, 1e-15), (err, gref.abs().max().item(), spread)


# ---- geometries, classes, parameters ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,K,h,w,H,W", [(2, 19, 17, 23, 66, 90), (2, 19, 32, 64, 128, 256), (2, 19, 40, 52, 40, 52),
                                         (2, 59, 17, 23, 66, 90), (1, 171, 33, 41, 130, 161)])
def test_rmi_geometries_and_class_chunks(B, K, h, w, H, W):
    # 171 classes on a label grid of 130 x 161: ~120 pixels per class keep the solves well conditioned (on 50 x 61 the
    # reference's own fp32 front end moves the gradient by 1.4e-3 of its maximum)
    check_rmi(B, K, h, w, H, W, seed=K + h)


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1, 2, 3, 4])
@pytest.mark.parametrize("way", [0, 1])
@pytest.mark.parametrize("stride", [1, 2, 3, 4])
def test_rmi_radius_pool_way_stride(radius, way, stride):
    check_rmi(2, 5, 11, 13, 43, 50, radius=radius, way=way, stride=stride, lambda_way=stride % 2, seed=radius * 10 + stride)


@pytest.mark.gpu
def test_rmi_label_edge_cases():
    B, K, h, w, H, W = 3, 7, 9, 11, 35, 41
    seg, target = _inputs(B, K, h, w, H, W, seed=3)
    target[0] = 2                                       # one class only
    target[1][target[1] == 4] = 0                       # class 4 absent from image 1
    check_rmi(B, K, h, w, H, W, seg=seg, target=target)


@pytest.mark.gpu
def test_rmi_every_pixel_ignored():
    B, K, h, w, H, W = 2, 5, 8, 9, 30, 33
    seg, _ = _inputs(B, K, h, w, H, W, seed=4)
    target = torch.full((B, H, W), 255, dtype=torch.int64)
    target[1] = -1
    x = seg.to(DEV).requires_grad_(True)
    loss = cs.upsample_rmi_loss(x, target.to(DEV), num_classes=K)
    loss.backward()
    ref = rmi_loss(seg, target, num_classes=K)
    assert torch.isfinite(loss).item()
    assert abs(loss.item() - ref.item()) <= 1e-5 * max(abs(ref.item()), 1e-3)
    assert torch.count_nonzero(x.grad).item() == 0


@pytest.mark.gpu
def test_rmi_ill_conditioned_within_the_reference_spread():
    """Strongly predictive logits: the 9x9 solves are ill-conditioned.  The engine's error is bounded by the spread of
    the oracle itself between the reference's fp32 front end and a float64 one."""
    B, K, h, w, H, W = 2, 6, 16, 20, 64, 80
    g = torch.Generator().manual_seed(9)
    target = torch.randint(0, K, (B, h, w), generator=g)
    target = torch.nn.functional.interpolate(target[:, None].float(), size=(H, W), mode="nearest")[:, 0].long()
    seg = torch.nn.functional.one_hot(target[:, ::4, ::4][:, :h, :w], K).permute(0, 3, 1, 2).double() * 24 - 12
    seg = (seg + 0.1 * torch.randn(seg.shape, generator=g, dtype=torch.float64)).float()
    kw = dict(num_classes=K)
    ref64 = rmi_loss(seg, target, **kw).item()
    ref32 = rmi_loss(seg, target, front=torch.float32, **kw).item()
    got = cs.upsample_rmi_loss(seg.to(DEV), target.to(DEV), **kw).item()
    assert abs(got - ref64) <= 4 * abs(ref32 - ref64) + 1e-6, (got, ref64, ref32)


@pytest.mark.gpu
def test_rmi_refusals():
    seg, target = _inputs(1, 3, 8, 8, 20, 20, seed=5)
    x, t = seg.to(DEV), target.to(DEV)
    with pytest.raises(_abi.PclError):
        cs.upsample_rmi_loss(x, t, num_classes=3, radius=5)
    with pytest.raises(_abi.PclError):
        cs.upsample_rmi_loss(x, t, num_classes=3, pool_way=2)
    with pytest.raises(_abi.PclError):
        cs.upsample_rmi_loss(x, t[:, :6, :6].contiguous(), num_classes=3)         # down-sampling
    with pytest.raises(_abi.PclError):
        cs.upsample_rmi_loss(x, t[:, :4, :4].contiguous() * 0, num_classes=3, pool_stride=4)   # pooled map 2 x 2 < r


# ---- full Cityscapes shape ----------------------------------------------------------------------------
def _rmi_config(with_memory=False, lambda_way=1):
    d = cs.cityscapes_contrast_config(with_memory=with_memory)
    d["contrast"]["use_rmi"] = True
    d["loss"]["params"].update(use_sigmoid=True, num_classes=19, rmi_radius=3, rmi_pool_way=0, rmi_pool_size=3,
                               rmi_pool_stride=3, loss_weight_lambda=0.5, loss_weight=1.0, lambda_way=lambda_way)
    d["network"]["loss_weights"] = {"seg_loss": 1.0, "aux_loss": 0.4}
    return d


@pytest.mark.gpu
def test_rmi_full_cityscapes_shape():
    B, K, h, w, H, W = 8, 19, 128, 256, 512, 1024
    seg, target = _inputs(B, K, h, w, H, W, seed=11)
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    # float64 oracle on the device
    ref, gref = rmi_loss_and_grad(x.detach(), t, 1.0, num_classes=K)
    _, g32 = rmi_loss_and_grad(x.detach(), t, 1.0, num_classes=K, front=torch.float32)
    loss = cs.upsample_rmi_loss(x, t, num_classes=K)
    loss.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    assert_grad_close(x.grad, gref, g32)
    del gref, g32
    # bit-identical forward over two calls
    again = cs.upsample_rmi_loss(x.detach(), t, num_classes=K)
    assert torch.equal(loss.detach(), again)
    # unfused: F.interpolate first, then the identity geometry
    up = torch.nn.functional.interpolate(x.detach(), size=(H, W), mode="bilinear", align_corners=True)
    unf = cs.upsample_rmi_loss(up, t, num_classes=K)
    assert abs(unf.item() - loss.item()) <= 1e-6 * abs(loss.item())
    # bf16 seg == the fp32 call on the converted tensor
    xb = x.detach().bfloat16().requires_grad_(True)
    lb = cs.upsample_rmi_loss(xb, t, num_classes=K)
    lb.backward()
    xf = xb.detach().float().requires_grad_(True)
    lf = cs.upsample_rmi_loss(xf, t, num_classes=K)
    lf.backward()
    assert torch.equal(lb.detach(), lf.detach())
    assert xb.grad.dtype == torch.bfloat16 and xb.grad.shape == xb.shape
    assert (xb.grad.float() - xf.grad.bfloat16().float()).abs().max().item() <= 1e-2 * xf.grad.abs().max().item()


@pytest.mark.gpu
def test_rmi_cuda_graph_replays_the_eager_loss():
    B, K, h, w, H, W = 8, 19, 128, 256, 512, 1024
    seg, target = _inputs(B, K, h, w, H, W, seed=12)
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    eager = cs.upsample_rmi_loss(x, t, num_classes=K)
    eager.backward()
    eager_loss, eager_grad = eager.detach().clone(), x.grad.clone()
    del eager
    xg = seg.to(DEV).requires_grad_(True)          # a leaf first used on the side stream (its AccumulateGrad stream)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xg.grad = None
            cs.upsample_rmi_loss(xg, t, num_classes=K).backward()
    torch.cuda.current_stream().wait_stream(s)
    xg.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = cs.upsample_rmi_loss(xg, t, num_classes=K)
        out.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.detach(), eager_loss)
    assert (xg.grad - eager_grad).abs().max().item() <= 1e-6 * eager_grad.abs().max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("mem", [False, True])
def test_rmi_wrappers_full_shape_fused_and_unfused(mem):
    B, K, h, w, H, W = 8, 19, 128, 256, 512, 1024
    seg, target = _inputs(B, K, h, w, H, W, seed=13 + mem)
    target[(target < 0) | (target >= K)] = -1           # the reference's contrast configs: ignore label -1
    seg_aux = seg * 0.5 + 0.3
    embed = torch.nn.functional.normalize(torch.randn(B, 256, h, w, generator=torch.Generator().manual_seed(2)), dim=1)
    losses = {}
    for fused in (True, False):
        d = _rmi_config(with_memory=mem)
        d["contrast"]["fused_seg_ce"] = fused
        cfg = cs.Configer(d)
        crit = cs.MemContrastCELoss(cfg) if mem else cs.ContrastAuxCELoss(cfg)
        preds = {"seg": seg.to(DEV), "embed": embed.to(DEV)}
        if not mem:
            preds["seg_aux"] = seg_aux.to(DEV)
        losses[fused] = crit(preds, target.to(DEV), with_embed=False).item()
    assert abs(losses[True] - losses[False]) <= 1e-6 * abs(losses[False]) + 1e-6
    rmi = rmi_loss(seg.to(DEV), target.to(DEV), num_classes=K).item()
    if mem:
        expect = rmi
    else:
        ce = torch.nn.functional.cross_entropy(
            torch.nn.functional.interpolate(seg_aux.to(DEV).double(), size=(H, W), mode="bilinear", align_corners=True),
            target.to(DEV), ignore_index=-1).item()
        expect = rmi + 0.4 * ce
    assert abs(losses[True] - expect) <= 1e-5 * abs(expect)


# ---- the wrappers against the reference's goldens ---------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rmi_wrapper_aux", "rmi_wrapper_mem"])
def test_rmi_wrapper_goldens(name):
    from test_oracle_rmi import golden_wrapper_loss
    got, ref = golden_wrapper_loss(name, DEV)
    assert abs(got - ref) <= 1e-4 * abs(ref), (got, ref)
