"""Fused Lovasz-softmax seg loss (csrc/pcl_segce.cu, third part; functional.upsample_lovasz_softmax, FSCELOVASZLoss)
against the float64 restatement in oracle/lovasz_port.py: up-sampling geometries, class counts up to 171, sort edge
cases, exact ties, saturated logits, ignored and out-of-range labels, half inputs, reproducibility, CUDA-graph capture
and the full Cityscapes shape through MemContrastCELoss.  tests/test_emu_lovasz.py runs the small cases on the emulated kernels.

Gradient bounds: relative Frobenius norm over all elements, and max-abs over the low-resolution logits whose bilinear
footprint holds no near-tie pixel (a pixel whose float64 error lies within a few fp32 ulps of the error of an
opposite-fg pixel of the same class: fp32 may order the pair differently, which moves its gradient by O(1/U))."""
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi
from oracle.lovasz_port import footprint_mask, lovasz_loss, lovasz_loss_and_grad

DEV = "cuda"
NEAR_TIE_ULPS = 64
LOSS_REL = 1e-5
# 3x the worst value measured on an H100 80GB HBM3 (700 W): 5.5e-5 and 3.3e-5, both on a 1 x 2047 label row (DESIGN, row f6)
GRAD_FRO = 1.7e-4          # relative Frobenius norm of dseg - dseg_ref
GRAD_MAX = 1e-4            # max |dseg - dseg_ref| off the near-tie footprints, relative to max |dseg_ref|


def _inputs(B, K, h, w, H, W, seed, ignored=0.15, scale=4.0, ignore_index=-1):
    g = torch.Generator().manual_seed(seed)
    seg = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * scale
    target = torch.randint(0, K, (B, H, W), generator=g)
    drop = torch.rand(B, H, W, generator=g) < ignored
    target[drop] = ignore_index
    return seg, target


def check_lovasz(seg, target, ignore_index=-1, grad_out=0.7, loss_rel=LOSS_REL, grad_fro=GRAD_FRO, grad_max=GRAD_MAX,
                 front=torch.float64):
    B, K, h, w = seg.shape
    ref, gref, near = lovasz_loss_and_grad(seg, target, grad_out, ignore_index=ignore_index, near_tie_ulps=NEAR_TIE_ULPS,
                                           front=front)
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    t_before = t.clone()
    loss = cs.upsample_lovasz_softmax(x, t, ignore_index=ignore_index)
    (loss * grad_out).backward()
    torch.cuda.synchronize()
    assert torch.equal(t, t_before), "target must not be modified"
    assert abs(loss.item() - ref.item()) <= loss_rel * max(abs(ref.item()), 1e-6), (loss.item(), ref.item())
    g, gref = x.grad.double().cpu(), gref.cpu()
    scale = gref.abs().max().item()
    if scale == 0.0:
        assert torch.count_nonzero(g).item() == 0
        return loss, x.grad, {"fro": 0.0, "max": 0.0}
    fro = ((g - gref).norm() / gref.norm()).item()
    keep = ~footprint_mask(near.cpu(), h, w)
    diff = (g - gref).abs().amax(dim=1)                       # (B, h, w): worst class plane
    mx = (diff[keep].max().item() if keep.any() else 0.0) / scale
    print(f"lovasz {tuple(seg.shape)} -> {tuple(target.shape[1:])}: grad fro {fro:.3e} max {mx:.3e} "
          f"(near-tie footprints {int((~keep).sum())} of {keep.numel()})")
    assert fro <= grad_fro, (fro, grad_fro)
    assert mx <= grad_max, (mx, grad_max, int(keep.sum()), keep.numel())
    return loss, x.grad, {"fro": fro, "max": mx}


# ---- geometries and class counts -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B,K,h,w,H,W", [(2, 19, 17, 23, 66, 90), (2, 19, 32, 64, 128, 256), (2, 19, 40, 52, 40, 52),
                                         (2, 59, 17, 23, 66, 90), (1, 171, 33, 41, 130, 161), (2, 7, 13, 9, 45, 31)])
def test_lovasz_geometries_and_classes(B, K, h, w, H, W):
    seg, target = _inputs(B, K, h, w, H, W, seed=K + h)
    check_lovasz(seg, target)


# ---- sort edge cases ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_lovasz_single_pixel_class_and_absent_class():
    B, K, h, w, H, W = 2, 6, 9, 11, 36, 44
    seg, target = _inputs(B, K, h, w, H, W, seed=21)
    target[target == 3] = 0
    target[target == 5] = 1
    target[1, 7, 9] = 5                                      # class 5: one pixel; class 3 absent
    check_lovasz(seg, target)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2047, 2048, 2049, 4097])
def test_lovasz_counts_around_the_sort_tile(n):
    # label pixels N = n (one image, 1 x n row) around the sort's 2048-key tile
    seg, target = _inputs(1, 4, 1, max(2, n // 8), 1, n, seed=n, ignored=0.1)
    check_lovasz(seg, target)


# ---- exact ties ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_lovasz_exact_ties_follow_the_stable_order():
    """Identity geometry, every pixel's logit vector one of 3 patterns: fp32 and float64 tie in the same places, so the
    gradient must equal the oracle's stable order (ties by ascending pixel index)."""
    B, K, H, W = 2, 5, 24, 40
    g = torch.Generator().manual_seed(7)
    pats = (torch.rand(3, K, generator=g) * 4 - 2)
    which = torch.randint(0, 3, (B, H, W), generator=g)
    seg = pats[which].permute(0, 3, 1, 2).contiguous()
    target = torch.randint(0, K, (B, H, W), generator=g)
    ref, gref = lovasz_loss_and_grad(seg, target, 1.0)
    x = seg.to(DEV).requires_grad_(True)
    loss = cs.upsample_lovasz_softmax(x, target.to(DEV))
    loss.backward()
    assert abs(loss.item() - ref.item()) <= LOSS_REL * abs(ref.item())
    err = (x.grad.double().cpu() - gref).abs().max().item()
    assert err <= 1e-5 * gref.abs().max().item(), (err, gref.abs().max().item())


# ---- saturation, ignored pixels, labels, weights --------------------------------------------------------------
@pytest.mark.gpu
def test_lovasz_saturated_logits():
    """Logits of +-40: p is exactly 0 or 1 in fp32, where |fg - p| has a zero gradient, as in the reference's fp32
    front end (float64 does not saturate, and its gradient there differs by 3e-2 in Frobenius norm).  So the oracle runs
    the up-sampling and softmax in fp32 here; bounds at 3x the worst measured on the H100."""
    B, K, h, w, H, W = 2, 4, 8, 10, 32, 40
    seg, target = _inputs(B, K, h, w, H, W, seed=31)
    seg = torch.where(seg > 0, torch.full_like(seg, 40.0), torch.full_like(seg, -40.0))
    seg[:, :, :2] = seg[:, :, :2] * 0.05                    # a band of unsaturated logits
    check_lovasz(seg, target, front=torch.float32, grad_fro=1.2e-4, grad_max=1.4e-5)


@pytest.mark.gpu
def test_lovasz_every_pixel_ignored():
    B, K, h, w, H, W = 2, 5, 8, 9, 30, 33
    seg, _ = _inputs(B, K, h, w, H, W, seed=4)
    target = torch.full((B, H, W), -1, dtype=torch.int64)
    target[1, :3] = 77                                       # out of range: ignored as well
    x = seg.to(DEV).requires_grad_(True)
    loss = cs.upsample_lovasz_softmax(x, target.to(DEV))
    loss.backward()
    assert loss.item() == 0.0
    assert torch.count_nonzero(x.grad).item() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("ignore_index", [-1, 255])
def test_lovasz_ignore_index_and_out_of_range_labels(ignore_index):
    B, K, h, w, H, W = 2, 6, 10, 12, 40, 48
    seg, target = _inputs(B, K, h, w, H, W, seed=41, ignore_index=ignore_index)
    g = torch.Generator().manual_seed(42)
    odd = torch.rand(B, H, W, generator=g) < 0.05
    target[odd] = torch.tensor([-7, K, K + 9, 300])[torch.randint(0, 4, (int(odd.sum()),), generator=g)]
    check_lovasz(seg, target, ignore_index=ignore_index)


def _lovasz_config(ignore_index=-1, ce_weight=None, with_memory=True):
    d = cs.cityscapes_contrast_config(with_memory=with_memory)
    d["contrast"]["use_lovasz"] = True
    d["loss"]["params"]["ce_ignore_index"] = ignore_index
    if ce_weight is not None:
        d["loss"]["params"]["ce_weight"] = ce_weight
    return d


@pytest.mark.gpu
def test_fscelovasz_module_with_ce_weight():
    B, K, H, W = 2, 19, 48, 64
    seg, target = _inputs(B, K, H, W, H, W, seed=51)
    wts = [0.5 + 0.05 * i for i in range(K)]
    crit = cs.FSCELOVASZLoss(cs.Configer(_lovasz_config(ce_weight=wts)))
    crit.ce_loss.to(DEV)
    x = seg.to(DEV).requires_grad_(True)
    loss = crit(x, target.to(DEV))
    loss.backward()
    ce = torch.nn.functional.cross_entropy(seg.double(), target, weight=torch.tensor(wts, dtype=torch.float64),
                                           ignore_index=-1)
    expect = ce.item() + lovasz_loss(seg, target).item()
    assert abs(loss.item() - expect) <= 1e-5 * abs(expect)
    # list input: the weighted CE sum, no Lovasz term
    lst = crit([x.detach(), x.detach() * 0.5], target.to(DEV), weights=[1.0, 0.25])
    ce2 = torch.nn.functional.cross_entropy(seg.double() * 0.5, target, weight=torch.tensor(wts, dtype=torch.float64),
                                            ignore_index=-1)
    assert abs(lst.item() - (ce.item() + 0.25 * ce2.item())) <= 1e-5 * abs(lst.item())


# ---- half inputs ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_lovasz_half_inputs_equal_the_fp32_call(dtype):
    seg, target = _inputs(2, 19, 17, 23, 66, 90, seed=61)
    t = target.to(DEV)
    xh = seg.to(DEV, dtype).requires_grad_(True)
    lh = cs.upsample_lovasz_softmax(xh, t)
    lh.backward()
    xf = xh.detach().float().requires_grad_(True)
    lf = cs.upsample_lovasz_softmax(xf, t)
    lf.backward()
    assert torch.equal(lh.detach(), lf.detach())
    assert xh.grad.dtype == dtype and torch.equal(xh.grad, xf.grad.to(dtype))


# ---- determinism and capture -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_lovasz_bit_reproducible_and_graph_replays_eager():
    B, K, h, w, H, W = 2, 19, 32, 64, 128, 256
    seg, target = _inputs(B, K, h, w, H, W, seed=71)
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    eager = cs.upsample_lovasz_softmax(x, t)
    eager.backward()
    again = cs.upsample_lovasz_softmax(x.detach(), t)
    assert torch.equal(eager.detach(), again)
    eager_loss, eager_grad = eager.detach().clone(), x.grad.clone()
    xg = seg.to(DEV).requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xg.grad = None
            cs.upsample_lovasz_softmax(xg, t).backward()
    torch.cuda.current_stream().wait_stream(s)
    xg.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = cs.upsample_lovasz_softmax(xg, t)
        out.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.detach(), eager_loss)
    assert (xg.grad - eager_grad).abs().max().item() <= 1e-6 * eager_grad.abs().max().item()


@pytest.mark.gpu
def test_lovasz_refusals():
    seg, target = _inputs(1, 3, 8, 8, 20, 20, seed=5)
    with pytest.raises(_abi.PclError):
        cs.upsample_lovasz_softmax(seg.to(DEV), target[:, :6, :6].to(DEV))            # down-sampling
    with pytest.raises(_abi.PclError):
        cs.upsample_lovasz_softmax(torch.zeros(1, 257, 4, 4, device=DEV), torch.zeros(1, 4, 4, dtype=torch.int64,
                                                                                       device=DEV))


# ---- full Cityscapes shape through the memory wrapper ------------------------------------------------------------
@pytest.mark.gpu
def test_lovasz_full_shape_through_mem_contrast_wrapper():
    B, K, h, w, H, W = 8, 19, 128, 256, 512, 1024
    seg, target = _inputs(B, K, h, w, H, W, seed=81)
    cfg = cs.Configer(_lovasz_config())
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    embed = torch.nn.functional.normalize(torch.randn(B, 256, h, w, device=DEV), dim=1).requires_grad_(True)
    crit = cs.MemContrastCELoss(cfg, seg_criterion=cs.FSCELOVASZLoss(cfg))
    mb = cs.MemoryBank(K, 32, 256).to(DEV)
    preds = {"seg": x, "embed": embed, "segment_queue": mb.segment_queue, "pixel_queue": mb.pixel_queue}
    loss = crit(preds, t, with_embed=False)
    loss.backward()
    xd = x.detach()
    ref, gref, near = lovasz_loss_and_grad(xd, t, 1.0, near_tie_ulps=NEAR_TIE_ULPS)
    xc = xd.double().requires_grad_(True)
    ce = torch.nn.functional.cross_entropy(
        torch.nn.functional.interpolate(xc, size=(H, W), mode="bilinear", align_corners=True), t, ignore_index=-1)
    ce.backward()
    expect = ce.item() + ref.item()
    assert abs(loss.item() - expect) <= LOSS_REL * abs(expect), (loss.item(), expect)
    gtot = gref + xc.grad
    fro = ((x.grad.double() - gtot).norm() / gtot.norm()).item()
    keep = ~footprint_mask(near, h, w)
    mx = (x.grad.double() - gtot).abs().amax(dim=1)[keep].max().item() / gtot.abs().max().item()
    print(f"lovasz full shape: grad fro {fro:.3e} max {mx:.3e} (near-tie footprints {int((~keep).sum())})")
    assert fro <= GRAD_FRO, fro
    assert mx <= GRAD_MAX, mx
