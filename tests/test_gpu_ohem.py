"""Fused OHEM cross-entropy (csrc/pcl_segce.cu, fourth part; functional.upsample_ohem_cross_entropy, FSOhemCELoss,
FSAuxOhemCELoss) against the float64 restatement in oracle/ohem_port.py: up-sampling geometries, class counts up to 171,
both branches (fp32(thresh) decides, or the exact select of the kth value runs), exact ties, min_kept >= n, n = 0 and
n = 1, weights and 'sum', half inputs, reproducibility, CUDA-graph capture and the full Cityscapes shape through
ContrastCELoss and ContrastAuxCELoss.  tests/test_emu_ohem.py runs the small cases on the emulated kernels.

Inputs are built with a gap around the threshold (oracle/ohem_port.gap_labels ignores the pixels whose float64 p_t lies
within 64 fp32 ulps of it), so the engine must select exactly the oracle's pixels; the loss and gradient bounds then
only cover fp32 rounding."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi
from contrastiveseg_b200.functional import ohem_selection
from oracle.lovasz_port import footprint_mask
from oracle.ohem_port import gap_labels, ohem_loss, ohem_loss_and_grad

DEV = "cuda"
NEAR_ULPS = 64
# 3x the worst value measured on an H100 80GB HBM3 (700 W) over this file's cases: 6.9e-8 and 1.26e-6 (DESIGN, row f7)
LOSS_REL = 2.1e-7          # |loss - loss_ref| / |loss_ref|, float64 oracle on the same selection
GRAD_MAX = 3.8e-6          # max |dseg - dseg_ref| / max |dseg_ref|
# full S1 shape against the oracle's fp32 op sequence
FULL_LOSS_REL = LOSS_REL    # measured 0 (bit-equal) at both wrappers


def _inputs(B, K, h, w, H, W, seed, ignored=0.15, scale=4.0, ignore_index=-1):
    g = torch.Generator().manual_seed(seed)
    seg = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * scale
    target = torch.randint(0, K, (B, H, W), generator=g)
    target[torch.rand(B, H, W, generator=g) < ignored] = ignore_index
    return seg, target


def branch_min_kept(seg, target, branch, thresh, ignore_index=-1):
    """A min_kept that makes `branch` happen: below count(p_t < thresh) for the threshold branch, above it (but below n)
    for the select branch."""
    d = ohem_loss(seg, target, ignore_index=ignore_index, thresh=thresh, details=True)
    valid = (target != ignore_index) & (target >= 0) & (target < seg.shape[1])
    below = int(((d["p"] < float(np.float32(thresh))) & valid).sum())
    if branch == "threshold":
        return max(1, below // 2)
    return below + max(1, (d["n"] - below) // 3)


def median_thresh(seg, target, ignore_index=-1):
    """The median p_t of the counted pixels (rounded to 4 digits): a thresh with room for both branches at any K."""
    d = ohem_loss(seg, target, ignore_index=ignore_index, details=True)
    valid = (target != ignore_index) & (target >= 0) & (target < seg.shape[1])
    return round(float(d["p"][valid].median()), 4)


def check_ohem(seg, target, weight=None, ignore_index=-1, thresh=0.7, min_kept=100, reduction="mean", grad_out=0.7,
               branch=None, gap=True):
    """Engine vs oracle on a gapped copy of target: the selected set exactly, the loss and the gradient within the
    bounds.  Returns the measured relative loss and gradient errors."""
    kw = dict(weight=weight, ignore_index=ignore_index, thresh=thresh, min_kept=min_kept, reduction=reduction)
    if gap:
        target = gap_labels(seg.to(DEV), target.to(DEV), near_ulps=NEAR_ULPS, **kw).cpu()
    x = seg.detach().to(DEV, copy=True).requires_grad_(True)
    t = target.to(DEV)
    t_before = t.clone()
    wd = None if weight is None else weight.to(DEV)
    d, gref = ohem_loss_and_grad(x.detach(), t, grad_out, near_ulps=NEAR_ULPS, **dict(kw, weight=wd))
    sel = ohem_selection(x.detach(), t, wd, ignore_index, thresh, min_kept, reduction)
    if branch is not None:
        assert sel["branch"] == branch, (sel["branch"], branch)
    assert sel["n"] == d["n"] and sel["count"] == d["count"], (sel["n"], d["n"], sel["count"], d["count"])
    assert torch.equal(sel["selected"], d["selected"]), int((sel["selected"] != d["selected"]).sum())
    loss = cs.upsample_ohem_cross_entropy(x, t, wd, ignore_index, thresh, min_kept, reduction)
    (loss * grad_out).backward()
    torch.cuda.synchronize()
    assert torch.equal(t, t_before), "target must not be modified"
    ref = d["loss"].item()
    if math.isnan(ref):
        assert math.isnan(loss.item())
        assert torch.count_nonzero(x.grad).item() == 0
        return {"loss": 0.0, "grad": 0.0, "branch": sel["branch"]}
    lerr = abs(loss.item() - ref) / max(abs(ref), 1e-30)
    assert lerr <= LOSS_REL or (ref == 0.0 and loss.item() == 0.0), (loss.item(), ref)
    scale = gref.abs().max().item()
    if scale == 0.0:
        assert torch.count_nonzero(x.grad).item() == 0
        return {"loss": lerr, "grad": 0.0, "branch": sel["branch"]}
    gerr = (x.grad.double() - gref).abs().max().item() / scale
    print(f"ohem {tuple(seg.shape)} -> {tuple(target.shape[1:])} {sel['branch']}: n {d['n']} selected {d['count']} "
          f"loss rel {lerr:.3e} grad max {gerr:.3e}")
    assert gerr <= GRAD_MAX, (gerr, GRAD_MAX)
    return {"loss": lerr, "grad": gerr, "branch": sel["branch"]}


# ---- geometries, class counts, both branches -------------------------------------------------------------------
GEOMS = [(2, 19, 40, 52, 40, 52), (2, 19, 17, 23, 68, 92), (1, 19, 97, 97, 769, 769), (2, 19, 13, 9, 45, 31),
         (2, 59, 17, 23, 66, 90), (1, 150, 33, 41, 130, 161), (1, 171, 33, 41, 130, 161)]


@pytest.mark.gpu
@pytest.mark.parametrize("branch", ["threshold", "select"])
@pytest.mark.parametrize("B,K,h,w,H,W", GEOMS)
def test_ohem_geometries_classes_and_branches(B, K, h, w, H, W, branch):
    seg, target = _inputs(B, K, h, w, H, W, seed=K + h)
    thresh = median_thresh(seg, target)
    mk = branch_min_kept(seg, target, branch, thresh)
    check_ohem(seg, target, thresh=thresh, min_kept=mk, branch=branch)


@pytest.mark.gpu
@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_weights_and_reductions(reduction):
    B, K, h, w, H, W = 2, 19, 17, 23, 66, 90
    seg, target = _inputs(B, K, h, w, H, W, seed=5)
    weight = torch.tensor([0.5 + 0.08 * i for i in range(K)])
    for branch in ("threshold", "select"):
        mk = branch_min_kept(seg, target, branch, 0.4)
        check_ohem(seg, target, weight=weight, thresh=0.4, min_kept=mk, reduction=reduction, branch=branch)


@pytest.mark.gpu
@pytest.mark.parametrize("ignore_index", [-1, 255])
def test_ohem_ignore_index_and_out_of_range_labels(ignore_index):
    B, K, h, w, H, W = 2, 6, 10, 12, 40, 48
    seg, target = _inputs(B, K, h, w, H, W, seed=41, ignore_index=ignore_index)
    g = torch.Generator().manual_seed(42)
    odd = torch.rand(B, H, W, generator=g) < 0.05
    target[odd] = torch.tensor([-7, K, K + 9, 300])[torch.randint(0, 4, (int(odd.sum()),), generator=g)]
    check_ohem(seg, target, ignore_index=ignore_index, thresh=0.5, min_kept=300)


@pytest.mark.gpu
def test_ohem_min_kept_at_least_n():
    seg, target = _inputs(2, 7, 9, 11, 36, 44, seed=8)
    r = check_ohem(seg, target, thresh=0.5, min_kept=10 ** 9, branch="select")
    d = ohem_loss(seg, gap_labels(seg, target, thresh=0.5, min_kept=10 ** 9), thresh=0.5, min_kept=10 ** 9, details=True)
    assert d["count"] == d["n"] - 1 and r["branch"] == "select"


# ---- exact ties ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_exact_ties_are_in_or_out_together(reduction):
    """Identity geometry, block-constant logits quantised to 1/8, a few patterns: each (pattern, label) group shares one
    p_t in fp32 and in float64.  min_kept lands inside a group, so kth is that group's p_t and the strict comparison
    leaves the whole group out."""
    B, K, H, W = 2, 5, 24, 40
    g = torch.Generator().manual_seed(7)
    pats = torch.round((torch.rand(4, K, generator=g) * 4 - 2) * 8) / 8
    which = torch.randint(0, 4, (B, H // 4, W // 4), generator=g).repeat_interleave(4, 1).repeat_interleave(4, 2)
    seg = pats[which].permute(0, 3, 1, 2).contiguous()
    target = torch.randint(0, K, (B, H // 4, W // 4), generator=g).repeat_interleave(4, 1).repeat_interleave(4, 2)
    d = ohem_loss(seg, target, thresh=0.0, details=True)
    p = d["p"]
    vals = torch.unique(p)
    mid = vals[len(vals) // 2]
    mk = int((p < mid).sum()) + 3                              # inside the group of p_t == mid
    x = seg.to(DEV)
    sel = ohem_selection(x, target.to(DEV), thresh=0.0, min_kept=mk, reduction=reduction)
    ref = ohem_loss(seg, target, thresh=0.0, min_kept=mk, reduction=reduction, details=True)
    assert sel["branch"] == "select" and sel["count"] == ref["count"] == int((p < mid).sum())
    assert torch.equal(sel["selected"].cpu(), ref["selected"])
    for v in vals:                                             # every group in or out as a whole
        grp = (p == v).to(DEV)
        assert bool(sel["selected"][grp].all()) or not bool(sel["selected"][grp].any())
    check_ohem(seg, target, thresh=0.0, min_kept=mk, reduction=reduction, branch="select", gap=False)


# ---- degenerate counts ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_no_labelled_pixel_gives_zero(reduction):
    seg, _ = _inputs(2, 5, 8, 9, 30, 33, seed=4)
    target = torch.full((2, 30, 33), -1, dtype=torch.int64)
    target[1, :3] = 77                                         # out of range: ignored as well
    x = seg.to(DEV).requires_grad_(True)
    loss = cs.upsample_ohem_cross_entropy(x, target.to(DEV), thresh=0.7, min_kept=100, reduction=reduction)
    loss.backward()
    assert loss.item() == 0.0 and torch.count_nonzero(x.grad).item() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_empty_selection(reduction):
    """n = 1 with thresh below its p_t, and every p_t equal: nothing lies below the threshold.  NaN for 'mean', 0 for
    'sum', a zero gradient either way (the reference's mean and sum of an empty selection)."""
    seg, _ = _inputs(1, 5, 8, 9, 30, 33, seed=6)
    one = torch.full((1, 30, 33), -1, dtype=torch.int64)
    one[0, 11, 12] = 2
    flat = torch.zeros(1, 5, 8, 9)
    full = torch.full((1, 30, 33), 3, dtype=torch.int64)
    for s, t in ((seg, one), (flat, full)):
        x = s.to(DEV).requires_grad_(True)
        loss = cs.upsample_ohem_cross_entropy(x, t.to(DEV), thresh=0.0, min_kept=5, reduction=reduction)
        loss.backward()
        if reduction == "mean":
            assert math.isnan(loss.item())
        else:
            assert loss.item() == 0.0
        assert torch.count_nonzero(x.grad).item() == 0


# ---- half inputs ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ohem_half_inputs_equal_the_fp32_call(dtype):
    seg, target = _inputs(2, 19, 17, 23, 66, 90, seed=61)
    t = target.to(DEV)
    for mk in (10, 8000):
        xh = seg.to(DEV, dtype).requires_grad_(True)
        lh = cs.upsample_ohem_cross_entropy(xh, t, thresh=0.3, min_kept=mk)
        lh.backward()
        xf = xh.detach().float().requires_grad_(True)
        lf = cs.upsample_ohem_cross_entropy(xf, t, thresh=0.3, min_kept=mk)
        lf.backward()
        assert torch.equal(lh.detach(), lf.detach())
        assert xh.grad.dtype == dtype and torch.equal(xh.grad, xf.grad.to(dtype))


# ---- determinism and capture -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("branch", ["threshold", "select"])
def test_ohem_bit_reproducible_and_graph_replays_eager(branch):
    B, K, h, w, H, W = 2, 19, 32, 64, 128, 256
    seg, target = _inputs(B, K, h, w, H, W, seed=71)
    mk = branch_min_kept(seg, target, branch, 0.3)
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    eager = cs.upsample_ohem_cross_entropy(x, t, thresh=0.3, min_kept=mk)
    eager.backward()
    assert ohem_selection(x.detach(), t, thresh=0.3, min_kept=mk)["branch"] == branch
    for _ in range(3):
        assert torch.equal(eager.detach(), cs.upsample_ohem_cross_entropy(x.detach(), t, thresh=0.3, min_kept=mk))
    eager_loss, eager_grad = eager.detach().clone(), x.grad.clone()
    xg = seg.to(DEV).requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xg.grad = None
            cs.upsample_ohem_cross_entropy(xg, t, thresh=0.3, min_kept=mk).backward()
    torch.cuda.current_stream().wait_stream(s)
    xg.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = cs.upsample_ohem_cross_entropy(xg, t, thresh=0.3, min_kept=mk)
        out.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.detach(), eager_loss)
    assert (xg.grad - eager_grad).abs().max().item() <= 1e-6 * eager_grad.abs().max().item()


@pytest.mark.gpu
def test_ohem_refusals():
    seg, target = _inputs(1, 3, 8, 8, 20, 20, seed=5)
    with pytest.raises(_abi.PclError):
        cs.upsample_ohem_cross_entropy(seg.to(DEV), target[:, :6, :6].to(DEV))              # down-sampling
    with pytest.raises(_abi.PclError):
        cs.upsample_ohem_cross_entropy(torch.zeros(1, 257, 4, 4, device=DEV),
                                       torch.zeros(1, 4, 4, dtype=torch.int64, device=DEV))
    with pytest.raises(NotImplementedError):
        cs.upsample_ohem_cross_entropy(seg.to(DEV), target.to(DEV), reduction="none")


# ---- full Cityscapes shape through the wrappers -------------------------------------------------------------------
def _ohem_config(with_memory=False, thresh=0.7, min_kept=100000):
    d = cs.cityscapes_contrast_config(with_memory=with_memory)
    d["loss"]["params"].update(ohem_thresh=thresh, ohem_minkeep=min_kept, ce_ignore_index=-1)
    d["network"]["loss_weights"] = {"seg_loss": 1.0, "aux_loss": 0.4}
    return d


def _check_full(loss, expect, grads, near_up, h, w):
    lerr = abs(loss.item() - expect.item()) / abs(expect.item())
    print(f"ohem full shape: loss rel {lerr:.3e}")
    assert lerr <= FULL_LOSS_REL, (loss.item(), expect.item())
    keep = ~footprint_mask(near_up, h, w)
    for g, gref in grads:
        err = (g.double() - gref.double()).abs().amax(dim=1)[keep].max().item() / gref.abs().max().item()
        print(f"ohem full shape: grad max {err:.3e} (near-threshold footprints {int((~keep).sum())})")
        assert err <= GRAD_MAX, err


@pytest.mark.gpu
def test_ohem_full_shape_through_contrast_ce_wrapper():
    """ContrastCELoss(seg_criterion=FSOhemCELoss) at B=8, 19 x 128x256 -> 512x1024 against the oracle's fp32 op
    sequence (the reference's own precision) on the up-sampled logits; the gradient off the near-threshold footprints."""
    B, K, h, w, H, W = 8, 19, 128, 256, 512, 1024
    seg, target = _inputs(B, K, h, w, H, W, seed=81)
    cfg = cs.Configer(_ohem_config())
    x = seg.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    embed = F.normalize(torch.randn(B, 256, h, w, device=DEV), dim=1).requires_grad_(True)
    crit = cs.ContrastCELoss(cfg, seg_criterion=cs.FSOhemCELoss(cfg))
    loss = crit({"seg": x, "embed": embed}, t, with_embed=False)
    loss.backward()
    xr = x.detach().clone().requires_grad_(True)
    d = ohem_loss(xr, t, thresh=0.7, min_kept=100000, front=torch.float32, near_ulps=NEAR_ULPS, details=True)
    d["loss"].backward()
    _check_full(loss, d["loss"], [(x.grad, xr.grad)], d["near"], h, w)


@pytest.mark.gpu
def test_ohem_full_shape_through_contrast_auxce_wrapper():
    B, K, h, w, H, W = 8, 19, 128, 256, 512, 1024
    seg, target = _inputs(B, K, h, w, H, W, seed=83)
    aux, _ = _inputs(B, K, h, w, H, W, seed=84, scale=2.0)
    cfg = cs.Configer(_ohem_config())
    x, xa = seg.to(DEV).requires_grad_(True), aux.to(DEV).requires_grad_(True)
    t = target.to(DEV)
    embed = F.normalize(torch.randn(B, 256, h, w, device=DEV), dim=1).requires_grad_(True)
    crit = cs.ContrastAuxCELoss(cfg, seg_criterion=cs.FSAuxOhemCELoss(cfg))
    loss = crit({"seg": x, "seg_aux": xa, "embed": embed}, t, with_embed=False)
    loss.backward()
    xr, xar = x.detach().clone().requires_grad_(True), xa.detach().clone().requires_grad_(True)
    d = ohem_loss(xr, t, thresh=0.7, min_kept=100000, front=torch.float32, near_ulps=NEAR_ULPS, details=True)
    up_aux = F.interpolate(xar, size=(H, W), mode="bilinear", align_corners=True)
    expect = 1.0 * d["loss"] + 0.4 * F.cross_entropy(up_aux, t, ignore_index=-1)
    expect.backward()
    _check_full(loss, expect, [(x.grad, xr.grad), (xa.grad, xar.grad)], d["near"], h, w)
