"""The seg CE forward and backward in one tile pass (pcl_seg_ce_fwd_bwd, functional.seg_ce_loss_and_grad) and the whole
contrast criterion replayed as one CUDA graph (GraphedContrastCriterion).

Kernel: the loss is the two-call form's (pcl_seg_ce_fwd) to the bit, dseg within 1e-6 max|g| of pcl_seg_ce_bwd with the
same upstream gradient and within 1e-5 max|g| of float64 F.interpolate + F.cross_entropy.

Criterion: against the eager wrapper's seg terms plus loss_weight times a twin GraphedContrastStep built from the same
options and seed.  tests/test_emu_graphed_criterion.py runs these functions on the emulated kernels."""
import gc

import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi, functional as Fn
import test_gpu_many_classes as M

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------
# A. pcl_seg_ce_fwd_bwd
# ---------------------------------------------------------------------------------------------------
KERNEL_CASES = [
    # B, K, h, w, H, W, weighted, ignore_index
    (2, 2, 9, 11, 37, 45, False, -1),          # label grid not a multiple of the 32 x 8 tile
    (2, 19, 17, 23, 66, 90, True, -1),
    (2, 19, 17, 23, 66, 90, False, 255),
    (2, 25, 17, 23, 66, 90, True, 255),        # two class chunks (24 + 1): the pre stages every chunk, the fill again
    (2, 25, 13, 21, 50, 70, False, -1),
    (1, 171, 13, 13, 52, 52, True, -1),
    (1, 171, 13, 13, 52, 52, False, 255),
    (2, 19, 33, 41, 33, 41, True, -1),         # identity geometry
]


def check_fwd_bwd(B, K, h, w, H, W, weighted, ignore_index, seed=0, grad=0.7, all_ignored=False):
    seg, target, weight = M._seg_ce_inputs(B, K, h, w, H, W, weighted, ignore_index, seed)
    if all_ignored:
        target.fill_(ignore_index)
    s, t = seg.to(DEV), target.to(DEV)
    wt = weight.to(DEV) if weighted else None
    loss, dseg = Fn.seg_ce_loss_and_grad(s, t, wt, ignore_index, grad_scale=torch.tensor(grad, device=DEV))
    s2 = s.clone().requires_grad_(True)                       # the two-call form: pcl_seg_ce_fwd + pcl_seg_ce_bwd
    pair = cs.upsample_cross_entropy(s2, t, wt, ignore_index)
    pair.backward(torch.tensor(grad, device=DEV))
    if all_ignored:
        assert torch.isnan(loss) and torch.isnan(pair)
        assert not bool(dseg.any()) and not bool(s2.grad.any())
        return
    assert torch.equal(loss, pair), (loss.item(), pair.item())
    gmax = s2.grad.abs().max().item()
    assert (dseg - s2.grad).abs().max().item() <= 1e-6 * gmax
    s64 = s.double().requires_grad_(True)
    ref = M.seg_ce_reference(s64, t, wt.double() if weighted else None, ignore_index)
    ref.backward(torch.tensor(grad, dtype=torch.float64, device=DEV))
    gmax = s64.grad.abs().max().item()
    assert (dseg.double() - s64.grad).abs().max().item() <= 1e-5 * gmax
    assert abs(loss.item() - ref.item()) <= 2e-6 * abs(ref.item())


@pytest.mark.parametrize("B,K,h,w,H,W,weighted,ignore_index", KERNEL_CASES)
def test_seg_ce_fwd_bwd_matches_the_two_call_form(B, K, h, w, H, W, weighted, ignore_index):
    check_fwd_bwd(B, K, h, w, H, W, weighted, ignore_index, seed=K + h + W)


@pytest.mark.parametrize("ignore_index", [-1, 255])
def test_seg_ce_fwd_bwd_every_pixel_ignored(ignore_index):
    check_fwd_bwd(2, 19, 9, 11, 37, 45, True, ignore_index, all_ignored=True)


def check_two_call_every_pixel_ignored(H, W, ignore_index=255, B=2, K=5, h=9, w=11):
    """A label grid smaller than seg (the two-call form's gather backward) with every pixel ignored: NaN loss and a zero
    gradient, as with up-sampling and in torch (the gather divided by the zero weight sum: NaN everywhere)."""
    seg, target, _ = M._seg_ce_inputs(B, K, h, w, H, W, False, ignore_index, seed=H * W)
    target.fill_(ignore_index)
    x = seg.to(DEV).requires_grad_(True)
    loss = cs.upsample_cross_entropy(x, target.to(DEV), None, ignore_index)
    loss.backward(torch.tensor(0.7, device=DEV))
    assert torch.isnan(loss).item()
    assert torch.count_nonzero(x.grad).item() == 0          # (NaN counts as non-zero)


@pytest.mark.parametrize("H,W", [(5, 11), (9, 6), (4, 5)])
def test_seg_ce_two_call_every_pixel_ignored_below_the_logit_grid(H, W):
    check_two_call_every_pixel_ignored(H, W)


def test_seg_ce_fwd_bwd_refuses_down_sampling():
    seg = torch.randn(2, 5, 40, 40, device=DEV)
    target = torch.zeros(2, 20, 50, dtype=torch.int64, device=DEV)
    with pytest.raises(_abi.PclError):
        Fn.seg_ce_loss_and_grad(seg, target)


# ---------------------------------------------------------------------------------------------------
# B. GraphedContrastCriterion against the eager seg terms + loss_weight * a twin GraphedContrastStep
# ---------------------------------------------------------------------------------------------------
K_CRIT = 19
# name: (wrapper, seg criterion class or None for the wrapper's default, contrast.use_rmi)
CRITERIA = {
    "ce": (cs.ContrastCELoss, None, False),
    "ce_lovasz": (cs.ContrastCELoss, cs.FSCELOVASZLoss, False),
    "ce_ohem": (cs.ContrastCELoss, cs.FSOhemCELoss, False),
    "aux_ce": (cs.ContrastAuxCELoss, None, False),
    "aux_rmi": (cs.ContrastAuxCELoss, None, True),
    "aux_ohem": (cs.ContrastAuxCELoss, cs.FSAuxOhemCELoss, False),
    "mem_ce": (cs.MemContrastCELoss, None, False),
    "mem_rmi": (cs.MemContrastCELoss, None, True),
    "mem_lovasz": (cs.MemContrastCELoss, cs.FSCELOVASZLoss, False),
    "mem_ohem": (cs.MemContrastCELoss, cs.FSOhemCELoss, False),
}


def make_criterion(name, ms=256, extra=None, K=K_CRIT, params=None, loss_weights=None):
    """The criterion `name` with this file's configuration; K, `params` (loss.params entries) and `loss_weights`
    (network.loss_weights) override it (the criterion fuzzer of tests/emu_fuzz.py draws them)."""
    wrapper, seg_cls, use_rmi = CRITERIA[name]
    d = cs.cityscapes_contrast_config(with_memory=wrapper is cs.MemContrastCELoss)
    d["data"]["num_classes"] = K
    d["contrast"].update(dict(max_samples=ms, max_views=8, use_rmi=use_rmi), **(extra or {}))
    d["loss"]["params"].update(dict(use_sigmoid=True, num_classes=K, rmi_radius=3, rmi_pool_way=0, rmi_pool_size=3,
                                    rmi_pool_stride=3, loss_weight_lambda=0.5, loss_weight=1.0, lambda_way=1,
                                    ohem_thresh=0.7, ohem_minkeep=1000), **(params or {}))
    d["network"]["loss_weights"] = dict(loss_weights or {"seg_loss": 1.0, "aux_loss": 0.4})
    cfg = cs.Configer(d)
    return wrapper(cfg, seg_criterion=seg_cls(cfg)) if seg_cls is not None else wrapper(cfg)


def _batch(seed, B, D, h, w, aux):
    from contrastiveseg_b200.synth import make_contrast_batch
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K_CRIT, img_stride=4, block=8, seed=seed)
    out = {"seg": data["seg"], "embed": data["embed"]}
    if aux:
        out["seg_aux"] = data["seg"] * 0.5 + 0.3 * torch.randn(data["seg"].shape, generator=torch.Generator().manual_seed(seed))
    return out, data["target"]


def _close(g, ge, parts=None):
    """Within 1e-6 max|g| of the eager gradient; a half gradient may also differ by one rounding of its dtype (the two
    sides round fp32 gradients that agree to the last ulp or two).  parts (the criterion fuzzer): the fp32 gradients of
    the head's terms.  With them a half gradient may also differ by one subnormal step below its normal range (fp16
    gradients of a large label grid are that small), and with several terms, each rounded to the head's dtype before
    they are added, by three roundings on each side, which scale with the terms' magnitudes, not the sum's."""
    gmax = ge.float().abs().max().item()
    tol = 1e-6 * gmax
    if ge.dtype != torch.float32:
        fi = torch.finfo(ge.dtype)
        tol = tol + ge.float().abs() * fi.eps
        if parts is not None:
            if len(parts) > 1:
                tol = 1e-6 * gmax * len(parts) + 2 * sum(p.abs() for p in parts) * fi.eps
            tol = tol + fi.tiny * fi.eps
    return bool(((g.float() - ge.float()).abs() <= tol).all())


def check_criterion(name, dtype, B=2, D=64, h=16, w=16, replays=3, enqueue=False):
    from contrastiveseg_b200.synth import make_bank
    crit = make_criterion(name).to(DEV)
    mem = crit.with_memory
    heads = ["seg"] + (["seg_aux"] if isinstance(crit, cs.ContrastAuxCELoss) else [])
    first, target = _batch(100, B, D, h, w, len(heads) > 1)
    target = target.to(DEV)
    static = {k: first[k].to(DEV).to(dtype).requires_grad_(True) for k in heads}
    static["embed"] = first["embed"].to(DEV).requires_grad_(True)
    banks, enq = [], [None, None]
    if mem:
        for i in range(2):                      # the criterion's and the twin's (a bank step writes its bank)
            if enqueue:
                b = cs.MemoryBank(K_CRIT, 40, D).to(DEV)
                init = make_bank(K_CRIT, 40, D, seed=7)
                b.segment_queue.copy_(init["segment_queue"]), b.pixel_queue.copy_(init["pixel_queue"])
                enq[i] = dict(bank=b, network_stride=4, pixel_update_freq=4)
                banks.append((b.segment_queue, b.pixel_queue))
            else:
                init = make_bank(K_CRIT, 40, D, seed=7)
                banks.append((init["segment_queue"].to(DEV), init["pixel_queue"].to(DEV)))
        static["segment_queue"], static["pixel_queue"] = banks[0]
    gc_ = cs.GraphedContrastCriterion(crit, static, target, enqueue=enq[0])
    opts = crit.contrast_criterion.options()
    opts.num_classes = K_CRIT
    twin = cs.GraphedContrastStep(static["embed"].detach(), target, seg=static["seg"].detach(),
                                  segment_queue=banks[1][0] if mem else None, pixel_queue=banks[1][1] if mem else None,
                                  options=opts, grad_scale=crit.loss_weight, enqueue=enq[1])
    for r in range(replays):
        if r:                                   # refill the static inputs in place
            nxt, _ = _batch(100 + r, B, D, h, w, len(heads) > 1)
            with torch.no_grad():
                for k in heads + ["embed"]:
                    static[k].copy_(nxt[k].to(DEV).to(dtype) if k != "embed" else nxt[k].to(DEV))
        scale = 2.0 if r == replays - 1 else 1.0
        if r == replays - 1:
            gc_.set_grad_scale(scale)
            twin.set_grad_scale(scale * crit.loss_weight)
        loss, grads = gc_.replay()
        lc, gcon = twin.replay()
        eager = {k: static[k].detach().clone().requires_grad_(True) for k in heads}
        seg_loss = crit._seg_loss(eager, target)
        seg_loss.backward(torch.tensor(scale, device=DEV))
        torch.cuda.synchronize()
        assert torch.equal(loss, seg_loss.detach() + crit.loss_weight * lc), (name, r, loss.item(), seg_loss.item())
        assert torch.equal(grads["embed"], gcon)
        for k in heads:
            assert grads[k].dtype == dtype and _close(grads[k], eager[k].grad), (name, k, r)
        if enqueue:
            assert torch.equal(banks[0][0], banks[1][0]) and torch.equal(banks[0][1], banks[1][1])
    gc_.set_grad_scale(1.0)
    for k in heads + ["embed"]:
        static[k].grad = None
    gc_.apply(static).backward()
    for k in heads + ["embed"]:
        assert torch.equal(static[k].grad, grads[k]), k


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("name", list(CRITERIA))
def test_graphed_criterion_matches_eager_and_twin(name, dtype):
    check_criterion(name, dtype)


@pytest.mark.parametrize("name", ["mem_ce", "mem_lovasz"])
def test_graphed_criterion_bank_step(name):
    check_criterion(name, torch.float32, enqueue=True)


def check_refusals(B=2, D=64, h=16, w=16):
    preds, target = _batch(1, B, D, h, w, True)
    preds = {k: v.to(DEV) for k, v in preds.items()}
    target = target.to(DEV)

    def refused(crit, p=preds, t=target):
        with pytest.raises(_abi.PclError):
            cs.GraphedContrastCriterion(crit, p, t)

    refused(make_criterion("ce", extra={"fused_seg_ce": False}))
    refused(make_criterion("aux_rmi", extra={"fused_seg_ce": False}))
    refused(make_criterion("ce", extra={"rng": "torch_cpu"}))
    refused(make_criterion("mem_ce"))                                        # no queues
    refused(make_criterion("ce"), p=dict(preds, seg=preds["seg"].transpose(2, 3)))
    refused(make_criterion("ce"), t=target.to(torch.int32))
    refused(make_criterion("aux_ce"), p={k: v for k, v in preds.items() if k != "seg_aux"})
    custom = make_criterion("ce")
    custom.seg_criterion = torch.nn.Identity()
    refused(custom)


def test_graphed_criterion_refusals():
    check_refusals()


# ---------------------------------------------------------------------------------------------------
# C. The captured criterion against float64 (tests/emu_fuzz.py: fuzz_graphed_criterion, graphed_criterion_case)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.timeout(1800)
def test_fuzz_captured_criteria_on_the_device():
    """Real graph replays, nothing patched: every wrapper x seg term with drawn term parameters, K up to 40 and one
    draw at 150-171 classes, B up to 8, h x w up to 120 x 120 (label grids within 8M B K H W elements), max_samples
    up to 1024; labels, heads and embed refilled between replays; every coverage category reached on scored replays."""
    import emu_fuzz
    import test_gpu_parity as G
    bad, cov = emu_fuzz.fuzz_graphed_criterion(seed=41, n=30, check_sampling=G._check_device_sampling, device=DEV,
                                               scale=10)
    assert bad == [], bad
    assert all(cov[k] >= 1 for k in emu_fuzz.CRIT_CATEGORIES), cov
    assert cov["scored"] >= 2 * cov["skipped"], cov


@pytest.mark.timeout(900)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("name", ["ce", "aux_ce"])
def test_captured_criterion_at_the_s1_shape(name, dtype):
    """tools/criterion_bench.py's S1 shape (8 x 19 x 128 x 256 logits, 512 x 1024 labels, D 256, 1024 anchors), three
    replays with refilled labels, heads and embed, grad_scale changed before the last, against float64 on the device."""
    import emu_fuzz
    import test_gpu_parity as G
    c = dict(name=name, K=19, B=8, D=256, h=128, w=256, H=512, W=1024, ms=1024, mv=100, seq="random", block=32,
             ignore=0.1, params={"ce_ignore_index": -1}, lw={"seg_loss": 1.0, "aux_loss": 0.4}, seg_dtype=dtype,
             aux_dtype=dtype, embed_dtype=torch.float32, bank="none", grad_scale=1.0, scale2=2.0, n_rep=3, r_set=2, all_ignored=False,
             seed=1234, T=None, bT=None, precision="fp32", normalize=False, nan_safe=False, ignore_label=-1,
             refused=False, stride=1, M=None, freq=None)
    cov = {k: 0 for k in emu_fuzz.CRIT_CATEGORIES + ("scored", "skipped", "refused")}
    bad = emu_fuzz.graphed_criterion_case(c, DEV, G._check_device_sampling, cov, f"S1 {name} {dtype}")
    assert bad == [], bad
    assert cov["scored"] == 3 and cov[name] == 1, cov
