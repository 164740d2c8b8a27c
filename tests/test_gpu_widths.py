"""Every embedding width the exact fp32 path takes (D % 32 == 0, D <= 256: include/pcl.h) against float64.  The rest of
the suite runs 32, 64 and 256 only, yet several kernels change behaviour with D, not just their trip counts:

  * the SIMT sweeps (csrc/pcl_infonce_simt.cu, pcl_simt_tile.cuh): load_tile_T walks D in four 8-channel quarters of
    every 32 channels, the backward keeps nq = D / 16 of its 16 accumulator columns live, and the dynamic shared memory
    (2 * D * 68 floats plus the gradient tile) crosses the 48 KB opt-in line between widths;
  * the step's gather and scatter (csrc/pcl_select.cu): k_zero_scatter runs one CTA per (image, channel) plane, the
    normalise path's k_scatter strides D by 32 lanes, half-precision gradients are written in embed's dtype;
  * the bank (csrc/pcl_bank.cu): the packet's segment sums split D into groups of 8 channels, rows and the apply step D
    by 32 lanes; the bank takes any D > 0, so a width that is not a multiple of 32 runs too;
  * the L2-normalise kernel (csrc/pcl_norm.cu) keeps 256 channels in registers and streams the rest.

Tolerances are those of the exact path (tests/test_gpu_parity.py): loss 2e-6 relative, gradient 1e-5 * max|g|, positive
counts exact, bank rows 1.5e-7 / segment means 1e-6, half-precision embeds bit for bit against their fp32 copies.  Widths
outside the rule are refused before anything runs.  The functions take DEV and their sizes as arguments so that
tests/test_emu_widths.py runs them on the emulated kernels."""
import ctypes as C
import gc
import math

import pytest
import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi, functional as Fn
from contrastiveseg_b200.synth import make_bank, make_contrast_batch, make_sweep_point
from oracle import ref_port as P
from helpers import rel_err
import test_gpu_topk as TK

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda:0"

WIDTHS = (32, 64, 96, 128, 160, 192, 224, 256)
TOPK_WIDTHS = (32, 96, 160, 256)
BANK_WIDTHS = WIDTHS + (100,)              # the bank takes any D > 0: 100 leaves a partial 8-channel group
NORM_CHANNELS = (255, 256, 257, 288)       # around the normalise kernel's 256 register-resident channels
OPT_IN_ORDER = (256, 32, 160, 64, 224, 96)
HALF = (torch.bfloat16, torch.float16)

# (A, N or bank rows M0, pixel rows M1): A and N off the 64 x 64 tile
SWEEP_SIZES = {"explicit": (200, 700, None), "self": (333, None, None), "bank": (150, 37, 23), "bank_m1_0": (150, 50, 0)}
TOPK_SIZES = {"explicit": (130, 333), "self": (150, None), "bank": (90, 12)}
TOPK_KS = (1, 9, 10 ** 6)                  # k = 1, a middle value, k >= N (nothing dropped)


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _d(t):
    """A device copy that never aliases the host tensor (on the emulator DEV is the CPU)."""
    return None if t is None else t.detach().clone().to(DEV)


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


def _sorted_by_class_rank(a, ya, K):
    """The engine's row layout of bank-mode anchors: class rank 1, 2, ..., K-1, then 0."""
    order = torch.argsort(torch.where(ya == 0, K, ya), stable=True)
    return a[order], ya[order]


# ---------------------------------------------------------------------------------------------------
# exact sweeps
# ---------------------------------------------------------------------------------------------------
def check_sweep(mode, D, A, N, M1, T=0.1, bT=0.07):
    """Fn.infonce_forward / infonce_backward in one mode against the float64 closed form."""
    seed = D * 10 + A
    if mode == "explicit":
        pt = make_sweep_point(A, N, D=D, num_classes=6, seed=seed, clustered=0.5)
        a, ya, c, yc = pt["anchors"], pt["ya"], pt["contrast"], pt["yc"]
        diag = torch.arange(A) % N
        loss, st, state = Fn.infonce_forward(_d(a), _d(ya), contrast=_d(c), contrast_cls=_d(yc), diag_col=_d(diag),
                                             temperature=T, base_temperature=bT)
        cf = P.infonce_closed_form(a.double(), ya, c.double(), yc, T, bT, self_contrast=False, diag_cols=diag)
    elif mode == "self":
        pt = make_sweep_point(A, 1, D=D, num_classes=6, seed=seed, clustered=0.5)
        a, ya = pt["anchors"], pt["ya"]
        loss, st, state = Fn.infonce_forward(_d(a), _d(ya), temperature=T, base_temperature=bT)
        cf = P.infonce_closed_form(a.double(), ya, a.double(), ya, T, bT, self_contrast=True)
    else:                                  # bank: N segment rows and M1 pixel rows per class (M1 = 0: no pixel queue)
        K = 5
        pt = make_sweep_point(A, 1, D=D, num_classes=K, seed=seed, clustered=0.5)
        a, ya = _sorted_by_class_rank(pt["anchors"], pt["ya"], K)
        queues = (make_bank(K, N, D, seed)["segment_queue"],)
        if M1:
            queues += (make_bank(K, M1, D, seed + 1)["pixel_queue"],)
        contrast, yc = P.flatten_queue(torch.cat(queues, 1).double())
        loss, st, state = Fn.infonce_forward(_d(a), _d(ya), queues=tuple(_d(q) for q in queues),
                                             diag_col=_d(torch.arange(A)), temperature=T, base_temperature=bT)
        cf = P.infonce_closed_form(a.double(), ya, contrast, yc.long(), T, bT, self_contrast=False)
    dA = Fn.infonce_backward(state, st)
    _sync()
    assert torch.isfinite(cf["loss"]) and cf["npos"].min().item() > 0
    assert rel_err(loss.item(), cf["loss"].item()) < 2e-6, (loss.item(), cf["loss"].item())
    assert torch.equal(st[4].cpu().double(), cf["npos"])
    gmax = cf["dA"].abs().max().item()
    err = (dA.cpu().double() - cf["dA"]).abs().max().item()
    assert err <= 1e-5 * gmax, (err, gmax)


@pytest.mark.parametrize("mode,D", [pytest.param(m, D, id=f"{m}-{D}-w") for m in SWEEP_SIZES for D in WIDTHS])
def test_exact_sweeps_at_every_width(mode, D):
    check_sweep(mode, D, *SWEEP_SIZES[mode])


# ---------------------------------------------------------------------------------------------------
# top-k sweeps (H1-H3, NEGW, POS, BWDW): dyadic operands, so every logit is exact in fp32 and ties are real
# ---------------------------------------------------------------------------------------------------
def check_topk(mode, D, k, A, N):
    # a power-of-two temperature that grows with D keeps the logits exact and the self-contrast diagonal (|a|^2 / T, about
    # D / 4 / T for these rows) within exp's fp32 range
    T, bT = 0.125 * 2 ** max(0, math.ceil(math.log2(D / 32))), 0.25
    seed = D * 7 + k % 1000 + A
    if mode == "bank":
        K, M = 5, N
        g = torch.Generator().manual_seed(seed)
        segq = torch.randint(-3, 4, (K, M, D), generator=g).double() / 4
        pixq = torch.randint(-3, 4, (K, M, D), generator=g).double() / 4
        pixq[:, ::3] = 0                   # exact-zero bank rows tie with the analytic zero tail
        a = torch.randint(-3, 4, (A, D), generator=g).double() / 4
        a, ya = _sorted_by_class_rank(a, torch.randint(0, K, (A,), generator=g), K)
        contrast, yc = P.flatten_queue(torch.cat((segq, pixq), 1))
        o = P.infonce_topk(a, ya, contrast, yc.long(), T, bT, k, False)
        loss, st, state = Fn.infonce_forward(_d(a.float()), _d(ya), queues=(_d(segq.float()), _d(pixq.float())),
                                             diag_col=_d(torch.arange(A)), temperature=T, base_temperature=bT, topk=k)
    elif mode == "self":
        a, _, ya, _ = TK._dyadic(A, 8, D, 4, seed=seed, zero_every=0)
        o = P.infonce_topk(a, ya, a, ya, T, bT, k, True)
        loss, st, state = Fn.infonce_forward(_d(a.float()), _d(ya), temperature=T, base_temperature=bT, topk=k)
    else:
        a, c, ya, yc = TK._dyadic(A, N, D, 5, seed=seed)
        diag = torch.arange(A) % N
        o = P.infonce_topk(a, ya, c, yc, T, bT, k, False, diag_cols=diag)
        loss, st, state = Fn.infonce_forward(_d(a.float()), _d(ya), contrast=_d(c.float()), contrast_cls=_d(yc),
                                             diag_col=_d(diag), temperature=T, base_temperature=bT, topk=k)
    dA = Fn.infonce_backward(state, st)
    _sync()
    assert rel_err(loss.item(), o["loss"].item()) < 2e-6, (loss.item(), o["loss"].item())
    assert torch.equal(st[4].cpu().double(), o["npos"])
    gmax = o["dA"].abs().max().item()
    err = (dA.cpu().double() - o["dA"]).abs().max().item()
    assert err <= 1e-5 * gmax, (err, gmax)


@pytest.mark.parametrize("mode,D,k", [pytest.param(m, D, k, id=f"{m}-{D}-k{k}") for m in TOPK_SIZES
                                      for D in TOPK_WIDTHS for k in TOPK_KS])
def test_topk_sweeps_at_widths(mode, D, k):
    check_topk(mode, D, k, *TOPK_SIZES[mode])


# ---------------------------------------------------------------------------------------------------
# the whole eager step: scan, selection and gather, sweeps, scatter
# ---------------------------------------------------------------------------------------------------
def check_eager_step(D, mem, normalize, dtype, B=2, h=24, w=32, ms=200, mv=12, K=6, M=30):
    """cs.pixel_contrast_loss on injected permutations against the float64 pixel_contrast_loss of the reference, with or
    without a bank, on the normalised embedding or (normalize=True) the raw projection.  A half-precision embed is
    compared with the same call on its fp32 copy: the same anchors and loss bit for bit, the gradient the fp32 one
    rounded once."""
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=D + 2 * mem + normalize)
    x = data["embed_raw"] * 3.0 if normalize else data["embed"]
    if dtype != torch.float32:
        x = x.to(dtype).float()            # the values the half embed holds
    target, seg = data["target"], data["seg"]
    bank = make_bank(K, M, D, D + 1) if mem else None
    rec = P.PermRecorder(torch.Generator().manual_seed(D))
    x64 = x.double().requires_grad_(True)
    feats = F.normalize(x64, p=2, dim=1) if normalize else x64
    queue = torch.cat((bank["segment_queue"], bank["pixel_queue"]), 1).double() if mem else None
    ref = P.pixel_contrast_loss(feats, target, seg.argmax(1), temperature=0.1, base_temperature=0.07, max_samples=ms,
                                max_views=mv, queue=queue, perm_fn=rec)
    ref.backward()

    def run(e_in):
        opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, num_classes=K,
                                  normalize=normalize, perm_fn=P.PermReplay(rec.draws))
        kw = dict(segment_queue=_d(bank["segment_queue"]), pixel_queue=_d(bank["pixel_queue"])) if mem else {}
        e = _d(e_in).requires_grad_(True)
        loss = cs.pixel_contrast_loss(e, _d(target), seg=_d(seg), options=opts, **kw)
        meta = Fn.last_workspace(e.device).anchor_meta.clone()
        loss.backward()
        _sync()
        return loss.detach(), e.grad, meta

    l32, g32, m32 = run(x)
    assert rel_err(l32.item(), ref.item()) < 2e-6, (l32.item(), ref.item())
    gmax = x64.grad.abs().max().item()
    err = (g32.cpu().double() - x64.grad).abs().max().item()
    assert err <= 1e-5 * gmax, (err, gmax)
    if dtype != torch.float32:
        lh, gh, mh = run(x.to(dtype))
        assert torch.equal(mh, m32) and torch.equal(lh, l32)
        assert gh.dtype == dtype and torch.equal(gh, g32.to(dtype))


def _step_cases():
    cases = []
    for D in WIDTHS:
        for mem in (False, True):
            for normalize in (False, True):
                for dtype, name in ((torch.float32, "fp32"), (torch.bfloat16, "bf16"), (torch.float16, "fp16")):
                    cases.append(pytest.param(D, mem, normalize, dtype, id=f"{'bank' if mem else 'self'}-{D}-"
                                              f"{'raw' if normalize else 'unit'}-{name}"))
    return cases


@pytest.mark.parametrize("D,mem,normalize,dtype", _step_cases())
def test_eager_step_at_every_width(D, mem, normalize, dtype):
    check_eager_step(D, mem, normalize, dtype)


# ---------------------------------------------------------------------------------------------------
# captured step (the streaming path: the one-kernel InfoNCE is D = 256 only)
# ---------------------------------------------------------------------------------------------------
def check_captured_step(D, mem, B=2, h=24, w=32, ms=200, mv=12, K=6, M=30, replays=3):
    """Replay r of GraphedContrastStep(precision='fp32') equals the eager step with step counter r + 1, bit for bit."""
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=D + 5)
    embed, tgt, seg = _d(data["embed"]), _d(data["target"]), _d(data["seg"])
    kw = {}
    if mem:
        bank = make_bank(K, M, D, D + 6)
        kw = dict(segment_queue=_d(bank["segment_queue"]), pixel_queue=_d(bank["pixel_queue"]))
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, seed=4,
                              precision="fp32", num_classes=K)
    step = cs.GraphedContrastStep(embed, tgt, seg=seg, options=opts, **kw)
    assert not step.fused
    for r in range(replays):
        loss, grad = step.replay()
        _sync()
        loss, grad = loss.clone(), grad.clone()
        Fn._step_counter[0] = r
        e = embed.clone().requires_grad_(True)
        l = cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts, **kw)
        l.backward()
        _sync()
        assert torch.isfinite(loss) and grad.abs().max().item() > 0
        assert torch.equal(l.detach(), loss) and torch.equal(e.grad, grad), r


@pytest.mark.parametrize("mem,D", [pytest.param(m, D, id=f"{'bank' if m else 'self'}-{D}-fp32") for m in (False, True)
                                   for D in (96, 160)])
def test_captured_step_at_widths(mem, D):
    check_captured_step(D, mem)


# ---------------------------------------------------------------------------------------------------
# bank enqueue
# ---------------------------------------------------------------------------------------------------
def check_bank_enqueue(D, K=6, M=12, freq=5, B=2, h=16, w=16, stride=2, steps=3):
    """Three enqueues against the reference's _dequeue_and_enqueue on replayed permutations: pointers exact, rows within
    the bounds of test_bank_enqueue_matches_reference; the incrementally kept bf16 shadow equals a rebuild."""
    g = torch.Generator().manual_seed(D)
    torch.manual_seed(D)
    bank = cs.MemoryBank(K, M, D, with_shadow=True).to(DEV)
    bank.sync_shadow()
    sq, sp = bank.segment_queue.cpu().clone(), bank.segment_queue_ptr.cpu().clone()
    pq, pp = bank.pixel_queue.cpu().clone(), bank.pixel_queue_ptr.cpu().clone()
    for s in range(steps):
        keys = torch.randn(B, D, h, w, generator=g)
        labels = torch.randint(-1, K, (B, h, w), generator=g)
        labels = labels.repeat_interleave(stride, 1).repeat_interleave(stride, 2)
        rec = P.PermRecorder(torch.Generator().manual_seed(100 + s))
        P.dequeue_and_enqueue(keys, labels, sq, sp, pq, pp, network_stride=stride, memory_size=M, pixel_update_freq=freq,
                              perm_fn=rec)
        replay = P.PermReplay(rec.draws)
        bank.enqueue(_d(keys), _d(labels), network_stride=stride, pixel_update_freq=freq, perm_fn=replay)
        _sync()
        assert replay.pos == len(replay.draws)
        assert torch.equal(bank.segment_queue_ptr.cpu(), sp) and torch.equal(bank.pixel_queue_ptr.cpu(), pp)
        assert (bank.pixel_queue.cpu() - pq).abs().max().item() <= 1.5e-7
        assert (bank.segment_queue.cpu() - sq).abs().max().item() <= 1e-6
    assert int(sp.max()) > 1 and int(pp.max()) > 0
    inc = bank.shadow.clone()
    assert torch.equal(inc, bank.sync_shadow())


@pytest.mark.parametrize("D", BANK_WIDTHS, ids=[f"D{D}" for D in BANK_WIDTHS])
def test_bank_enqueue_at_widths(D):
    check_bank_enqueue(D)


# ---------------------------------------------------------------------------------------------------
# L2 normalise around its register / streamed split
# ---------------------------------------------------------------------------------------------------
def check_l2_normalize(C, B=2, H=5, W=7):
    g = torch.Generator().manual_seed(C)
    x = torch.randn(B, C, H, W, generator=g)
    gy = torch.randn(B, C, H, W, generator=g)
    xd = _d(x).requires_grad_(True)
    y = cs.l2_normalize(xd)
    y.backward(_d(gy))
    x64 = x.double().requires_grad_(True)
    y64 = P.l2_normalize(x64)
    y64.backward(gy.double())
    assert torch.allclose(y.detach().cpu().double(), y64.detach(), rtol=1e-6, atol=1e-7)
    assert torch.allclose(xd.grad.cpu().double(), x64.grad, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("C", NORM_CHANNELS)
def test_l2_normalize_around_the_register_split(C):
    check_l2_normalize(C)


# ---------------------------------------------------------------------------------------------------
# shared-memory opt-in across widths
# ---------------------------------------------------------------------------------------------------
def _step_at(D, topk, B=2, h=16, w=32, ms=150, mv=8, K=5):
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=D + 9)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, num_classes=K,
                              topk_negatives=topk, perm_fn=P.PermRecorder(torch.Generator().manual_seed(D)))
    e = _d(data["embed"]).requires_grad_(True)
    loss = cs.pixel_contrast_loss(e, _d(data["target"]), seg=_d(data["seg"]), options=opts)
    loss.backward()
    _sync()
    return loss.detach().clone(), e.grad.clone()


def check_opt_in_order(order=OPT_IN_ORDER, **sizes):
    """Forward and backward (stock and top-k sweeps) in a width order that raises and lowers the dynamic shared memory
    from launch to launch: every result equals the same width run again after Fn.clear_workspaces()."""
    seq = {D: (_step_at(D, None, **sizes), _step_at(D, 5, **sizes)) for D in order}
    for D in order:
        Fn.clear_workspaces()
        alone = (_step_at(D, None, **sizes), _step_at(D, 5, **sizes))
        for (l0, g0), (l1, g1) in zip(seq[D], alone):
            assert torch.isfinite(l0) and torch.equal(l0, l1) and torch.equal(g0, g1), D


def test_smem_opt_in_across_widths():
    check_opt_in_order()


# ---------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------
def check_width_refused(D, K=5, M=8):
    """A width outside D % 32 == 0, D <= 256 is an error before any launch: the sizing calls refuse it, and the loss
    raises without leaving a gradient, a cached workspace, a pending bank reader or a change to the bank behind."""
    lib = _abi.load()
    geom = _abi.Geom(2, D, 8, 8, 16, 16, K, 32, 4, -1)
    assert lib.pcl_select_sizes(C.byref(geom), C.byref(_abi.SelectSizes())) != 0
    data = make_contrast_batch(B=2, D=D, h=8, w=8, num_classes=K, img_stride=2, block=4, seed=D)
    embed = _d(data["embed"]).requires_grad_(True)
    tgt, seg = _d(data["target"]), _d(data["seg"])
    torch.manual_seed(D)
    bank = cs.MemoryBank(K, M, D).to(DEV)
    names = ("segment_queue", "segment_queue_ptr", "pixel_queue", "pixel_queue_ptr")
    before = [getattr(bank, n).clone() for n in names]
    cache = set(Fn._WS_CACHE)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=32, max_views=4, num_classes=K)
    for kw in ({}, dict(segment_queue=bank.segment_queue, pixel_queue=bank.pixel_queue)):
        with pytest.raises(_abi.PclError):
            cs.pixel_contrast_loss(embed, tgt, seg=seg, options=opts, **kw)
    with pytest.raises(_abi.PclError):
        Fn.infonce_forward(embed.detach()[0, :, 0, :].t().contiguous(), torch.zeros(8, dtype=torch.long, device=DEV))
    assert embed.grad is None
    assert set(Fn._WS_CACHE) == cache
    assert Fn.bank_reader(bank.segment_queue.device.index, bank.segment_queue.data_ptr()) is None
    for n, t in zip(names, before):
        assert torch.equal(getattr(bank, n), t), n
    # no bank write is held back for a backward that will never run: an enqueue lands at once
    bank.enqueue(embed.detach(), tgt, network_stride=2, pixel_update_freq=2)
    _sync()
    assert not torch.equal(bank.segment_queue_ptr, before[1])


@pytest.mark.parametrize("D", [16, 48, 288])
def test_unsupported_width_is_refused_without_side_effects(D):
    check_width_refused(D)


def check_bf16_refused_below_256(D=128, K=5):
    data = make_contrast_batch(B=2, D=D, h=8, w=8, num_classes=K, img_stride=2, block=4, seed=D)
    embed, tgt, seg = _d(data["embed"]), _d(data["target"]), _d(data["seg"])
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=32, max_views=4, num_classes=K,
                              precision="bf16")
    e = embed.clone().requires_grad_(True)
    with pytest.raises(_abi.PclError):
        cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts)
    assert e.grad is None
    with pytest.raises(_abi.PclError):
        cs.GraphedContrastStep(embed, tgt, seg=seg, options=opts, capture=False)
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, proj_dim=D, fused=True)


def test_tensor_path_and_fused_head_refuse_widths_below_256():
    check_bf16_refused_below_256()
