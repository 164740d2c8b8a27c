"""GPU parity tests of the a10 extension (per-anchor top-k hard negatives, csrc/pcl_topk.cuh) against the oracle's
sort-based definition.  a10 is not in the reference code, default off and excluded from the reference parity bar
(SURVEY §8 a10); these tests pin the kernels to the oracle semantics.

STATUS: strict (all cases pass on the GPU); the same cases also run on
the CPU emulator (tests/test_emu_kernels.py)."""
import os

import numpy as np
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import functional as Fn
from oracle import ref_port as P
from helpers import load_golden, unpack_perms, rel_err

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda:0"


def _key_to_float(keys: torch.Tensor) -> np.ndarray:
    k = keys.cpu().numpy().astype(np.uint32)
    u = np.where(k & np.uint32(0x80000000), k & np.uint32(0x7FFFFFFF), ~k).astype(np.uint32)
    return u.view(np.float32)


def _dyadic(A, N, D, ncls, seed, zero_every=7):
    g = torch.Generator().manual_seed(seed)
    anchors = torch.randint(-3, 4, (A, D), generator=g).double() / 4
    contrast = torch.randint(-3, 4, (N, D), generator=g).double() / 4
    if zero_every:
        contrast[::zero_every] = 0
    ya = torch.randint(0, ncls, (A,), generator=g)
    yc = torch.randint(0, ncls, (N,), generator=g)
    return anchors, contrast, ya, yc


@pytest.mark.parametrize("A,N,k", [(70, 333, 9), (130, 1000, 1), (64, 200, 64), (200, 129, 40)])
def test_topk_explicit_exact_data(A, N, k):
    """Logits exact in fp32 (dyadic operands, T = 1/8), many ties: selection (tau, G, E), loss and dA equal the oracle."""
    a, c, ya, yc = _dyadic(A, N, 32, 5, seed=A + N + k)
    T, bT = 0.125, 0.25
    o = P.infonce_topk(a, ya, c, yc, T, bT, k, False, diag_cols=torch.arange(A) % N)
    loss, rowstats, st = Fn.infonce_forward(a.float().to(DEV), ya.to(DEV), contrast=c.float().to(DEV),
                                            contrast_cls=yc.to(DEV), diag_col=(torch.arange(A) % N).to(DEV),
                                            temperature=T, base_temperature=bT, topk=k)
    key, tw, G, E = Fn.topk_selection(st, A)
    sel = (o["n_ties"] > 0).numpy()                       # rows that really select (more than k negatives)
    assert np.array_equal(_key_to_float(key)[sel], o["tau"].numpy().astype(np.float32)[sel])
    assert np.array_equal(G.cpu().numpy()[sel], o["n_above"].numpy()[sel])
    assert np.array_equal(E.cpu().numpy()[sel], o["n_ties"].numpy()[sel])
    assert (key.cpu().numpy()[~sel] == 0).all() and (tw.cpu().numpy()[~sel] == 1).all()
    assert rel_err(loss.item(), o["loss"].item()) < 2e-6
    m_dev, neg_dev = rowstats[0].cpu().double(), rowstats[1].cpu().double()
    neg_ref = o["neg"] * torch.exp(o["m"] - m_dev)        # the stabiliser may differ, the product may not
    assert torch.allclose(neg_dev, neg_ref, rtol=5e-6)
    dA = Fn.infonce_backward(st, rowstats).cpu().double()
    assert (dA - o["dA"]).abs().max().item() <= 1e-5 * o["dA"].abs().max().item()


@pytest.mark.parametrize("k", [3, 50])
def test_topk_self_contrast_exact_data(k):
    A = 150
    a, _, ya, _ = _dyadic(A, 8, 32, 4, seed=k, zero_every=0)
    o = P.infonce_topk(a, ya, a, ya, 0.125, 0.25, k, True)
    loss, rowstats, st = Fn.infonce_forward(a.float().to(DEV), ya.to(DEV), temperature=0.125, base_temperature=0.25, topk=k)
    assert rel_err(loss.item(), o["loss"].item()) < 2e-6
    dA = Fn.infonce_backward(st, rowstats).cpu().double()
    assert (dA - o["dA"]).abs().max().item() <= 1e-5 * o["dA"].abs().max().item()


@pytest.mark.parametrize("k", [5, 37, 10 ** 6])
def test_topk_bank_mode_with_zero_tail(k):
    """Bank mode: the analytic zero tail (Q3) takes part in the selection; exact-zero bank rows tie with it."""
    K, M, D, A = 5, 12, 32, 90
    g = torch.Generator().manual_seed(k)
    segq = torch.randint(-3, 4, (K, M, D), generator=g).double() / 4
    pixq = torch.randint(-3, 4, (K, M, D), generator=g).double() / 4
    pixq[:, ::3] = 0
    a = torch.randint(-3, 4, (A, D), generator=g).double() / 4
    ya = torch.randint(0, K, (A,), generator=g)
    ya = ya[torch.argsort(torch.where(ya == 0, K, ya), stable=True)]     # engine row layout: class rank 1..K-1, 0
    contrast, yc = P.flatten_queue(torch.cat((segq, pixq), 1))
    o = P.infonce_topk(a, ya, contrast, yc.long(), 0.125, 0.25, k if k < 10 ** 6 else None, False)
    loss, rowstats, st = Fn.infonce_forward(a.float().to(DEV), ya.to(DEV), queues=(segq.float().to(DEV), pixq.float().to(DEV)),
                                            diag_col=torch.arange(A).to(DEV), temperature=0.125, base_temperature=0.25,
                                            topk=k)
    assert rel_err(loss.item(), o["loss"].item()) < 2e-6
    dA = Fn.infonce_backward(st, rowstats).cpu().double()
    assert (dA - o["dA"]).abs().max().item() <= 1e-5 * max(o["dA"].abs().max().item(), 1e-30)
    if k == 10 ** 6:                                      # nothing is dropped: identical to the stock sweep
        l0, rs0, st0 = Fn.infonce_forward(a.float().to(DEV), ya.to(DEV), queues=(segq.float().to(DEV), pixq.float().to(DEV)),
                                          diag_col=torch.arange(A).to(DEV), temperature=0.125, base_temperature=0.25)
        assert rel_err(loss.item(), l0.item()) < 1e-6


def test_topk_normalised_embeddings_loss():
    """Unit-norm random rows (inexact logits): the loss is insensitive to which of two near-equal negatives is taken."""
    g = torch.Generator().manual_seed(5)
    A, N, D, k = 300, 4000, 256, 64
    a = torch.nn.functional.normalize(torch.randn(A, D, generator=g), dim=1)
    c = torch.nn.functional.normalize(torch.randn(N, D, generator=g), dim=1)
    ya, yc = torch.randint(0, 19, (A,), generator=g), torch.randint(0, 19, (N,), generator=g)
    o = P.infonce_topk(a.double(), ya, c.double(), yc, 0.1, 0.07, k, False)
    loss, rowstats, st = Fn.infonce_forward(a.to(DEV), ya.to(DEV), contrast=c.to(DEV), contrast_cls=yc.to(DEV),
                                            diag_col=torch.arange(A).to(DEV), temperature=0.1, base_temperature=0.07, topk=k)
    assert rel_err(loss.item(), o["loss"].item()) < 5e-6
    key, tw, G, E = Fn.topk_selection(st, A)
    assert np.allclose(_key_to_float(key), o["tau"].numpy(), atol=2e-5)
    assert ((G + E).cpu() >= k).all() and (G.cpu() < k).all()
    dA = Fn.infonce_backward(st, rowstats).cpu().double()
    assert torch.linalg.norm(dA - o["dA"]) <= 1e-3 * torch.linalg.norm(o["dA"])


@pytest.mark.parametrize("name", ["nomem_small", "mem_small"])
def test_topk_through_the_loss_module(name):
    """contrast.topk_negatives through PixelContrastLoss on the golden inputs (injected permutations): loss and the
    dense embedding gradient against the oracle on the same anchors."""
    g = load_golden(name)
    T, bT, ms, mv, K, ign = g["params"].tolist()
    k = 5
    cfg = {"data": {"num_classes": int(K)},
           "contrast": {"temperature": T, "base_temperature": bT, "max_samples": int(ms), "max_views": int(mv),
                        "loss_weight": 0.1, "topk_negatives": k},
           "loss": {"params": {"ce_ignore_index": -1}}, "network": {"stride": 8}}
    crit = cs.PixelContrastLoss(cs.Configer(cfg))
    crit.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    queue = None
    queue_o = None
    if "segment_queue" in g:
        queue = (torch.from_numpy(g["segment_queue"]).to(DEV), torch.from_numpy(g["pixel_queue"]).to(DEV))
        queue_o = torch.cat((torch.from_numpy(g["segment_queue"]), torch.from_numpy(g["pixel_queue"])), 1)
    loss = crit(embed, torch.from_numpy(g["target"]).to(DEV), torch.from_numpy(g["predict"]).to(DEV), queue)
    loss.backward()
    e64 = torch.from_numpy(g["embed"]).double().requires_grad_(True)
    _, det = P.pixel_contrast_loss(e64, torch.from_numpy(g["target"]), torch.from_numpy(g["predict"]),
                                   temperature=T, base_temperature=bT, max_samples=int(ms), max_views=int(mv),
                                   ignore_label=int(ign), queue=queue_o,
                                   perm_fn=P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"])), return_details=True)
    lo = P.infonce_dense_topk(det["anchors"], det["ya"], det["contrast"], det["yc"], T, bT, k)
    lo.backward()
    assert rel_err(loss.item(), lo.item()) < 5e-6
    gerr = (embed.grad.cpu().double() - e64.grad).abs().max().item()
    assert gerr <= 2e-3 * e64.grad.abs().max().item()    # one near-tie swap moves one negative's share of a row


@pytest.mark.parametrize("precision,D", [("fp32", 64), ("bf16", 256)])
def test_topk_inside_the_captured_step_equals_the_eager_step(precision, D):
    """a10 wired into GraphedContrastStep: the three histogram sweeps, the scans, the weighted NEG sweep, POS, finalize and
    the top-k backward are part of the captured sequence; replay r == eager step with counter r+1 bit for bit (exact
    sweep and tensor sweep)."""
    from contrastiveseg_b200.synth import make_contrast_batch
    K = 6
    data = make_contrast_batch(B=2, D=D, h=32, w=32, num_classes=K, img_stride=4, block=16, seed=17)
    embed, tgt, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=96, max_views=8, seed=2,
                              precision=precision, num_classes=K, topk_negatives=11)
    step = cs.GraphedContrastStep(embed, tgt, seg=seg, options=opts)
    assert not step.fused
    for r in range(3):
        loss, grad = step.replay()
        torch.cuda.synchronize()
        loss, grad = loss.clone(), grad.clone()
        Fn._step_counter[0] = r
        e = embed.clone().requires_grad_(True)
        l = cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts)
        l.backward()
        torch.cuda.synchronize()
        assert torch.equal(l.detach(), loss) and torch.equal(e.grad, grad)
    opts_all = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=96, max_views=8, seed=2,
                                  precision=precision, num_classes=K)
    Fn._step_counter[0] = 2
    e = embed.clone().requires_grad_(True)
    l_all = cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts_all)
    assert l_all.item() > loss.item()                     # fewer negatives in the denominator -> smaller loss


# ---------------------------------------------------------------------------------------------------
# a10 on the tensor path: the radix select runs in the wgmma sweep's epilogue (csrc/pcl_infonce_tc.cu TC_H1..H3, TC_NEGW)
# on the fp32-accumulated logits of the bf16 operands.  Dyadic operands (multiples of 1/4, |x| <= 3/4) are exact in bf16 and
# their 256-term dot products exact in fp32, so selection state, loss and gradient must equal the oracle's like on the
# exact path; the key is in log2 units (x = s * log2(e) / T), so tau is compared through the ordering, not bitwise.
# ---------------------------------------------------------------------------------------------------
def _bf16_rows(x, rows_alloc):
    return Fn.to_bf16_rows(x.float().to(DEV), rows_alloc)


@pytest.mark.parametrize("A,N,k", [(70, 333, 9), (130, 1000, 1), (200, 600, 40), (300, 5000, 128)])
def test_tc_topk_explicit_exact_data(A, N, k):
    a, c, ya, yc = _dyadic(A, N, 256, 5, seed=A + N + k)
    order = torch.argsort(yc, stable=True)                       # the tensor sweep wants class-grouped contrast rows
    c, yc = c[order], yc[order]
    T, bT = 0.125, 0.25
    diag = torch.arange(A) % N
    o = P.infonce_topk(a, ya, c, yc, T, bT, k, False, diag_cols=diag)
    c16 = _bf16_rows(c, -(-N // 256) * 256)
    loss, rowstats, st = Fn.infonce_tc_forward(a.float().to(DEV), ya.to(DEV), contrast_bf16=c16, contrast_cls=yc.to(DEV),
                                               n_cols=N, diag_col=diag.to(DEV), temperature=T, base_temperature=bT, topk=k)
    key, tw, G, E = Fn.topk_selection(st, A)
    sel = (o["n_ties"] > 0).numpy()
    assert np.array_equal(G.cpu().numpy()[sel], o["n_above"].numpy()[sel])
    assert np.array_equal(E.cpu().numpy()[sel], o["n_ties"].numpy()[sel])
    tau_nat = _key_to_float(key) / 1.4426950408889634            # log2 units -> natural-log logit
    assert np.allclose(tau_nat[sel], o["tau"].numpy()[sel], rtol=2e-6, atol=1e-6)
    assert rel_err(loss.item(), o["loss"].item()) < 2e-5
    dA = Fn.infonce_tc_backward(st, rowstats).cpu().double()
    assert (dA - o["dA"]).abs().max().item() <= 4e-3 * o["dA"].abs().max().item()      # bf16 gradient tile


@pytest.mark.parametrize("k", [3, 50])
def test_tc_topk_self_contrast_exact_data(k):
    A = 300
    a, _, ya, _ = _dyadic(A, 8, 256, 4, seed=k, zero_every=0)
    order = torch.argsort(ya, stable=True)                       # class-grouped anchors (the engine's layout)
    a, ya = a[order], ya[order]
    o = P.infonce_topk(a, ya, a, ya, 0.125, 0.25, k, True)
    loss, rowstats, st = Fn.infonce_tc_forward(a.float().to(DEV), ya.to(DEV), temperature=0.125, base_temperature=0.25, topk=k)
    assert rel_err(loss.item(), o["loss"].item()) < 2e-5
    dA = Fn.infonce_tc_backward(st, rowstats).cpu().double()
    assert (dA - o["dA"]).abs().max().item() <= 4e-3 * o["dA"].abs().max().item()


@pytest.mark.parametrize("k", [5, 37, 10 ** 6])
def test_tc_topk_bank_mode_with_zero_tail(k):
    """Bank mode on the tensor path: the analytic zero tail takes part in the selection (scan + weighted POS prologue)."""
    from contrastiveseg_b200.bank import shadow_rows
    K, M, D, A = 5, 12, 256, 90
    g = torch.Generator().manual_seed(k)
    segq = torch.randint(-3, 4, (K, M, D), generator=g).double() / 4
    pixq = torch.randint(-3, 4, (K, M, D), generator=g).double() / 4
    pixq[:, ::3] = 0
    a = torch.randint(-3, 4, (A, D), generator=g).double() / 4
    ya = torch.randint(0, K, (A,), generator=g)
    ya = ya[torch.argsort(torch.where(ya == 0, K, ya), stable=True)]
    contrast, yc = P.flatten_queue(torch.cat((segq, pixq), 1))
    o = P.infonce_topk(a, ya, contrast, yc.long(), 0.125, 0.25, k if k < 10 ** 6 else None, False)
    shadow = torch.zeros((shadow_rows(K, M), D), dtype=torch.bfloat16, device=DEV)
    shadow[:(K - 1) * 2 * M] = contrast[:(K - 1) * 2 * M].to(torch.bfloat16).to(DEV)
    loss, rowstats, st = Fn.infonce_tc_forward(a.float().to(DEV), ya.to(DEV), bank=(shadow, K, 2 * M),
                                               diag_col=torch.arange(A).to(DEV), temperature=0.125, base_temperature=0.25,
                                               norm_bound=1.0, topk=k)     # (stabiliser only: keeps exp2 in range)
    assert rel_err(loss.item(), o["loss"].item()) < 2e-5
    dA = Fn.infonce_tc_backward(st, rowstats).cpu().double()
    assert (dA - o["dA"]).abs().max().item() <= 4e-3 * max(o["dA"].abs().max().item(), 1e-30)


@pytest.mark.parametrize("name", ["nomem_d256", "mem_d256"])
def test_tc_topk_through_the_loss_module(name):
    """contrast.topk_negatives with contrast.precision = 'bf16' through PixelContrastLoss on the D = 256 goldens: loss
    and dense gradient against the oracle's top-k on the bf16-rounded operands (same anchors)."""
    g = load_golden(name)
    T, bT, ms, mv, K, ign = g["params"].tolist()
    k = 7
    cfg = {"data": {"num_classes": int(K)},
           "contrast": {"temperature": T, "base_temperature": bT, "max_samples": int(ms), "max_views": int(mv),
                        "loss_weight": 0.1, "topk_negatives": k, "precision": "bf16"},
           "loss": {"params": {"ce_ignore_index": -1}}, "network": {"stride": 8}}
    crit = cs.PixelContrastLoss(cs.Configer(cfg))
    crit.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    queue = queue_o = None
    if "segment_queue" in g:
        queue = (torch.from_numpy(g["segment_queue"]).to(DEV), torch.from_numpy(g["pixel_queue"]).to(DEV))
        queue_o = torch.cat((torch.from_numpy(g["segment_queue"]), torch.from_numpy(g["pixel_queue"])), 1)
    loss = crit(embed, torch.from_numpy(g["target"]).to(DEV), torch.from_numpy(g["predict"]).to(DEV), queue)
    loss.backward()
    bf = lambda x: x.to(torch.bfloat16).double()
    e64 = torch.from_numpy(g["embed"]).double()
    _, det = P.pixel_contrast_loss(e64, torch.from_numpy(g["target"]), torch.from_numpy(g["predict"]),
                                   temperature=T, base_temperature=bT, max_samples=int(ms), max_views=int(mv),
                                   ignore_label=int(ign), queue=queue_o,
                                   perm_fn=P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"])), return_details=True)
    anchors = bf(det["anchors"]).requires_grad_(True)
    contrast = anchors if queue_o is None else bf(det["contrast"])
    lo = P.infonce_dense_topk(anchors, det["ya"], contrast, det["yc"], T, bT, k)
    lo.backward()
    assert rel_err(loss.item(), lo.item()) < 1e-4
    # gradient rows of the sampled pixels, in the oracle's (view-major) row order
    B, D, h, w = g["embed"].shape
    flat = embed.grad.permute(0, 2, 3, 1).reshape(B, h * w, D).cpu().double()
    TC, V = det["idx"].shape
    rows = torch.stack([flat[int(det["img"][t]), int(det["idx"][t, v])] for v in range(V) for t in range(TC)])
    assert (rows - anchors.grad).abs().max().item() <= 6e-3 * anchors.grad.abs().max().item()
