"""GPU parity tests: the CUDA path (through the C ABI) against the oracle and the reference-generated golden
vectors.  Tolerances (fp32 exact path): loss <= 2e-6 relative to the float64 oracle and <= 1e-5 relative to the
fp32 reference golden (north_star bar: 1e-4); gradient <= 1e-5 * max|g|; sampled anchors and bank pointers
bit-exact; bank rows <= 1.5e-7 abs (2 ulp: the L2 norm is summed in a different order), bank segment means 1e-6
(fp32 sums in the reference, exact integer accumulation here)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import functional as Fn
from oracle import ref_port as P
from helpers import load_golden, unpack_perms, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

LOSS_CASES = ["nomem_small", "nomem_oddv", "nomem_mv1", "nomem_nondiv", "nomem_d256", "mem_small", "mem_d256"]


def _cfg(T, bT, ms, mv, K, extra=None):
    d = {"data": {"num_classes": int(K)},
         "contrast": {"temperature": T, "base_temperature": bT, "max_samples": int(ms), "max_views": int(mv),
                      "loss_weight": 0.1, "use_rmi": False, "use_lovasz": False},
         "loss": {"params": {"ce_ignore_index": -1, "ce_reduction": "elementwise_mean"}},
         "network": {"stride": 8}}
    if extra:
        d["contrast"].update(extra)
    return cs.Configer(d)


def _oracle(g, dtype=torch.float64):
    T, bT, ms, mv, K, ign = g["params"].tolist()
    embed = torch.from_numpy(g["embed"]).to(dtype).requires_grad_(True)
    queue = None
    if "segment_queue" in g:
        queue = torch.cat((torch.from_numpy(g["segment_queue"]), torch.from_numpy(g["pixel_queue"])), 1)
    loss, det = P.pixel_contrast_loss(embed, torch.from_numpy(g["target"]), torch.from_numpy(g["predict"]),
                                      temperature=T, base_temperature=bT, max_samples=int(ms), max_views=int(mv),
                                      ignore_label=int(ign), queue=queue,
                                      perm_fn=P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"])),
                                      return_details=True)
    loss.backward()
    return loss.item(), embed.grad, det


@pytest.mark.parametrize("name", LOSS_CASES)
def test_loss_and_grad_match_reference(name):
    g = load_golden(name)
    T, bT, ms, mv, K, ign = g["params"].tolist()
    crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K))
    crit.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    target = torch.from_numpy(g["target"]).to(DEV)
    predict = torch.from_numpy(g["predict"]).to(DEV)
    queue = None
    if "segment_queue" in g:
        queue = (torch.from_numpy(g["segment_queue"]).to(DEV), torch.from_numpy(g["pixel_queue"]).to(DEV))
    loss = crit(embed, target, predict, queue)
    loss.backward()
    torch.cuda.synchronize()
    o_loss, o_grad, det = _oracle(g)
    assert rel_err(loss.item(), o_loss) < 2e-6, (loss.item(), o_loss)
    assert rel_err(loss.item(), g["loss"]) < 1e-5
    gmax = o_grad.abs().max().item()
    assert (embed.grad.cpu().double() - o_grad).abs().max().item() <= 1e-5 * gmax
    assert (embed.grad.cpu() - torch.from_numpy(g["grad_embed"])).abs().max().item() <= 1e-5 * gmax
    # the sampled anchors are the reference's, bit for bit
    ws = Fn.last_workspace(embed.device)
    hdr = ws.plan_header()
    TC, V, A = hdr[0], hdr[1], hdr[2]
    assert (TC, V) == tuple(g["X_"].shape[:2])
    meta = ws.anchor_meta.view(4, -1)[:, :A].cpu()
    ref_rows = meta[3].long()
    X = torch.zeros((A, g["X_"].shape[2]))
    X[ref_rows] = ws.anchors_f32[:A].cpu()
    X_ = X.view(V, TC, -1).permute(1, 0, 2)
    assert torch.equal(X_, torch.from_numpy(g["X_"]))
    cls_by_ref = torch.zeros(A, dtype=torch.long)
    cls_by_ref[ref_rows] = meta[2].long()
    assert torch.equal(cls_by_ref[:TC].float(), torch.from_numpy(g["y_"]))


@pytest.mark.parametrize("name", ["mem_small"])
def test_concatenated_queue_tensor_is_accepted(name):
    g = load_golden(name)
    T, bT, ms, mv, K, ign = g["params"].tolist()
    crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K))
    crit.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    queue = torch.cat((torch.from_numpy(g["segment_queue"]), torch.from_numpy(g["pixel_queue"])), 1).to(DEV)
    loss = crit(torch.from_numpy(g["embed"]).to(DEV), torch.from_numpy(g["target"]).to(DEV),
                torch.from_numpy(g["predict"]).to(DEV), queue)
    assert rel_err(loss.item(), g["loss"]) < 1e-5


@pytest.mark.parametrize("name,mem", [("wrapper_nomem_embed", False), ("wrapper_nomem_warmup", False),
                                      ("wrapper_mem_embed", True)])
def test_contrast_ce_wrapper(name, mem):
    g = load_golden(name)
    T, bT, ms, mv, K, ign, lw, with_embed, _ = g["params"].tolist()
    cfg = _cfg(T, bT, ms, mv, K, {"loss_weight": lw})
    crit = (cs.MemContrastCELoss if mem else cs.ContrastCELoss)(cfg).to(DEV)
    crit.contrast_criterion.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    seg = torch.from_numpy(g["seg"]).to(DEV).requires_grad_(True)
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    preds = {"seg": seg, "embed": embed}
    if mem:
        preds["segment_queue"] = torch.from_numpy(g["segment_queue"]).to(DEV)
        preds["pixel_queue"] = torch.from_numpy(g["pixel_queue"]).to(DEV)
    loss = crit(preds, torch.from_numpy(g["target"]).to(DEV), with_embed=bool(with_embed))
    loss.backward()
    assert rel_err(loss.item(), g["loss"]) < 1e-5
    assert torch.allclose(seg.grad.cpu(), torch.from_numpy(g["grad_seg"]), rtol=1e-4, atol=1e-7)
    gref = torch.from_numpy(g["grad_embed"])
    assert (embed.grad.cpu() - gref).abs().max().item() <= 1e-5 * max(gref.abs().max().item(), 1e-12) + 1e-12


@pytest.mark.parametrize("name", ["wrapper_aux_embed", "wrapper_aux_warmup_weighted"])
@pytest.mark.parametrize("fused", [True, False])
def test_contrast_auxce_wrapper(name, fused):
    """ContrastAuxCELoss (lib/loss/loss_contrast.py:192-234, registry key 'contrast_auxce_loss': the class the DeepLab
    and HRNet-OCR contrast scripts select) against goldens produced by the unmodified reference: loss 1e-5, all three
    gradients; with the fused up-sample + CE kernels (default) and with the PyTorch seg-CE ops."""
    g = load_golden(name)
    T, bT, ms, mv, K, ign, lw, with_embed, w_seg, w_aux = g["params"].tolist()
    cfg = _cfg(T, bT, ms, mv, K, {"loss_weight": lw, "fused_seg_ce": fused})
    cfg.add(["network", "loss_weights"], {"seg_loss": w_seg, "aux_loss": w_aux})
    if g["ce_weight"].size:
        params = dict(cfg.get("loss", "params")); params["ce_weight"] = g["ce_weight"].tolist()
        cfg.add(["loss", "params"], params)
    crit = cs.get_seg_loss(cfg, "contrast_auxce_loss").to(DEV)
    assert isinstance(crit, cs.ContrastAuxCELoss)
    crit.contrast_criterion.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    seg = torch.from_numpy(g["seg"]).to(DEV).requires_grad_(True)
    seg_aux = torch.from_numpy(g["seg_aux"]).to(DEV).requires_grad_(True)
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    loss = crit({"seg": seg, "seg_aux": seg_aux, "embed": embed}, torch.from_numpy(g["target"]).to(DEV),
                with_embed=bool(with_embed))
    loss.backward()
    assert rel_err(loss.item(), g["loss"]) < 1e-5
    for got, key in ((seg.grad, "grad_seg"), (seg_aux.grad, "grad_seg_aux")):
        assert torch.allclose(got.cpu(), torch.from_numpy(g[key]), rtol=1e-4, atol=1e-7), key
    gref = torch.from_numpy(g["grad_embed"])
    assert (embed.grad.cpu() - gref).abs().max().item() <= 1e-5 * max(gref.abs().max().item(), 1e-12) + 1e-12


@pytest.mark.parametrize("name", ["enqueue_aligned", "enqueue_q6"])
def test_bank_enqueue_matches_reference(name):
    g = load_golden(name)
    net_stride, M, Fq, steps, K = g["params"].tolist()
    sq, pq = torch.from_numpy(g["sq0"]).to(DEV), torch.from_numpy(g["pq0"]).to(DEV)
    sp = torch.zeros(K, dtype=torch.long, device=DEV)
    pp = torch.zeros(K, dtype=torch.long, device=DEV)
    for s in range(steps):
        replay = P.PermReplay(unpack_perms(g[f"perm_flat{s}"], g[f"perm_lens{s}"]))
        cs.dequeue_and_enqueue(torch.from_numpy(g[f"keys{s}"]).to(DEV), torch.from_numpy(g[f"labels{s}"]).to(DEV),
                               sq, sp, pq, pp, network_stride=net_stride, memory_size=M, pixel_update_freq=Fq,
                               perm_fn=replay)
        assert replay.pos == len(replay.draws)
        assert torch.equal(sp.cpu(), torch.from_numpy(g[f"sp{s + 1}"]))
        assert torch.equal(pp.cpu(), torch.from_numpy(g[f"pp{s + 1}"]))
        # rows are the reference's rows up to the rounding of the L2 norm (summation order): <= 2 ulp of 0.5
        assert (pq.cpu() - torch.from_numpy(g[f"pq{s + 1}"])).abs().max().item() <= 1.5e-7
        assert (sq.cpu() - torch.from_numpy(g[f"sq{s + 1}"])).abs().max().item() <= 1e-6


def test_bank_enqueue_shape_error_like_reference():
    # label grid larger than the feature map: the reference raises an index error, the engine PCL_ERR_SHAPE
    bank = cs.MemoryBank(4, 8, 32).to(DEV)
    keys = torch.randn(1, 32, 4, 4, device=DEV)
    labels = torch.ones(1, 32, 32, dtype=torch.long, device=DEV)
    with pytest.raises(Exception):
        bank.enqueue(keys, labels, network_stride=2, pixel_update_freq=2)


@pytest.mark.parametrize("shape", [(2, 256, 16, 32), (1, 32, 7, 9), (3, 320, 5, 8)])
def test_l2_normalize_matches_torch(shape):
    torch.manual_seed(0)
    x = torch.randn(shape, device=DEV, requires_grad=True)
    y = cs.l2_normalize(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    x2 = x.detach().clone().requires_grad_(True)
    y2 = F.normalize(x2, p=2, dim=1)
    y2.backward(gy)
    assert torch.allclose(y, y2, rtol=1e-6, atol=1e-7)
    assert torch.allclose(x.grad, x2.grad, rtol=1e-5, atol=1e-6)


def test_fused_normalize_path_equals_normalise_then_loss():
    """normalize=True: raw projection in, only the sampled columns are normalised; gradient is w.r.t. raw."""
    g = load_golden("nomem_small")
    T, bT, ms, mv, K, ign = g["params"].tolist()
    torch.manual_seed(1)
    raw = torch.randn(g["embed"].shape, device=DEV) * 3.0
    target = torch.from_numpy(g["target"]).to(DEV)
    predict = torch.from_numpy(g["predict"]).to(DEV)
    perms = []
    rec = P.PermRecorder(torch.Generator().manual_seed(5))
    crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K))
    crit.perm_fn = rec
    r1 = raw.clone().requires_grad_(True)
    l1 = crit(r1, target, predict, normalize=True)
    l1.backward()
    crit.perm_fn = P.PermReplay(rec.draws)
    r2 = raw.clone().requires_grad_(True)
    l2 = crit(F.normalize(r2, p=2, dim=1), target, predict)
    l2.backward()
    assert rel_err(l1.item(), l2.item()) < 1e-6
    assert (r1.grad - r2.grad).abs().max().item() <= 1e-5 * r2.grad.abs().max().item()


def _check_device_sampling(ws, lab, prd, ms, mv):
    hdr = ws.plan_header()
    TC, V, A = hdr[0], hdr[1], hdr[2]
    meta = ws.anchor_meta.view(4, -1)[:, :A].cpu().long()
    pix, img, cls, ref = meta
    # rows are a permutation of the reference rows, every (image,class) pair has V distinct pixels of its class
    assert sorted(ref.tolist()) == list(range(A))
    B = lab.shape[0]
    kept = [(b, c) for b in range(B) for c in P.kept_classes(lab[b], -1, mv)]
    assert TC == len(kept) and V == min(ms // TC, mv)
    for t, (b, c) in enumerate(kept):
        rows = ((ref % TC) == t).nonzero()[:, 0]
        assert rows.numel() == V
        assert (img[rows] == b).all() and (cls[rows] == c).all()
        px = pix[rows]
        assert px.unique().numel() == V
        assert (lab[b][px] == c).all()
        nh = int(((lab[b] == c) & (prd[b] != c)).sum()); ne = int(((lab[b] == c) & (prd[b] == c)).sum())
        kh, ke = P.split_hard_easy(nh, ne, V)
        assert int((prd[b][px] != c).sum()) == kh and int((prd[b][px] == c).sum()) == ke
    return TC, V, A, meta


@pytest.mark.parametrize("mem", [False, True])
def test_device_rng_sampling_is_valid_and_loss_matches_oracle_on_same_indices(mem):
    from contrastiveseg_b200.synth import make_bank, make_contrast_batch
    K, D, ms, mv = 7, 64, 200, 12
    data = make_contrast_batch(B=3, D=D, h=24, w=40, num_classes=K, img_stride=4, block=16, seed=77)
    bank = make_bank(K, 30, D, 78)
    crit = cs.PixelContrastLoss(_cfg(0.1, 0.07, ms, mv, K))
    embed = data["embed"].to(DEV).requires_grad_(True)
    queue = (bank["segment_queue"].to(DEV), bank["pixel_queue"].to(DEV)) if mem else None
    loss = crit(embed, data["target"].to(DEV), seg=data["seg"].to(DEV), queue=queue)
    loss.backward()
    ws = Fn.last_workspace(embed.device)
    lab = P.downsample_labels(data["target"], 24, 40).reshape(3, -1)
    prd = data["seg"].argmax(1).reshape(3, -1)
    TC, V, A, meta = _check_device_sampling(ws, lab, prd, ms, mv)
    pix, img, cls, ref = meta
    # oracle on exactly these anchors (reference row order)
    X = data["embed"].permute(0, 2, 3, 1).reshape(3, -1, D).double()
    anchors = torch.zeros((A, D), dtype=torch.float64)
    ya = torch.zeros(A, dtype=torch.long)
    anchors[ref] = X[img, pix]
    ya[ref] = cls
    a = anchors.clone().requires_grad_(True)
    if mem:
        contrast, yc = P.flatten_queue(torch.cat((bank["segment_queue"], bank["pixel_queue"]), 1).double())
        lo = P.infonce_dense(a, ya.double(), contrast, yc, 0.1, 0.07)
    else:
        lo = P.infonce_dense(a, ya.double(), a, ya.double(), 0.1, 0.07)
    lo.backward()
    assert rel_err(loss.item(), lo.item()) < 2e-6
    gd = torch.zeros(3, 24 * 40, D, dtype=torch.float64)
    gd[img, pix] = a.grad[ref]
    gd = gd.view(3, 24, 40, D).permute(0, 3, 1, 2)
    assert (embed.grad.cpu().double() - gd).abs().max().item() <= 1e-5 * gd.abs().max().item()


def test_device_rng_changes_between_steps_and_is_seed_reproducible():
    from contrastiveseg_b200.synth import make_contrast_batch
    data = make_contrast_batch(B=2, D=32, h=24, w=24, num_classes=5, img_stride=2, block=8, seed=9)
    crit = cs.PixelContrastLoss(_cfg(0.1, 0.07, 40, 6, 5))
    e = data["embed"].to(DEV)
    t, s = data["target"].to(DEV), data["seg"].to(DEV)
    crit(e, t, seg=s)
    ws = Fn.last_workspace(e.device)
    p1 = ws.anchor_meta.view(4, -1)[0].clone()
    crit(e, t, seg=s)
    p2 = ws.anchor_meta.view(4, -1)[0].clone()
    assert not torch.equal(p1, p2)


def test_explicit_infonce_modes_and_nan_semantics():
    from contrastiveseg_b200.synth import make_sweep_point
    pt = make_sweep_point(200, 700, D=64, num_classes=6, seed=3, clustered=0.5)
    a, ya, c, yc = pt["anchors"], pt["ya"], pt["contrast"], pt["yc"]
    diag = torch.arange(200)
    loss, st, state = Fn.infonce_forward(a.to(DEV), ya.to(DEV), contrast=c.to(DEV), contrast_cls=yc.to(DEV),
                                         diag_col=diag.to(DEV), temperature=0.07, base_temperature=0.07)
    dA = Fn.infonce_backward(state, st)
    cf = P.infonce_closed_form(a.double(), ya, c.double(), yc, 0.07, 0.07, self_contrast=False)
    assert rel_err(loss.item(), cf["loss"].item()) < 2e-6
    assert (dA.cpu().double() - cf["dA"]).abs().max().item() <= 1e-5 * cf["dA"].abs().max().item()
    assert torch.allclose(st[4].cpu().double(), cf["npos"])
    # self-contrast
    loss, st, state = Fn.infonce_forward(a.to(DEV), ya.to(DEV), temperature=0.1, base_temperature=0.07)
    dA = Fn.infonce_backward(state, st)
    cf = P.infonce_closed_form(a.double(), ya, a.double(), ya, 0.1, 0.07, self_contrast=True)
    assert rel_err(loss.item(), cf["loss"].item()) < 2e-6
    assert (dA.cpu().double() - cf["dA"]).abs().max().item() <= 1e-5 * cf["dA"].abs().max().item()
    # a row without positives: NaN like the reference (Q8), 0 with nan_safe
    ya2 = ya.clone(); ya2[0] = 17
    loss, _, _ = Fn.infonce_forward(a.to(DEV), ya2.to(DEV), contrast=c.to(DEV), contrast_cls=yc.to(DEV),
                                    temperature=0.1, base_temperature=0.07)
    assert torch.isnan(loss).item()
    loss, _, _ = Fn.infonce_forward(a.to(DEV), ya2.to(DEV), contrast=c.to(DEV), contrast_cls=yc.to(DEV),
                                    temperature=0.1, base_temperature=0.07, nan_safe=True)
    assert torch.isfinite(loss).item()


def test_empty_inputs_give_zero_loss_not_a_crash():
    # no class qualifies (everything ignored): the reference crashes (Q8); the engine returns 0 with a zero gradient
    crit = cs.PixelContrastLoss(_cfg(0.1, 0.07, 64, 4, 5))
    embed = F.normalize(torch.randn(2, 32, 8, 8, device=DEV), dim=1).requires_grad_(True)
    target = torch.full((2, 16, 16), -1, dtype=torch.long, device=DEV)
    loss = crit(embed, target, predict=torch.zeros(2, 8, 8, dtype=torch.long, device=DEV))
    loss.backward()
    assert loss.item() == 0.0 and embed.grad.abs().max().item() == 0.0


def test_full_size_cityscapes_batch_properties():
    """BASELINE config 2 (B=8, 256x128x256 embedding, 19 classes): size-independent checks — every anchor row is a
    valid distinct pixel of its class, loss equals the float64 oracle on the same anchors, the dense gradient is zero
    outside the sampled columns and sums to the per-anchor gradients."""
    from contrastiveseg_b200.synth import make_contrast_batch
    data = make_contrast_batch(B=8, D=256, h=128, w=256, num_classes=19, img_stride=4, block=32, seed=304)
    crit = cs.PixelContrastLoss(_cfg(0.1, 0.07, 1024, 100, 19))
    embed = data["embed"].to(DEV).requires_grad_(True)
    loss = crit(embed, data["target"].to(DEV), seg=data["seg"].to(DEV))
    loss.backward()
    ws = Fn.last_workspace(embed.device)
    lab = P.downsample_labels(data["target"], 128, 256).reshape(8, -1)
    prd = data["seg"].argmax(1).reshape(8, -1)
    TC, V, A, meta = _check_device_sampling(ws, lab, prd, 1024, 100)
    pix, img, cls, ref = meta
    X = data["embed"].permute(0, 2, 3, 1).reshape(8, -1, 256)
    anchors = torch.zeros((A, 256), dtype=torch.float64)
    ya = torch.zeros(A, dtype=torch.long)
    anchors[ref] = X[img, pix].double()
    ya[ref] = cls
    cf = P.infonce_closed_form(anchors, ya, anchors, ya, 0.1, 0.07, self_contrast=True)
    assert rel_err(loss.item(), cf["loss"].item()) < 2e-6
    g = embed.grad
    nz = (g != 0).any(dim=1).sum().item()
    assert nz <= A and nz >= A - 2
    got = g.permute(0, 2, 3, 1).reshape(8, -1, 256)[img.to(DEV), pix.to(DEV)].cpu().double()
    assert (got - cf["dA"][ref]).abs().max().item() <= 1e-5 * cf["dA"].abs().max().item()
    assert abs(g.double().sum().item() - cf["dA"].sum().item()) <= 1e-4 * cf["dA"].abs().sum().item()


# ---------------------------------------------------------------------------------------------------
# tensor-core (wgmma) path.  Tolerances: loss <= 2e-5 relative to the float64 oracle on the bf16-ROUNDED
# operands (fp32 accumulate + ex2/lg2.approx), <= 1e-4 relative to the fp32-operand oracle (north_star bar).
# ---------------------------------------------------------------------------------------------------
def _bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


@pytest.mark.parametrize("A,N", [(128, 256), (200, 1000), (512, 4096)])
def test_tc_pipeline_raw_logits(A, N):
    from contrastiveseg_b200.synth import make_sweep_point
    pt = make_sweep_point(A, N, D=256, seed=A + N)
    a, c = pt["anchors"].to(DEV), pt["contrast"].to(DEV)
    c16 = Fn.to_bf16_rows(c, -(-N // 256) * 256)
    S = Fn.tc_dump_logits(a, c16, N)
    ref = _bf(a).double() @ _bf(c).double().t()
    assert (S.double() - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("A,N,T,self_mode", [(200, 1000, 0.1, False), (912, 912, 0.1, True), (1024, 20000, 0.07, False)])
def test_tc_forward_matches_oracle(A, N, T, self_mode):
    from contrastiveseg_b200.synth import make_sweep_point
    pt = make_sweep_point(A, N, D=256, num_classes=19, seed=A * 7 + N, clustered=0.5)
    a, ya, c, yc = pt["anchors"], pt["ya"], pt["contrast"], pt["yc"]
    if self_mode:
        loss, st, _ = Fn.infonce_tc_forward(a.to(DEV), ya.to(DEV), temperature=T, base_temperature=0.07)
        cf16 = P.infonce_closed_form(_bf(a).double(), ya, _bf(a).double(), ya, T, 0.07, self_contrast=True)
        cf32 = P.infonce_closed_form(a.double(), ya, a.double(), ya, T, 0.07, self_contrast=True)
    else:
        c16 = Fn.to_bf16_rows(c.to(DEV), -(-N // 256) * 256)
        loss, st, _ = Fn.infonce_tc_forward(a.to(DEV), ya.to(DEV), contrast_bf16=c16, contrast_cls=yc.to(DEV), n_cols=N,
                                            diag_col=torch.arange(A).to(DEV), temperature=T, base_temperature=0.07)
        cf16 = P.infonce_closed_form(_bf(a).double(), ya, _bf(c).double(), yc, T, 0.07, self_contrast=False)
        cf32 = P.infonce_closed_form(a.double(), ya, c.double(), yc, T, 0.07, self_contrast=False)
    assert torch.equal(st[4].cpu().double(), cf16["npos"])
    assert rel_err(loss.item(), cf16["loss"].item()) < 2e-5
    assert rel_err(loss.item(), cf32["loss"].item()) < 1e-4


@pytest.mark.parametrize("A,N,T,self_mode", [(200, 1000, 0.1, False), (912, 912, 0.1, True), (1024, 20000, 0.07, False)])
def test_tc_backward_matches_oracle(A, N, T, self_mode):
    """Gradient tolerance of the bf16 path: max-abs 4e-3 * max|g|, relative Frobenius 2e-3 (bf16 operands perturb
    the logits by ~3e-3 at T = 0.07, and the gradient tile G is bf16; measured 1.2e-3 .. 2.5e-3, SURVEY §8c)."""
    from contrastiveseg_b200.synth import make_sweep_point
    pt = make_sweep_point(A, N, D=256, num_classes=19, seed=A * 3 + N, clustered=0.5)
    a, ya, c, yc = pt["anchors"], pt["ya"], pt["contrast"], pt["yc"]
    if self_mode:
        loss, st, state = Fn.infonce_tc_forward(a.to(DEV), ya.to(DEV), temperature=T, base_temperature=0.07)
        cf = P.infonce_closed_form(a.double(), ya, a.double(), ya, T, 0.07, self_contrast=True)
    else:
        c16 = Fn.to_bf16_rows(c.to(DEV), -(-N // 256) * 256)
        loss, st, state = Fn.infonce_tc_forward(a.to(DEV), ya.to(DEV), contrast_bf16=c16, contrast_cls=yc.to(DEV), n_cols=N,
                                                diag_col=torch.arange(A).to(DEV), temperature=T, base_temperature=0.07)
        cf = P.infonce_closed_form(a.double(), ya, c.double(), yc, T, 0.07, self_contrast=False)
    dA = Fn.infonce_tc_backward(state, st).cpu().double()
    assert (dA - cf["dA"]).abs().max().item() <= 4e-3 * cf["dA"].abs().max().item()
    assert ((dA - cf["dA"]).norm() / cf["dA"].norm()).item() < 2e-3


@pytest.mark.parametrize("name", ["nomem_d256", "mem_d256"])
def test_loss_module_on_tensor_path(name):
    """precision='bf16' through the drop-in module (golden D=256 cases): loss <= 1e-4 rel (north_star bar), gradient
    <= 4e-3 * max|g|; the bank is read through the bf16 shadow."""
    g = load_golden(name)
    T, bT, ms, mv, K, ign = g["params"].tolist()
    crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K, {"precision": "bf16"}))
    crit.perm_fn = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    queue = None
    if "segment_queue" in g:
        queue = (torch.from_numpy(g["segment_queue"]).to(DEV), torch.from_numpy(g["pixel_queue"]).to(DEV))
    loss = crit(embed, torch.from_numpy(g["target"]).to(DEV), torch.from_numpy(g["predict"]).to(DEV), queue)
    loss.backward()
    assert rel_err(loss.item(), g["loss"]) < 1e-4
    gref = torch.from_numpy(g["grad_embed"])
    assert (embed.grad.cpu() - gref).abs().max().item() <= 4e-3 * gref.abs().max().item()


def test_bank_shadow_tracks_enqueue_and_tensor_path_uses_it():
    from contrastiveseg_b200.synth import make_contrast_batch
    K, D, M = 6, 256, 64
    bank = cs.MemoryBank(K, M, D, with_shadow=True).to(DEV)
    data = make_contrast_batch(B=2, D=D, h=16, w=32, num_classes=K, img_stride=4, block=16, seed=5)
    bank.sync_shadow()
    for _ in range(3):
        bank.enqueue(data["embed"].to(DEV), data["target"].to(DEV), network_stride=4, pixel_update_freq=5)
    # the incrementally maintained shadow equals a full rebuild
    inc = bank.shadow.clone()
    full = bank.sync_shadow().clone()
    assert torch.equal(inc, full)
    rows = torch.cat((bank.segment_queue[1:], bank.pixel_queue[1:]), dim=1).reshape(-1, D)
    assert torch.equal(full[: rows.shape[0]].float(), rows.to(torch.bfloat16).float())
    # loss through the hook-style dict: exact path vs tensor path on the same samples
    rec = P.PermRecorder(torch.Generator().manual_seed(2))
    c32 = cs.PixelContrastLoss(_cfg(0.07, 0.07, 128, 8, K))
    c32.perm_fn = rec
    l32 = c32(data["embed"].to(DEV), data["target"].to(DEV), seg=data["seg"].to(DEV),
              queue=(bank.segment_queue, bank.pixel_queue))
    c16 = cs.PixelContrastLoss(_cfg(0.07, 0.07, 128, 8, K, {"precision": "bf16"}))
    c16.perm_fn = P.PermReplay(rec.draws)
    l16 = c16(data["embed"].to(DEV), data["target"].to(DEV), seg=data["seg"].to(DEV),
              queue=(bank.segment_queue, bank.pixel_queue), bank_shadow=bank.shadow)
    assert rel_err(l16.item(), l32.item()) < 1e-4


@pytest.mark.parametrize("K,M,A,seed", [(5, 300, 200, 1), (7, 200, 333, 2), (12, 70, 150, 3), (3, 500, 100, 4), (40, 130, 260, 5),
                                         (171, 8, 400, 6)])
def test_tensor_path_bank_positives_by_class_blocks(K, M, A, seed):
    """The transposed POS sweep of the bank mode (csrc/pcl_infonce_tc.cu k_tc_pos_t): anchor blocks of one class x that
    class's bank columns, tile units dealt evenly to the CTAs.  Sizes where a class has several column tiles (so a block
    is cut into several partial slots), several 64-anchor blocks, class-0 anchors (no columns: analytic zero tail) and
    more blocks than a class has tiles.  Loss and positive counts vs the float64 closed form on the bf16-rounded
    operands (loss_contrast_mem.py:107-152), gradient within the bf16 tolerance of the path."""
    from contrastiveseg_b200 import _abi
    from contrastiveseg_b200.bank import shadow_rows
    lib = _abi.load()
    g = torch.Generator().manual_seed(seed)
    ya = torch.randint(0, K, (A,), generator=g)
    ya = ya[torch.argsort(torch.where(ya == 0, K, ya), stable=True)]           # class-rank order: 1..K-1, 0
    a = F.normalize(torch.randn(A, 256, generator=g), dim=1)
    segq = F.normalize(torch.randn(K, M, 256, generator=g), dim=2)
    pixq = F.normalize(torch.randn(K, M, 256, generator=g), dim=2)
    shadow = torch.empty((shadow_rows(K, M), 256), dtype=torch.bfloat16, device=DEV)
    segq_d, pixq_d = segq.to(DEV), pixq.to(DEV)
    _abi.check(lib.pcl_bank_shadow_rebuild(segq_d.data_ptr(), pixq_d.data_ptr(), K, M, 256, shadow.data_ptr(), None))
    torch.cuda.synchronize()
    loss, st, state = Fn.infonce_tc_forward(a.to(DEV), ya.to(DEV), bank=(shadow, K, 2 * M), diag_col=torch.arange(A).to(DEV),
                                            temperature=0.1, base_temperature=0.07)
    dA = Fn.infonce_tc_backward(state, st).double().cpu()
    contrast, yc = P.flatten_queue(torch.cat((_bf(segq), _bf(pixq)), 1).double())
    cf = P.infonce_closed_form(_bf(a).double(), ya, contrast, yc.long(), 0.1, 0.07, self_contrast=False)
    assert torch.equal(st[4].double().cpu(), cf["npos"])
    assert abs(loss.item() - cf["loss"].item()) <= 5e-5 * abs(cf["loss"].item())
    gmax = cf["dA"].abs().max().item()
    assert (dA - cf["dA"]).abs().max().item() <= 6e-3 * gmax


def test_torch_cpu_rng_mode_draws_the_reference_stream():
    """rng='torch_cpu': same torch CPU seed -> the engine samples exactly what the reference code path samples."""
    g = load_golden("nomem_small")
    T, bT, ms, mv, K, ign = g["params"].tolist()
    embed = torch.from_numpy(g["embed"])
    target, predict = torch.from_numpy(g["target"]), torch.from_numpy(g["predict"])
    torch.manual_seed(1234)
    e1 = embed.clone().double().requires_grad_(True)
    ref = P.pixel_contrast_loss(e1, target, predict, temperature=T, base_temperature=bT, max_samples=int(ms),
                                max_views=int(mv))                       # draws torch.randperm like the reference
    crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K, {"rng": "torch_cpu"}))
    torch.manual_seed(1234)
    loss = crit(embed.to(DEV), target.to(DEV), predict.to(DEV))
    assert rel_err(loss.item(), ref.item()) < 2e-6


def test_trainer_hook_end_to_end_with_bank():
    """C1-style plumbing: a small stand-in network ({'seg','embed','key','lb_key'} contract of hrnet.py:183-188),
    the drop-in loss + bank through ContrastTrainerHook, SGD steps; first-step loss equals the oracle port."""
    import torch.nn as nn
    torch.manual_seed(0)
    K, D = 5, 32

    class TinyNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.body = nn.Sequential(nn.Conv2d(3, 16, 3, stride=2, padding=1), nn.ReLU(),
                                      nn.Conv2d(16, 24, 3, stride=2, padding=1), nn.ReLU())
            self.cls = nn.Conv2d(24, K, 1)
            self.proj = cs.ProjectionHead(24, D, proj="convmlp", bn_type="torchbn")

        def forward(self, x, targets):
            f = self.body(x)
            emb = self.proj(f)
            return {"seg": self.cls(f), "embed": emb, "key": emb.detach(), "lb_key": targets}

    cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": 4},
                       "loss": {"loss_type": "mem_contrast_ce_loss", "params": {"ce_ignore_index": -1}},
                       "contrast": {"temperature": 0.07, "base_temperature": 0.07, "max_samples": 64, "max_views": 4,
                                    "loss_weight": 0.1, "use_rmi": False, "use_lovasz": False, "warmup_iters": 1,
                                    "with_memory": True, "memory_size": 16, "pixel_update_freq": 3}})
    net = TinyNet().to(DEV)
    bank = cs.MemoryBank(K, 16, D).to(DEV)
    hook = cs.ContrastTrainerHook(cfg, bank)
    opt = torch.optim.SGD(net.parameters(), lr=0.01)
    x = torch.randn(2, 3, 64, 64, device=DEV)
    from contrastiveseg_b200.synth import block_label_map
    tgt = block_label_map(2, 64, 64, 16, K, torch.Generator().manual_seed(3)).to(DEV)
    ptr0 = bank.pixel_queue_ptr.clone()
    losses = []
    for it in range(3):
        out = net(x, tgt)
        if it == 1:          # compare the loss value of one post-warm-up step with the oracle on the same samples
            rec = P.PermRecorder(torch.Generator().manual_seed(9))
            hook.pixel_loss.contrast_criterion.perm_fn = rec
            sq, pq = bank.segment_queue.clone().cpu(), bank.pixel_queue.clone().cpu()
        loss = hook.loss_step(out, tgt, iters=it)
        if it == 1:
            hook.pixel_loss.contrast_criterion.perm_fn = None
            ref = P.contrast_ce_loss({"seg": out["seg"].detach().cpu(), "embed": out["embed"].detach().cpu(),
                                      "segment_queue": sq, "pixel_queue": pq}, tgt.cpu(), with_embed=True,
                                     loss_weight=0.1, temperature=0.07, base_temperature=0.07, max_samples=64, max_views=4,
                                     with_memory=True, perm_fn=P.PermReplay(rec.draws))
            assert rel_err(loss.item(), ref.item()) < 1e-5
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses))
    assert not torch.equal(bank.pixel_queue_ptr, ptr0)            # the bank advanced
    assert net.proj.proj[0].weight.grad is not None and net.proj.proj[0].weight.grad.abs().sum().item() > 0


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_coco_stuff_shape_171_classes_with_bank(precision):
    """BASELINE configs[3] geometry (520x520 -> 66x66 embedding, 171 classes, non-divisible nearest interpolation,
    bank) at a reduced memory size; both sweeps against the float64 oracle on replayed permutations."""
    from contrastiveseg_b200.synth import make_bank, make_contrast_batch
    K, D, M = 171, 256, 24
    data = make_contrast_batch(B=2, D=D, h=66, w=66, num_classes=K, img_stride=8, block=40, seed=171, himg=520, wimg=520)
    bank = make_bank(K, M, D, 172)
    rec = P.PermRecorder(torch.Generator().manual_seed(4))
    e64 = data["embed"].double().requires_grad_(True)
    queue = torch.cat((bank["segment_queue"], bank["pixel_queue"]), 1)
    ref = P.pixel_contrast_loss(e64, data["target"], data["seg"].argmax(1), temperature=0.07, base_temperature=0.07,
                                max_samples=1024, max_views=10, queue=queue.double(), perm_fn=rec)
    ref.backward()
    crit = cs.PixelContrastLoss(_cfg(0.07, 0.07, 1024, 10, K, {"precision": precision}))
    crit.perm_fn = P.PermReplay(rec.draws)
    embed = data["embed"].to(DEV).requires_grad_(True)
    loss = crit(embed, data["target"].to(DEV), seg=data["seg"].to(DEV),
                queue=(bank["segment_queue"].to(DEV), bank["pixel_queue"].to(DEV)))
    loss.backward()
    tol_l, tol_g = (2e-6, 1e-5) if precision == "fp32" else (1e-4, 4e-3)
    assert rel_err(loss.item(), ref.item()) < tol_l
    assert (embed.grad.cpu().double() - e64.grad).abs().max().item() <= tol_g * e64.grad.abs().max().item()


def test_bank_tensor_path_workspace_sizes_cover_runtime_slots():
    """Regression: the step's partial buffers must be sized for the persistent sweep's slot count with a device-side
    plan (one slot per SM), not the host-known case (a buffer overrun here corrupted neighbouring allocations)."""
    from contrastiveseg_b200.synth import make_bank, make_contrast_batch
    K, D, M = 19, 256, 2000
    data = make_contrast_batch(B=1, D=D, h=64, w=64, num_classes=K, img_stride=4, block=16, seed=3)
    bank = make_bank(K, M, D, 4)
    crit = cs.PixelContrastLoss(_cfg(0.07, 0.07, 1024, 100, K, {"precision": "bf16"}))
    embed = data["embed"].to(DEV).requires_grad_(True)
    guard = torch.zeros(1 << 20, device=DEV)                  # neighbour allocation that must stay untouched
    for _ in range(3):
        loss = crit(embed, data["target"].to(DEV), seg=data["seg"].to(DEV),
                    queue=(bank["segment_queue"].to(DEV), bank["pixel_queue"].to(DEV)))
        loss.backward()
    torch.cuda.synchronize()
    ws = Fn.last_workspace(embed.device)
    import ctypes as C
    from contrastiveseg_b200 import _abi
    td = _abi.TcDesc()
    td.a_rows, td.D, td.mode, td.bank_K, td.bank_R = 1024, D, 1, K, 2 * M
    td.plan = ws.plan.data_ptr()
    td.temperature = td.base_temperature = 1.0
    ss = _abi.SweepSizes()
    _abi.check(_abi.load().pcl_tc_sizes(C.byref(td), C.byref(ss)))
    assert ws.partials.numel() >= 5 * ss.partial_f32 and ws.dpartials.numel() >= ss.dpartial_f32
    assert guard.abs().max().item() == 0 and torch.isfinite(loss).item()


# ---------------------------------------------------------------------------------------------------
# §8f row 1: fused bilinear(align_corners) up-sampling + weighted CE with ignore_index.  Tolerance: loss 1e-6 rel,
# gradient 1e-5 * max|g| against the float64 torch ops of the reference (oracle.ref_port.seg_cross_entropy).
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,K,h,w,H,W,weighted", [(2, 5, 16, 20, 32, 40, False), (1, 19, 13, 10, 50, 37, True),
                                                  (2, 7, 8, 8, 8, 8, False), (1, 3, 5, 7, 1, 9, True)])
def test_fused_upsample_cross_entropy(B, K, h, w, H, W, weighted):
    g = torch.Generator().manual_seed(B * 100 + K)
    seg = torch.randn(B, K, h, w, generator=g) * 2.0
    target = torch.randint(-1, K, (B, H, W), generator=g)
    weight = (torch.rand(K, generator=g) + 0.5) if weighted else None
    s1 = seg.clone().to(DEV).requires_grad_(True)
    loss = cs.upsample_cross_entropy(s1, target.to(DEV), weight.to(DEV) if weighted else None, -1)
    gout = torch.tensor(0.7, device=DEV)
    loss.backward(gout)
    s2 = seg.clone().double().requires_grad_(True)
    ref = P.seg_cross_entropy(s2, target, -1, weight.double() if weighted else None)
    ref.backward(torch.tensor(0.7, dtype=torch.float64))
    assert rel_err(loss.item(), ref.item()) < 2e-6
    assert (s1.grad.cpu().double() - s2.grad).abs().max().item() <= 1e-5 * s2.grad.abs().max().item() + 1e-12


def test_fused_seg_ce_full_size_and_wrapper_toggle():
    """Cityscapes shape (B=8, 19 x 128 x 256 -> 512 x 1024): fused vs the PyTorch ops on the GPU, and the wrapper
    gives the same loss with fused_seg_ce on / off."""
    from contrastiveseg_b200.synth import make_contrast_batch
    data = make_contrast_batch(B=8, D=32, h=128, w=256, num_classes=19, img_stride=4, block=32, seed=304)
    seg, tgt = data["seg"].to(DEV), data["target"].to(DEV)
    s1 = seg.clone().requires_grad_(True)
    l1 = cs.upsample_cross_entropy(s1, tgt, None, -1)
    l1.backward()
    s2 = seg.clone().requires_grad_(True)
    l2 = F.cross_entropy(F.interpolate(s2, size=tgt.shape[1:], mode="bilinear", align_corners=True), tgt, ignore_index=-1)
    l2.backward()
    assert rel_err(l1.item(), l2.item()) < 5e-6
    assert (s1.grad - s2.grad).abs().max().item() <= 2e-5 * s2.grad.abs().max().item()
    losses = []
    for fused in (True, False):
        rec_seed = torch.Generator().manual_seed(1)
        crit = cs.ContrastCELoss(_cfg(0.1, 0.07, 256, 20, 19, {"fused_seg_ce": fused})).to(DEV)
        crit.contrast_criterion.perm_fn = P.PermRecorder(rec_seed)
        losses.append(crit({"seg": seg, "embed": data["embed"].to(DEV)}, tgt, with_embed=True).item())
    assert rel_err(losses[0], losses[1]) < 5e-6


def test_workspace_is_released_when_the_graph_is_dropped_without_backward():
    g = load_golden("nomem_small")
    T, bT, ms, mv, K, ign = g["params"].tolist()
    crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K))
    embed = torch.from_numpy(g["embed"]).to(DEV).requires_grad_(True)
    target, predict = torch.from_numpy(g["target"]).to(DEV), torch.from_numpy(g["predict"]).to(DEV)
    seen = set()
    for _ in range(6):
        loss = crit(embed, target, predict)          # logged only: no backward
        seen.add(id(Fn.last_workspace(embed.device)))
        del loss
    assert len(seen) <= 2                            # no workspace leak
    l1 = crit(embed, target, predict)
    w1 = Fn.last_workspace(embed.device)
    l2 = crit(embed, target, predict)                # two pending graphs -> two distinct workspaces
    w2 = Fn.last_workspace(embed.device)
    assert w1 is not w2 and w1.busy and w2.busy
    l1.backward(); l2.backward()
    assert torch.isfinite(embed.grad).all() and not w1.busy and not w2.busy
