"""The anchor-column hand-off between the contrast loss and the fused BN projection head (ProjectionHead(...,
sparse_grad=True)): pcl_step_backward_cols against pcl_step_backward on the same descriptor, the head's column backward
(pcl_proj_bn_bwd_cols_dt + pcl_proj_bn_input_grad_cols_dt) against a float64 torch head fed the dense gradient built
from the columns, the contrast wrappers end to end against the dense head, the fallbacks, and peak memory at S1.
test_emu_sparse_head.py runs the check functions at small shapes on the emulated kernels (DEV = "cpu")."""
import ctypes as C
import copy

import pytest
import torch

import contrastiveseg_b200 as cs
import test_gpu_projection as P
import test_gpu_projection_bnrelu as PB
import test_gpu_projection_conv1 as PC
from contrastiveseg_b200 import _abi, functional as Fn
from contrastiveseg_b200.synth import make_bank, make_contrast_batch

DEV = "cuda:0"
BF = torch.bfloat16


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# 1. columns are the dense gradient
# ------------------------------------------------------------------------------------------------------------------
STEP_MODES = {
    "simt": dict(),
    "tensor": dict(precision="bf16"),
    "topk": dict(topk_negatives=5),
    "topk_tensor": dict(precision="bf16", topk_negatives=5),
    "normalize": dict(normalize=True),
    "bank": dict(bank=True),
    "bank_tensor": dict(bank=True, precision="bf16"),
}


def check_cols_equal_dense(mode, dtype=torch.float32, B=2, D=256, h=12, w=10, K=5, ms=96):
    kw = dict(STEP_MODES[mode])
    bank = kw.pop("bank", False)
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=2, block=3, seed=41)
    embed = data["embed"].to(device=DEV, dtype=dtype).requires_grad_(True)
    segq = pixq = None
    if bank:
        bk = make_bank(K, 12, D, 42)
        segq, pixq = bk["segment_queue"].to(DEV), bk["pixel_queue"].to(DEV)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=8, **kw)
    loss = cs.pixel_contrast_loss(embed, data["target"].to(DEV), seg=data["seg"].to(DEV), segment_queue=segq,
                                  pixel_queue=pixq, options=opts)
    ws = Fn.last_workspace(embed.device)
    lib = _abi.load()
    go = torch.full((), 0.75, dtype=torch.float32, device=DEV)
    cols = torch.full((ms, D), float("nan"), dtype=torch.float32, device=DEV)
    col_pix = torch.full((ms,), 12345, dtype=torch.int32, device=DEV)
    _abi.check(lib.pcl_step_backward_cols(C.byref(ws.desc), go.data_ptr(), cols.data_ptr(), col_pix.data_ptr(),
                                          Fn._stream_ptr(embed.device)), "pcl_step_backward_cols")
    loss.backward(go)
    _sync()
    A = int(ws.plan[_abi.PLAN_A].item())
    assert 0 < A <= ms
    meta = ws.anchor_meta.view(4, ms)[:, :A].long()
    q = meta[1] * h * w + meta[0]
    assert torch.equal(col_pix[:A].long(), q), mode                                   # the A sampled pixels ...
    assert bool((col_pix[A:] == -1).all()) and bool((cols[A:] == 0).all())          # ... then -1
    g = embed.grad.view(B, D, h * w)
    dense = g[meta[1], :, meta[0]]                                                   # (A, D) in embed's dtype
    if dtype == torch.float32:
        assert torch.equal(cols[:A].view(torch.int32), dense.view(torch.int32)), mode   # bit for bit
    else:
        assert torch.equal(cols[:A].to(dtype).view(torch.int16), dense.view(torch.int16)), mode
    mask = torch.ones(B, h * w, dtype=torch.bool, device=DEV)
    mask[meta[1], meta[0]] = False
    assert int((g.transpose(1, 2)[mask] != 0).sum().item()) == 0                     # zero off the anchors


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(STEP_MODES))
def test_cols_equal_the_dense_gradient(mode):
    check_cols_equal_dense(mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["simt", "tensor", "normalize", "bank_tensor"])
def test_rounded_cols_equal_the_bf16_dense_gradient(mode):
    check_cols_equal_dense(mode, BF)


# ------------------------------------------------------------------------------------------------------------------
# 2. the head's column backward against float64
# ------------------------------------------------------------------------------------------------------------------
def _columns(B, H, W, n, dead, seed):
    """n distinct pixels (b HW + p) with random columns, then `dead` unused ones (-1); the columns are bf16 values so
    that a bf16 zn's dense gradient holds them exactly.  Returns cols, col_pix and the dense gzn (fp32)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randperm(B * H * W, generator=g)[:n].to(torch.int32)
    cols = torch.randn(n + dead, 256, generator=g).to(BF).float()
    cols[n:] = 0.
    col_pix = torch.cat([q, torch.full((dead,), -1, dtype=torch.int32)])
    gzn = torch.zeros(B, 256, H * W)
    gzn[q.long() // (H * W), :, q.long() % (H * W)] = cols[:n]
    return cols.to(DEV), col_pix.to(DEV), gzn.view(B, 256, H, W).to(DEV)


def _hand_off(zn, cols, col_pix):
    """What an engine loss whose embed is zn does in its backward: deposit the columns, return the placeholder."""
    sink = Fn._sink_of(zn)
    assert sink is not None
    return sink.deposit(cols, col_pix, zn.shape)


HEAD_SHAPES = [(2, 40, 6, 7), (1, 300, 12, 13), (2, 720, 9, 11)]


def check_head_cols(shape, mode, dtype, n=37, dead=5, seed=3):
    B, Cin, H, W = shape
    y, bn, w, b, _ = PB._inputs(shape, mode, dtype, seed=seed)
    cols, col_pix, gzn = _columns(B, H, W, min(n, B * H * W), dead, seed + 1)
    ref, st = PB._reference(y, bn, w, b, gzn.to(dtype))
    yy, ww, bb = y.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    zn = cs.bn_relu_project_normalize(yy, bn, ww, bb, sparse_grad=True)
    zn.backward(_hand_off(zn, cols, col_pix))
    _sync()
    got = {"zn": zn.detach(), "gy": yy.grad, "gw": ww.grad, "gb": bb.grad, "ggamma": bn.weight.grad,
           "gbeta": bn.bias.grad}
    e = P.errors(got, ref)
    d = (got["gy"].double() - ref["gy"]).masked_fill(st["kink"], 0.)
    e["gy"] = ((d.abs().max() / ref["gy"].abs().max()).item(),) + e["gy"][1:]
    for k in PB.NAMES:
        assert e[k][0] <= PB.MAXABS[k] and e[k][1] <= PB.FROB[k], (k, e)
    for k in ("running_mean", "running_var"):
        r = st[k]
        assert (getattr(bn, k).double() - r).abs().max().item() <= PB.STATS_REL * r.abs().max().item(), k
    return got


def check_head_cols_conv1(shape, mode, dtype, n=37, dead=5, seed=5):
    B, Cin, H, W = shape
    x, w1, b1, bn, w2, b2, _ = PC._head_inputs(shape, mode, dtype, seed)
    cols, col_pix, gzn = _columns(B, H, W, min(n, B * H * W), dead, seed + 1)
    ref, st = PC.head_reference(x, w1, b1, bn, w2, b2, gzn.to(dtype))
    xx = x.clone().requires_grad_(True)
    ps = [t.clone().requires_grad_(True) for t in (w1, b1, w2, b2)]
    zn = cs.conv_bn_relu_project_normalize(xx, ps[0], ps[1], bn, ps[2], ps[3], sparse_grad=True)
    zn.backward(_hand_off(zn, cols, col_pix))
    _sync()
    got = {"zn": zn.detach(), "gx": xx.grad, "gw1": ps[0].grad, "gb1": ps[1].grad, "ggamma": bn.weight.grad,
           "gbeta": bn.bias.grad, "gw2": ps[2].grad, "gb2": ps[3].grad}
    PC.check_head(PC.head_errors(got, ref, st, bn.training), bn.training)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", HEAD_SHAPES + [(8, 720, 128, 256)])
def test_head_cols_match_fp64(shape, mode, dtype):
    check_head_cols(shape, mode, dtype, n=1024 if shape[0] == 8 else 37)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", HEAD_SHAPES)
def test_head_cols_with_conv1_match_fp64(shape, mode, dtype):
    check_head_cols_conv1(shape, mode, dtype)


def check_head_cols_bit_reproducible(shape=(2, 40, 6, 7), mode="train"):
    B, Cin, H, W = shape
    y, bn, w, b, _ = PB._inputs(shape, mode, seed=8)
    cols, col_pix, _ = _columns(B, H, W, 30, 3, 9)
    outs = []
    for bn_k in (bn, copy.deepcopy(bn)):
        yy, ww = y.clone().requires_grad_(True), w.clone().requires_grad_(True)
        zn = cs.bn_relu_project_normalize(yy, bn_k, ww, b, sparse_grad=True)
        zn.backward(_hand_off(zn, cols, col_pix))
        _sync()
        outs.append((yy.grad, ww.grad, bn_k.weight.grad, bn_k.bias.grad))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


@pytest.mark.gpu
def test_head_cols_bit_reproducible():
    check_head_cols_bit_reproducible()


# ------------------------------------------------------------------------------------------------------------------
# 3. / 4. end to end against the dense head, and the fallbacks
# ------------------------------------------------------------------------------------------------------------------
def _cfg(K, precision="fp32", ms=64, **contrast):
    c = {"temperature": 0.1, "base_temperature": 0.07, "max_samples": ms, "max_views": 8, "loss_weight": 0.1,
         "precision": precision, "rng": "torch_cpu", "seed": 7}
    c.update(contrast)
    return cs.Configer({"data": {"num_classes": K}, "network": {"stride": 2, "loss_weights": {"seg_loss": 1.0,
                                                                                               "aux_loss": 0.4}},
                        "loss": {"params": {"ce_ignore_index": -1}}, "contrast": c})


def _heads(Cin, conv1, seed=13):
    torch.manual_seed(seed)
    dense = cs.ProjectionHead(Cin, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                              fuse_conv1=conv1).to(DEV)
    sparse = cs.ProjectionHead(Cin, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                               fuse_conv1=conv1, sparse_grad=True).to(DEV)
    sparse.load_state_dict(dense.state_dict())
    return dense, sparse


def _perm_fn(seed):
    g = torch.Generator().manual_seed(seed)
    return lambda n: torch.randperm(n, generator=g)


def _run(head, crit, x, target, seg, extra=None, bank=None, with_embed=True, wrap=None):
    """One loss + backward of `crit` on head(x); returns the loss, x's and every parameter's gradient, the BN buffers
    and the bank."""
    crit.contrast_criterion.perm_fn = _perm_fn(17)
    xx = x.clone().requires_grad_(True)
    head.zero_grad(set_to_none=True)
    zn = head(xx)
    if wrap is not None:
        zn = wrap(zn)
    preds = {"seg": seg, "embed": zn}
    preds.update(extra or {})
    if bank is not None:
        preds["segment_queue"], preds["pixel_queue"] = bank
    loss = crit(preds, target, with_embed=with_embed)
    if isinstance(loss, tuple):
        loss = loss[0]
    loss.backward()
    _sync()
    out = {"loss": loss.detach(), "gx": xx.grad}
    out.update({n: p.grad for n, p in head.named_parameters()})
    bn = head.proj[1][0]
    out.update({k: getattr(bn, k).clone() for k in ("running_mean", "running_var", "num_batches_tracked")})
    return out


def _e2e_inputs(B=2, Cin=40, h=12, w=10, K=5, dtype=torch.float32, seed=21):
    data = make_contrast_batch(B=B, D=Cin, h=h, w=w, num_classes=K, img_stride=2, block=3, seed=seed)
    return data["embed"].to(device=DEV, dtype=dtype), data["target"].to(DEV), data["seg"].to(DEV)


EXACT = ("loss", "running_mean", "running_var", "num_batches_tracked")


def _compare(got, ref, exact_grads=False):
    for k in ref:
        if ref[k] is None:
            assert got[k] is None, k
            continue
        if k in EXACT or exact_grads:
            assert torch.equal(got[k], ref[k]), k
        elif k == "proj.0.bias":
            # conv1's bias gradient is zero in exact arithmetic in training (the batch mean removes it): bounded
            # against max|gW1|, as test_gpu_projection_bnrelu does
            scale = ref["proj.0.weight"].double().abs().max().item()
            assert (got[k].double() - ref[k].double()).abs().max().item() <= 2 * P.FP32_REF_MAXABS["gx"] * scale, k
        else:
            r = ref[k].double()
            scale = max(r.abs().max().item(), 1e-30)
            assert (got[k].double() - r).abs().max().item() <= 2 * P.FP32_REF_MAXABS["gx"] * scale, k
            assert (got[k].double() - r).norm().item() <= 2 * P.FP32_REF_FROB["gx"] * max(r.norm().item(), 1e-30), k


WRAPPERS = ["contrast_ce", "contrast_auxce", "mem_contrast_ce"]


def check_end_to_end(wrapper, conv1, dtype=torch.float32, B=2, Cin=40, h=12, w=10, K=5):
    cfg = _cfg(K)
    crit = {"contrast_ce": cs.ContrastCELoss, "contrast_auxce": cs.ContrastAuxCELoss,
            "mem_contrast_ce": cs.MemContrastCELoss}[wrapper](cfg)
    x, target, seg = _e2e_inputs(B, Cin, h, w, K)
    extra = {"seg_aux": seg.flip(1)} if wrapper == "contrast_auxce" else None
    bank = None
    if wrapper == "mem_contrast_ce":
        bk = make_bank(K, 12, 256, 22)
        bank = (bk["segment_queue"].to(DEV), bk["pixel_queue"].to(DEV))
    dense, sparse = _heads(Cin, conv1)
    twin = copy.deepcopy(sparse)
    with torch.autocast("cuda" if str(DEV).startswith("cuda") else "cpu", dtype=BF, enabled=dtype == BF):
        ref = _run(dense, crit, x, target, seg, extra, bank)
        got = _run(sparse, crit, x, target, seg, extra, bank)
        again = _run(twin, crit, x, target, seg, extra, bank)
    _compare(got, ref)
    for k in got:                                          # two sparse runs are bit-identical
        assert (got[k] is None and again[k] is None) or torch.equal(got[k], again[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("conv1", [False, True], ids=["bn_relu", "conv1"])
@pytest.mark.parametrize("wrapper", WRAPPERS)
def test_end_to_end_matches_the_dense_head(wrapper, conv1):
    check_end_to_end(wrapper, conv1)


def check_trainer_hook_with_enqueue(B=2, Cin=40, h=12, w=10, K=5, M=12):
    """MemContrastCELoss through ContrastTrainerHook.loss_step with the bank enqueue: same loss, buffers and bank."""
    from contrastiveseg_b200 import bank as bank_mod
    x, target, seg = _e2e_inputs(B, Cin, h, w, K)
    cfg = _cfg(K, warmup_iters=0, with_memory=True, memory_size=M, pixel_update_freq=5)
    cfg.params_root["loss"]["loss_type"] = "mem_contrast_ce_loss"
    res = []
    for head in _heads(Cin, False):
        torch.manual_seed(31)                              # the bank's initial rows, the enqueue's permutations
        bank = cs.MemoryBank(K, M, 256).to(DEV)
        hook = cs.ContrastTrainerHook(cfg, bank)
        hook.pixel_loss.contrast_criterion.perm_fn = _perm_fn(17)
        Fn._step_counter[0] = 0
        bank_mod._enqueue_counter[0] = 0
        for it in range(2):                                # the second step reads what the first enqueued
            xx = x.clone().requires_grad_(True)
            head.zero_grad(set_to_none=True)
            zn = head(xx)
            loss = hook.loss_step({"seg": seg, "embed": zn, "key": zn.detach(), "lb_key": target}, target, iters=it)
            loss.backward()
        _sync()
        out = {"loss": loss.detach(), "gx": xx.grad}
        out.update({n: p.grad for n, p in head.named_parameters()})
        out.update({k: getattr(head.proj[1][0], k).clone() for k in ("running_mean", "running_var",
                                                                         "num_batches_tracked")})
        res.append((out, bank.segment_queue.clone(), bank.pixel_queue.clone()))
    (ref, sq_r, pq_r), (got, sq_g, pq_g) = res
    assert torch.equal(sq_g, sq_r) and torch.equal(pq_g, pq_r)
    _compare(got, ref)


FALLBACKS = ["other_term", "two_losses", "retain_grad", "hook", "no_loss", "warmup", "warmup_skip"]


def check_fallback(case, B=2, Cin=40, h=12, w=10, K=5):
    """Cases where the head does not get the placeholder alone: the result is the dense head's, bit for bit."""
    x, target, seg = _e2e_inputs(B, Cin, h, w, K)
    res = []
    for head in _heads(Cin, False):
        crit = cs.ContrastCELoss(_cfg(K, skip_warmup_contrast=case == "warmup_skip"))
        crit.contrast_criterion.perm_fn = _perm_fn(17)
        xx = x.clone().requires_grad_(True)
        head.zero_grad(set_to_none=True)
        zn = head(xx)
        extra = {}
        if case == "no_loss":
            loss = (zn.float() * torch.linspace(-1, 1, zn.numel(), device=zn.device).view(zn.shape)).sum()
        elif case in ("warmup", "warmup_skip"):
            loss = crit({"seg": seg, "embed": zn}, target, with_embed=False)
        else:
            if case == "retain_grad":
                zn.retain_grad()
            if case == "hook":
                zn.register_hook(lambda g: g * 1.0)
            loss = crit({"seg": seg, "embed": zn}, target, with_embed=True)
            if case == "other_term":
                loss = loss + (zn.float() ** 2).mean()
            if case == "two_losses":
                crit.contrast_criterion.perm_fn = _perm_fn(18)
                loss = loss + 0.5 * crit.contrast_criterion(zn, target, seg=seg)
        loss.backward()
        _sync()
        out = {"loss": loss.detach(), "gx": xx.grad}
        out.update({n: p.grad for n, p in head.named_parameters()})
        if case == "retain_grad":
            extra["zn_grad"] = zn.grad
        out.update(extra)
        res.append(out)
    ref, got = res
    _compare(got, ref, exact_grads=True)


@pytest.mark.gpu
def test_trainer_hook_with_enqueue_matches_the_dense_head():
    check_trainer_hook_with_enqueue()


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
def test_fallbacks_give_the_dense_result(case):
    check_fallback(case)


# ------------------------------------------------------------------------------------------------------------------
# 5. refusals
# ------------------------------------------------------------------------------------------------------------------
def test_refusals():
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "convmlp", fused=True, sparse_grad=True)
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "linear", fused=True, sparse_grad=True)
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "convmlp", sparse_grad=True)
    lib = _abi.load(build_if_missing=True)
    for code in (_abi.DT_F16, 7):
        assert lib.pcl_proj_bn_bwd_cols_dt(1, code, 1, 1, 1, 1, 1, 8, 1, 1, 64, 16, 1, 1, None, 1, None, None,
                                           None) != 0
        assert lib.pcl_proj_bn_input_grad_cols_dt(1, code, 1, 1, 1, 1, 8, 1, 64, 16, 1, 1, None) != 0
    assert lib.pcl_proj_bn_cols_workspace_bytes(0, 64) < 0
    assert lib.pcl_step_backward_cols(None, None, None, None, None) != 0


# ------------------------------------------------------------------------------------------------------------------
# 6. memory at S1
# ------------------------------------------------------------------------------------------------------------------
def _peak(sparse_grad, dtype, B=8, Cin=720, h=128, w=256, K=19):
    head = cs.ProjectionHead(Cin, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                             sparse_grad=sparse_grad).to(DEV)
    crit = cs.ContrastCELoss(_cfg(K, ms=1024, rng="device"))
    data = make_contrast_batch(B=B, D=8, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=51)
    x = torch.randn(B, Cin, h, w, device=DEV)
    target, seg = data["target"].to(DEV), data["seg"].to(DEV)
    with torch.autocast("cuda", dtype=BF, enabled=dtype == BF):
        zn = head(x)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        loss = crit({"seg": seg, "embed": zn}, target, with_embed=True)
        loss.backward()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, zn.element_size()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_peak_memory_drops_by_at_least_the_dense_gradient(dtype):
    dense, esize = _peak(False, dtype)
    Fn.clear_workspaces()
    sparse, _ = _peak(True, dtype)
    print(f"\nPEAK {dtype}: dense {dense / 2**20:.1f} MiB, sparse {sparse / 2**20:.1f} MiB")
    assert dense - sparse >= 8 * 256 * 128 * 256 * esize, (dense, sparse)
