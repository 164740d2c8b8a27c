"""TEST INFRASTRUCTURE: differential fuzzing of the engine (real SIMT kernel sources on the host-fiber emulator,
tests/emu) against the oracle over random geometries.  Used by tests/test_emu_fuzz.py (bounded) and
tools/emu_fuzz.py (long runs).  Every fuzzer returns a list of failure descriptions (empty = clean); fuzz_graphed_step,
fuzz_graphed_criterion and fuzz_projection_head also return how many cases reached each of their coverage
categories, so that a test can require all of them.

It found the out-of-bounds wrap write for pixel_update_freq > memory_size (now refused, csrc/pcl_bank.cu: make_dims),
the NaN gradient of the two-call seg CE with a label grid smaller than the logits and every pixel ignored (now 0,
csrc/pcl_segce.cu: k_segce_bwd_gather), and the sparse head's silent dense fallback on a feature map one pixel wide
(functional._ColumnSink.is_placeholder)."""
import math
import random

import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi, functional as Fn
from contrastiveseg_b200.synth import make_bank, make_contrast_batch
from oracle import ref_port as P


def _cfg(T, bT, ms, mv, K):
    return cs.Configer({"data": {"num_classes": K},
                        "contrast": {"temperature": T, "base_temperature": bT, "max_samples": ms, "max_views": mv,
                                     "loss_weight": 0.1},
                        "loss": {"params": {"ce_ignore_index": -1}}, "network": {"stride": 8}})


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-9)


def fuzz_loss(seed: int, n: int, device="cpu", scale: int = 1):
    """PixelContrastLoss (exact path, injected permutations) vs the float64 oracle: random batch / embedding / image
    sizes (divisible and not), class counts, sampling limits, with and without bank, seg logits or predictions.
    Degenerate inputs: the reference raises (no class qualifies, zero views) -> the engine returns an exact zero;
    rows without positives -> NaN on both sides.  `scale` multiplies the largest feature map and max_samples."""
    rng = random.Random(seed)
    bad = []
    for it in range(n):
        B, D, h, w = rng.randint(1, 3), rng.choice([32, 64]), rng.randint(3, 36 * scale), rng.randint(3, 36 * scale)
        K, ms, mv = rng.randint(2, 12), rng.randint(4, 160 * scale), rng.randint(1, 16 * scale)
        block, boost = rng.choice([2, 3, 5, 8, 16]), rng.choice([0.0, 1.0, 2.0, 4.0])
        if rng.random() < 0.5:
            st = rng.choice([1, 2, 4])
            himg, wimg = h * st, w * st
        else:
            himg, wimg = rng.randint(h, 4 * h + 3), rng.randint(w, 4 * w + 3)
        mem, M = rng.random() < 0.4, rng.randint(2, 24)
        T, bT, s = rng.choice([0.07, 0.1, 0.5]), rng.choice([0.07, 0.1]), rng.randint(0, 10 ** 6)
        use_seg = rng.random() < 0.5
        desc = (f"loss seed={seed} it={it} B={B} D={D} hw={h}x{w} img={himg}x{wimg} K={K} ms={ms} mv={mv} block={block} "
                f"boost={boost} mem={mem} M={M} T={T} seg={use_seg}")
        data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=1, block=block, boost=boost, seed=s,
                                   himg=himg, wimg=wimg)
        bank = make_bank(K, M, D, s + 1) if mem else None
        rec = P.PermRecorder(torch.Generator().manual_seed(s))
        e64 = data["embed"].double().requires_grad_(True)
        q = torch.cat((bank["segment_queue"], bank["pixel_queue"]), 1).double() if mem else None
        predict = data["seg"].argmax(1)
        why = None
        try:
            ref = P.pixel_contrast_loss(e64, data["target"], predict, temperature=T, base_temperature=bT, max_samples=ms,
                                        max_views=mv, queue=q, perm_fn=rec)
            ref.backward()
        except (RuntimeError, IndexError, ValueError) as ex:
            why = type(ex).__name__
        crit = cs.PixelContrastLoss(_cfg(T, bT, ms, mv, K))
        crit.perm_fn = P.PermReplay(rec.draws) if why is None else (lambda k: torch.randperm(k))
        embed = data["embed"].clone().to(device).requires_grad_(True)
        queue = (bank["segment_queue"].clone().to(device), bank["pixel_queue"].clone().to(device)) if mem else None
        loss = crit(embed, data["target"].to(device), predict=None if use_seg else predict.to(device),
                    seg=data["seg"].to(device) if use_seg else None, queue=queue)
        loss.backward()
        if why == "IndexError":
            continue          # more anchors than bank columns (Q1): the reference crashes, the engine masks nothing
        if why is not None:
            if not (loss.item() == 0.0 and embed.grad.abs().max().item() == 0.0):
                bad.append(f"degenerate input not answered with an exact zero: {desc} ({why}) loss={loss.item()}")
            continue
        lv, rv = loss.item(), ref.item()
        if math.isnan(rv):
            if not math.isnan(lv):
                bad.append(f"reference NaN, engine {lv}: {desc}")
            continue
        gerr = (embed.grad.double().cpu() - e64.grad).abs().max().item() / max(e64.grad.abs().max().item(), 1e-9)
        if _rel(lv, rv) > 5e-6 or gerr > 2e-5:
            bad.append(f"mismatch rel={_rel(lv, rv):.2e} gerr={gerr:.2e}: {desc}")
    return bad


def fuzz_bank(seed: int, n: int):
    """dequeue_and_enqueue over several steps (wrap-around, stride mismatch Q6, overlapping writes Q4) vs the oracle:
    pointers exact, rows to rounding; configurations the reference rejects must be rejected too."""
    rng = random.Random(seed)
    bad = []
    names = ("segment_queue", "segment_queue_ptr", "pixel_queue", "pixel_queue_ptr")
    for it in range(n):
        B, D, h, w, K = rng.randint(1, 3), rng.choice([32, 64]), rng.randint(3, 30), rng.randint(3, 30), rng.randint(2, 10)
        M, Fq, s, img_s = rng.randint(2, 20), rng.randint(1, 12), rng.choice([1, 2, 3, 4, 8]), rng.choice([1, 2, 4])
        block, steps, sd = rng.choice([2, 4, 8, 16]), rng.randint(1, 5), rng.randint(0, 10 ** 6)
        desc = f"bank seed={seed} it={it} B={B} D={D} hw={h}x{w} K={K} M={M} F={Fq} stride={s} img_stride={img_s} steps={steps}"
        b0 = make_bank(K, M, D, sd)
        ref = [b0[k].clone() for k in names]
        mine = [b0[k].clone() for k in names]
        done = True
        for st in range(steps):
            data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=img_s, block=block, seed=sd + st)
            rec = P.PermRecorder(torch.Generator().manual_seed(sd + st))
            r_ok = True
            try:
                P.dequeue_and_enqueue(data["embed"], data["target"], *ref, network_stride=s, memory_size=M,
                                      pixel_update_freq=Fq, perm_fn=rec)
            except (RuntimeError, IndexError):
                r_ok = False
            m_ok = True
            try:
                cs.dequeue_and_enqueue(data["embed"].clone(), data["target"], *mine, network_stride=s, memory_size=M,
                                       pixel_update_freq=Fq, distributed=False,
                                       perm_fn=P.PermReplay(rec.draws) if r_ok else (lambda k: torch.randperm(k)))
            except _abi.PclError:
                m_ok = False
            grid = -(-h * img_s // s) * -(-w * img_s // s)          # positions of labels[:, ::s, ::s]
            if r_ok and not m_ok and (Fq > M or grid > h * w):
                # refused up front from the geometry alone (documented): pixel_update_freq > memory_size, or a label
                # grid with more positions than feature columns (Q6) — the reference only fails there when the data
                # happens to put a labelled position / a large class beyond the limit
                done = False
                break
            if r_ok != m_ok:
                bad.append(f"refusal differs (reference ok={r_ok}, engine ok={m_ok}): {desc}")
                done = False
                break
            if not r_ok:
                done = False
                break
        if not done:
            continue
        if not (torch.equal(ref[1], mine[1]) and torch.equal(ref[3], mine[3])):
            bad.append(f"pointers differ: {desc}")
            continue
        e_seg, e_pix = (ref[0] - mine[0]).abs().max().item(), (ref[2] - mine[2]).abs().max().item()
        if e_seg > 2e-6 or e_pix > 2e-7:
            bad.append(f"rows differ seg={e_seg:.1e} pix={e_pix:.1e}: {desc}")
    return bad


def fuzz_segce(seed: int, n: int):
    """Fused bilinear(align_corners) up/down-sampling + weighted CE with ignore vs the float64 torch ops."""
    rng = random.Random(seed)
    bad = []
    for it in range(n):
        B, K, h, w = rng.randint(1, 3), rng.randint(2, 21), rng.randint(1, 20), rng.randint(1, 24)
        H, W, weighted, ign = rng.randint(1, 60), rng.randint(1, 60), rng.random() < 0.5, rng.choice([-1, 255, 0])
        g = torch.Generator().manual_seed(rng.randint(0, 10 ** 6))
        seg = torch.randn(B, K, h, w, generator=g) * 2
        target = torch.randint(0, K, (B, H, W), generator=g)
        target[torch.rand(B, H, W, generator=g) < 0.2] = ign
        weight = (torch.rand(K, generator=g) + 0.5) if weighted else None
        desc = f"segce seed={seed} it={it} B={B} K={K} {h}x{w}->{H}x{W} weighted={weighted} ignore={ign}"
        s1 = seg.clone().requires_grad_(True)
        loss = cs.upsample_cross_entropy(s1, target, weight, ign)
        loss.backward(torch.tensor(0.7))
        s2 = seg.clone().double().requires_grad_(True)
        ref = P.seg_cross_entropy(s2, target, ign, weight.double() if weighted else None)
        ref.backward(torch.tensor(0.7, dtype=torch.float64))
        if math.isnan(ref.item()):
            if not math.isnan(loss.item()):
                bad.append(f"reference NaN, engine {loss.item()}: {desc}")
            continue
        gerr = (s1.grad.double() - s2.grad).abs().max().item() / max(s2.grad.abs().max().item(), 1e-9)
        if _rel(loss.item(), ref.item()) > 3e-6 or gerr > 2e-5:
            bad.append(f"mismatch rel={_rel(loss.item(), ref.item()):.2e} gerr={gerr:.2e}: {desc}")
    return bad


def fuzz_device_sampling(seed: int, n: int, check_sampling, device="cpu", scale: int = 1):
    """Device RNG (keyed bijection, no injected permutations), optional fused normalise: every anchor a valid distinct
    pixel of its (image, class, hard|easy) group; loss / gradient vs the oracle evaluated on exactly those anchors.
    `scale` multiplies the largest feature map and max_samples."""
    rng = random.Random(seed)
    bad = []
    for it in range(n):
        B, D, h, w = rng.randint(1, 3), rng.choice([32, 64]), rng.randint(4, 40 * scale), rng.randint(4, 40 * scale)
        K, ms, mv = rng.randint(2, 10), rng.randint(4, 200 * scale), rng.randint(1, 16 * scale)
        block, st, boost = rng.choice([2, 4, 8, 16]), rng.choice([1, 2, 4]), rng.choice([0.0, 2.0, 4.0])
        mem, norm, sd = rng.random() < 0.4, rng.random() < 0.4, rng.randint(0, 10 ** 6)
        desc = f"devrng seed={seed} it={it} B={B} D={D} {h}x{w} K={K} ms={ms} mv={mv} block={block} st={st} mem={mem} norm={norm}"
        data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=st, block=block, boost=boost, seed=sd)
        bank = make_bank(K, rng.randint(8, 30), D, sd + 1)
        crit = cs.PixelContrastLoss(_cfg(0.1, 0.07, ms, mv, K))
        embed = (data["embed_raw"] if norm else data["embed"]).clone().to(device).requires_grad_(True)
        queue = (bank["segment_queue"].clone().to(device), bank["pixel_queue"].clone().to(device)) if mem else None
        loss = crit(embed, data["target"].to(device), seg=data["seg"].to(device), queue=queue, normalize=norm)
        loss.backward()
        ws = Fn.last_workspace(embed.device)
        TC, V, A = ws.plan_header()[:3]
        lab = P.downsample_labels(data["target"], h, w).reshape(B, -1)
        prd = data["seg"].argmax(1).reshape(B, -1)
        if TC == 0 or V == 0:
            if loss.item() != 0.0:
                bad.append(f"degenerate input, loss {loss.item()}: {desc}")
            continue
        try:
            _, _, A2, meta = check_sampling(ws, lab, prd, ms, mv)
        except AssertionError as ex:
            bad.append(f"invalid sample set ({str(ex)[:120]}): {desc}")
            continue
        pix, img, cls, refrow = meta
        if mem and A > bank["segment_queue"].shape[0] * 2 * bank["segment_queue"].shape[1]:
            continue
        e64 = (data["embed_raw"] if norm else data["embed"]).double().requires_grad_(True)
        Xf = (F.normalize(e64, dim=1) if norm else e64).permute(0, 2, 3, 1).reshape(B, -1, D)
        inv = torch.empty(A, dtype=torch.long)
        inv[refrow] = torch.arange(A)
        anchors, ya = Xf[img, pix][inv], cls[inv].double()
        if mem:
            contrast, yc = P.flatten_queue(torch.cat((bank["segment_queue"], bank["pixel_queue"]), 1).double())
            lo = P.infonce_dense(anchors, ya, contrast, yc, 0.1, 0.07)
        else:
            lo = P.infonce_dense(anchors, ya, anchors, ya, 0.1, 0.07)
        lo.backward()
        if math.isnan(lo.item()):
            if not math.isnan(loss.item()):
                bad.append(f"reference NaN, engine {loss.item()}: {desc}")
            continue
        gerr = (embed.grad.double().cpu() - e64.grad).abs().max().item() / max(e64.grad.abs().max().item(), 1e-9)
        if _rel(loss.item(), lo.item()) > 5e-6 or gerr > 3e-5:
            bad.append(f"mismatch rel={_rel(loss.item(), lo.item()):.2e} gerr={gerr:.2e}: {desc}")
    return bad


def fuzz_topk(seed: int, n: int, device="cpu", scale: int = 1):
    """a10 top-k kernels vs the sort-based oracle: explicit / self / bank (zero tail) operands; exact dyadic data (ties,
    strict gradient check) and unit-norm data (near-ties: loss strict, gradient in norm).  `scale` multiplies the
    largest A, N and bank size."""
    rng = random.Random(seed)
    bad = []
    for it in range(n):
        A, N, D, ncls = rng.randint(2, 150 * scale), rng.randint(2, 400 * scale), rng.choice([32, 64]), rng.randint(2, 8)
        k, exact, mode = rng.randint(1, 60), rng.random() < 0.5, rng.choice(["explicit", "self", "bank"])
        g = torch.Generator().manual_seed(rng.randint(0, 10 ** 6))
        desc = f"topk seed={seed} it={it} A={A} N={N} D={D} classes={ncls} k={k} exact={exact} mode={mode}"
        if exact:
            den = 4 if D == 32 else 8                       # keeps exp(l - m) inside the fp32 range
            mk = lambda *s: torch.randint(-3, 4, s, generator=g).double() / den      # noqa: E731
            T, bT = 0.125, 0.25
        else:
            mk = lambda *s: F.normalize(torch.randn(*s, generator=g), dim=-1).double()   # noqa: E731
            T, bT = 0.1, 0.07
        a, ya = mk(A, D), torch.randint(0, ncls, (A,), generator=g)
        if mode == "explicit":
            c, yc, diag = mk(N, D), torch.randint(0, ncls, (N,), generator=g), torch.arange(A) % N
            o = P.infonce_topk(a, ya, c, yc, T, bT, k, False, diag_cols=diag)
            loss, rs, st = Fn.infonce_forward(a.float().to(device), ya.to(device), contrast=c.float().to(device),
                                              contrast_cls=yc.to(device), diag_col=diag.to(device),
                                              temperature=T, base_temperature=bT, topk=k)
        elif mode == "self":
            o = P.infonce_topk(a, ya, a, ya, T, bT, k, True)
            loss, rs, st = Fn.infonce_forward(a.float().to(device), ya.to(device), temperature=T, base_temperature=bT,
                                              topk=k)
        else:
            K, M = ncls, rng.randint(1, 12 * scale)
            if A > K * 2 * M:
                continue
            segq, pixq = mk(K, M, D), mk(K, M, D)
            if exact:
                pixq[:, ::3] = 0
            ya = ya[torch.argsort(torch.where(ya == 0, K, ya), stable=True)]
            contrast, yc = P.flatten_queue(torch.cat((segq, pixq), 1))
            o = P.infonce_topk(a, ya, contrast, yc.long(), T, bT, k, False)
            loss, rs, st = Fn.infonce_forward(a.float().to(device), ya.to(device),
                                              queues=(segq.float().to(device), pixq.float().to(device)),
                                              diag_col=torch.arange(A).to(device), temperature=T, base_temperature=bT, topk=k)
        dA = Fn.infonce_backward(st, rs).double().cpu()
        lo = o["loss"].item()
        if math.isnan(lo):
            if not math.isnan(loss.item()):
                bad.append(f"reference NaN, engine {loss.item()}: {desc}")
            continue
        if exact:
            gerr, tol = (dA - o["dA"]).abs().max().item() / max(o["dA"].abs().max().item(), 1e-9), 2e-5
        else:
            gerr, tol = (torch.linalg.norm(dA - o["dA"]) / max(torch.linalg.norm(o["dA"]).item(), 1e-9)).item(), 5e-2
        if _rel(loss.item(), lo) > 1e-5 or gerr > tol:
            bad.append(f"mismatch rel={_rel(loss.item(), lo):.2e} gerr={gerr:.2e}: {desc}")
    return bad


def _bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


def fuzz_tensor_path(seed: int, n: int, device="cpu", scale: int = 1):
    """wgmma sweeps (functional model) on explicit operands: self-contrast, explicit contrast set (sorted / unsorted
    labels), bank through the bf16 shadow; ragged A and N (not multiples of the 128 x 256 tile), few / many classes.
    Loss and positive counts against the float64 closed form on the bf16-rounded operands; gradient within the bf16
    tolerance of the path (max-abs 6e-3 * max|g|, relative Frobenius 5e-3).  `scale` multiplies the largest A, N and
    bank size (on a GPU: enough (row tile, column tile) pairs to fill the SMs several times)."""
    rng = random.Random(seed)
    bad = []
    for it in range(n):
        A, N, ncls = rng.randint(1, 420 * scale), rng.randint(1, 1500 * scale), rng.randint(1, 20)
        T, mode, clustered = rng.choice([0.07, 0.1, 0.5]), rng.choice(["self", "sorted", "unsorted", "bank"]), rng.choice([0.0, 0.5])
        g = torch.Generator().manual_seed(rng.randint(0, 10 ** 6))
        M = rng.randint(1, 40 * scale) if mode == "bank" else None
        why = tensor_case(A, N, ncls, T, mode, clustered, g, M=M, device=device, ref_device=device)
        if why:
            bad.append(f"{why}: tensor seed={seed} it={it} A={A} N={N} classes={ncls} T={T} mode={mode} clustered={clustered}")
    return bad


def tensor_case(A, N, ncls, T, mode, clustered, g, M=None, device="cpu", ref_device="cpu"):
    """One tensor-path call (forward + backward) against the float64 closed form (fuzz_tensor_path's bounds), operands
    drawn from `g`.  mode "bank": K = max(ncls, 2) classes of M rows in each queue (A > 2 K M is skipped: the closed
    form needs a contrast column per anchor).  Returns None, or what differs."""
    from contrastiveseg_b200.bank import shadow_rows
    lib = _abi.load()
    centers = F.normalize(torch.randn(ncls + 1, 256, generator=g), dim=1)
    ya = torch.randint(0, ncls, (A,), generator=g)
    a = F.normalize(torch.randn(A, 256, generator=g) + clustered * 16 * centers[ya], dim=1)
    if mode == "self":
        loss, st, state = Fn.infonce_tc_forward(a.to(device), ya.to(device), temperature=T, base_temperature=0.07)
        cf = P.infonce_closed_form(_bf(a).double().to(ref_device), ya.to(ref_device), _bf(a).double().to(ref_device),
                                   ya.to(ref_device), T, 0.07, self_contrast=True)
    elif mode in ("sorted", "unsorted"):
        yc = torch.randint(0, ncls, (N,), generator=g)
        if mode == "sorted":
            yc = torch.sort(yc).values
        c = F.normalize(torch.randn(N, 256, generator=g) + clustered * 16 * centers[yc], dim=1)
        c16 = Fn.to_bf16_rows(c.to(device), -(-N // 256) * 256)
        diag = torch.arange(A) % N
        loss, st, state = Fn.infonce_tc_forward(a.to(device), ya.to(device), contrast_bf16=c16, contrast_cls=yc.to(device),
                                                n_cols=N, diag_col=diag.to(device), temperature=T, base_temperature=0.07,
                                                sorted_cols=(mode == "sorted"))
        cf = P.infonce_closed_form(_bf(a).double().to(ref_device), ya.to(ref_device), _bf(c).double().to(ref_device),
                                   yc.to(ref_device), T, 0.07, self_contrast=False, diag_cols=diag)
    else:
        K = max(ncls, 2)
        if A > K * 2 * M:
            return None
        ya = torch.randint(0, K, (A,), generator=g)
        ya = ya[torch.argsort(torch.where(ya == 0, K, ya), stable=True)]
        a = F.normalize(torch.randn(A, 256, generator=g) + clustered * 16 * centers[ya], dim=1)
        segq = F.normalize(torch.randn(K, M, 256, generator=g), dim=2)
        pixq = F.normalize(torch.randn(K, M, 256, generator=g), dim=2)
        shadow = torch.empty((shadow_rows(K, M), 256), dtype=torch.bfloat16, device=device)
        segq_d, pixq_d = segq.to(device), pixq.to(device)
        _abi.check(lib.pcl_bank_shadow_rebuild(segq_d.data_ptr(), pixq_d.data_ptr(), K, M, 256, shadow.data_ptr(), None))
        loss, st, state = Fn.infonce_tc_forward(a.to(device), ya.to(device), bank=(shadow, K, 2 * M),
                                                diag_col=torch.arange(A).to(device), temperature=T, base_temperature=0.07)
        contrast, yc = P.flatten_queue(torch.cat((_bf(segq), _bf(pixq)), 1).double())
        cf = P.infonce_closed_form(_bf(a).double().to(ref_device), ya.to(ref_device), contrast.to(ref_device),
                                   yc.long().to(ref_device), T, 0.07, self_contrast=False)
    dA = Fn.infonce_tc_backward(state, st).double().cpu()
    cf = {k: cf[k].cpu() for k in ("loss", "npos", "dA")}
    lo = cf["loss"].item()
    if math.isnan(lo):
        return None if math.isnan(loss.item()) else f"reference NaN, engine {loss.item()}"
    if not torch.equal(st[4].double().cpu(), cf["npos"]):
        return "positive counts differ"
    # the gradient reference uses the same bf16-rounded operands (the rounding of the operands is not under test)
    gmax = cf["dA"].abs().max().item()
    gabs = (dA - cf["dA"]).abs().max().item() / max(gmax, 1e-9)
    gfro = ((dA - cf["dA"]).norm() / max(cf["dA"].norm().item(), 1e-9)).item()
    # (a loss that is exactly 0 in real arithmetic — a single class, no negatives — comes out as ~1e-8 of ex2/lg2
    # approximation noise on the tensor path: absolute floor next to the relative bound)
    if abs(loss.item() - lo) > 5e-5 * abs(lo) + 1e-6 or gabs > 6e-3 or gfro > 5e-3:   # (tiny contrast sets average less)
        return f"mismatch rel={_rel(loss.item(), lo):.2e} gabs={gabs:.2e} gfro={gfro:.2e}"
    return None


GRAPH_CATEGORIES = ("fused full-fill", "fused sparse", "streaming bf16", "exact fp32", "bank", "bank + enqueue",
                    "half embed", "A = 0 replay", "tile-edge crossing", "non-integer label ratio")
# max_samples draws lean on the tile edges of the tensor path (128-row, 256-column tiles) and on the ends of the range
_MS_EDGES = (1, 127, 128, 129, 255, 256, 257, 511, 513, 700, 1023, 1024)
_BANK_NAMES = ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr")


def _sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize(device)


def _same_bits(a, b):
    """Bit-identical tensors (the sign of a zero counts; NaN equals NaN whatever its payload)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    it = {2: torch.int16, 4: torch.int32}[a.element_size()]
    z = torch.zeros((), dtype=a.dtype, device=a.device)
    return torch.equal(torch.where(na, z, a).view(it), torch.where(nb, z, b).view(it))


def _tiles(A):
    return -(-A // 128), -(-A // 256)


def graph_step_inputs(B, D, h, w, K, himg, wimg, block, ignore, seq, seed):
    """draw(r): the CPU inputs of replay r (make_contrast_batch at himg x wimg, a fraction `ignore` of the labels set to
    the ignore label).  seq "empty": replay 1 has one labelled pixel, so no class qualifies (A = 0); seq "edge": odd
    replays keep one class of the label map, so A jumps between replays (across tile edges when max_samples allows)."""
    def draw(r):
        data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=1, block=block, seed=seed + 7919 * r,
                                   himg=himg, wimg=wimg)
        tgt = data["target"]
        g = torch.Generator().manual_seed(seed + 31 * r + 1)
        tgt[torch.rand(tgt.shape, generator=g) < ignore] = -1
        if seq == "empty" and r == 1:
            tgt.fill_(-1)
            tgt[0, 0, 0] = 0
        elif seq == "edge" and r % 2 == 1:
            tgt[tgt != int(torch.randint(0, K, (1,), generator=g))] = -1
        return data
    return draw


def _f64_reference(c, X, cls, refrow, queue):
    """Loss and d loss / d embed rows of the drawn anchors in float64 (closed form), in the step's row order.
    X: the drawn embed rows as stored (float64); queue: the (K, 2M, D) bank as the replay read it, or None.  The tensor
    path computes on bf16 operands: the reference rounds them the same way.  None when the closed form cannot score the
    draw (a bank step with more anchors than bank columns: the diagonal column of a row does not exist)."""
    T, bT, A = c["T"], c["bT"], X.shape[0]
    tensor = c["precision"] == "bf16"
    y = F.normalize(X, dim=1) if c["normalize"] else X
    a = _bf(y.float()).double() if tensor else y
    if queue is None:
        contrast, yc, diag, self_c = a, cls, None, True
    else:
        q = _bf(queue.float()).double() if tensor else queue
        contrast, yc = P.flatten_queue(q)
        yc, diag, self_c = yc.long(), refrow, False
        if A > contrast.shape[0]:
            return None
    cf = P.infonce_closed_form(a, cls, contrast, yc, T, bT, self_contrast=self_c, diag_cols=diag)
    loss, dA = cf["loss"], cf["dA"]
    if c["nan_safe"]:            # rows without positives contribute 0 to the loss and nothing to the gradient
        ok = cf["npos"] > 0
        G = torch.where(ok[:, None], cf["G"], torch.zeros_like(cf["G"]))
        dA = G @ contrast / T + ((G.t() @ a) / T if self_c else 0)
        loss = torch.where(ok, cf["row_loss"], torch.zeros_like(cf["row_loss"])).sum() / A
    if c["normalize"]:           # through the normalisation: (g - y (y . g)) / |x|
        dA = (dA - y * (y * dA).sum(1, keepdim=True)) / X.norm(dim=1, keepdim=True)
    return loss.item(), dA


def score_step_replay(c, ref, step, embed32, labels, seg, pred, q_before, scale, check_sampling, cov, reached, prev_A,
                      why):
    """The float64 scoring of one replay of a captured contrast step: the drawn anchors are a valid sample of the
    replay's labels (check_sampling), loss and gradient rows of `ref` (the fp32 step with the anchors of `step`: step
    itself, or its fp32 twin when embed is half) match the closed form on the drawn rows (q_before: the bank as the
    replay read it), and every element of step.grad at no drawn anchor is +0.  scale: the step's grad_scale.  Counts the
    replay in cov["scored"] / cov["skipped"] and sets reached["A = 0 replay"] / ["tile-edge crossing"].
    Returns (failure or None, A, whether the closed form scored the replay, the float64 contrast loss: 0 when A = 0,
    None when unscored)."""
    dev = labels.device
    B, D, h, w, ms, mv, bT = (c[k] for k in ("B", "D", "h", "w", "ms", "mv", "bT"))
    tensor = c["precision"] == "bf16"
    TC, V, A = ref.ws.plan_header()[:3]
    lv, gv = ref.loss.item(), ref.grad
    scored, lo = False, None
    # the drawn anchors: a valid sample of the replay's labels
    lab = P.downsample_labels(labels.cpu(), h, w).reshape(B, -1)
    lab[lab == c.get("ignore_label", -1)] = -1
    prd = (seg.float().argmax(1) if seg is not None else pred).cpu().reshape(B, -1)
    if TC == 0 or V == 0:
        kept = sum(len(P.kept_classes(lab[b], -1, mv)) for b in range(B))
        if A != 0 or kept != TC or step.loss.item() != 0.0:
            return (f"no anchors: A = {A}, {kept} classes qualify for {TC}, loss {step.loss.item()}: {why}", A, False,
                    None)
        reached["A = 0 replay"] = True
        pix = img = torch.zeros(0, dtype=torch.long)
        lo = 0.0
    else:
        try:
            _, _, A, (pix, img, cls, refrow) = check_sampling(ref.ws, lab, prd, ms, mv)
        except AssertionError as ex:
            return (f"invalid sample set ({str(ex)[:120]}): {why}", A, False, None)
        if prev_A and _tiles(prev_A) != _tiles(A):
            reached["tile-edge crossing"] = True
        # float64 closed form on the drawn rows (the values embed holds)
        X = embed32.permute(0, 2, 3, 1).reshape(B, h * w, D)[img.to(dev), pix.to(dev)].double().cpu()
        out = _f64_reference(c, X, cls, refrow, q_before)
        if out is None:
            cov["skipped"] = cov.get("skipped", 0) + 1
        else:
            lo, dA = out
            dA = scale * dA
            g_rows = gv.float().permute(0, 2, 3, 1).reshape(B, h * w, D)[img.to(dev), pix.to(dev)].double().cpu()
            if math.isnan(lo):
                if not math.isnan(lv):
                    return (f"reference NaN, engine {lv}: {why}", A, False, None)
            else:
                # (a loss or gradient that is 0 in real arithmetic — one class, no negatives — comes out as rounding
                # noise: absolute floors next to the relative bounds, the gradient's at 1e-3 of its natural scale;
                # grad_scale 0 needs exact zeros)
                gmax = max(dA.abs().max().item(), abs(scale) * 1e-3 / (bT * A), 1e-300)
                gabs = (g_rows - dA).abs().max().item() / gmax
                gfro = ((g_rows - dA).norm() / max(dA.norm().item(), gmax)).item()
                if tensor:
                    ok = abs(lv - lo) <= 5e-5 * abs(lo) + 1e-6 and gabs <= 6e-3 and gfro <= 5e-3
                else:
                    ok = abs(lv - lo) <= 2e-6 * abs(lo) + 1e-6 and gabs <= 1e-5
                if not ok:
                    return (f"float64: loss {lv} vs {lo}, gradient max-abs {gabs:.2e} Frobenius {gfro:.2e}: {why}", A,
                            False, None)
            scored = True
            cov["scored"] = cov.get("scored", 0) + 1
    # every element at no drawn anchor is +0
    z = step.grad.clone()
    if A:
        z.view(B, D, h * w)[img.to(dev), :, pix.to(dev)] = 0
    if bool(((z != 0) | torch.signbit(z)).any()):
        n_bad = int(((z != 0) | torch.signbit(z)).sum())
        return (f"{n_bad} gradient elements at no drawn anchor are not +0: {why}", A, False, None)
    return None, A, scored, lo


def graphed_step_case(c, draw, n_rep, device, check_sampling, cov, desc):
    """One GraphedContrastStep (configuration `c`), `n_rep` replays, the static inputs refilled in place from draw(r)
    before replay r.  Every replay: the anchors are a valid sample (check_sampling) and those of eager step r + 1,
    loss and gradient match the eager step and the float64 closed form on the drawn rows, every gradient element at no
    drawn anchor is +0 (the buffer is NaN before a full-fill replay), a bank written by the step equals the eager trainer
    order.  Half embed: an fp32 twin step on the same values must give the same loss bits and the gradient rounded
    once.  Adds the categories the case reached to `cov` (counted when a replay of the case was scored against float64;
    cov["scored"] / cov["skipped"]: replays the closed form scored / could not score).
    Returns the failures."""
    from contrastiveseg_b200 import bank as bank_mod
    dev = torch.device(device)
    B, D, h, w, K, ms, mv, T, bT = (c[k] for k in ("B", "D", "h", "w", "K", "ms", "mv", "T", "bT"))
    scale = c["grad_scale"]
    tensor = c["precision"] == "bf16"
    d0 = draw(0)
    src = lambda d: d["embed_raw"] if c["normalize"] else d["embed"]        # noqa: E731
    embed = src(d0).to(dev, c["embed_dtype"]).contiguous()
    half = embed.dtype != torch.float32
    embed32 = embed.float() if half else embed
    labels = d0["target"].to(dev)
    seg = d0["seg"].to(dev, c["seg_dtype"]) if c["seg_dtype"] is not None else None
    pred = d0["seg"].argmax(1).to(dev) if seg is None else None
    bank = bank_e = enq = None
    kw, kw_e = {}, {}
    if c["bank"] != "none":
        b0 = make_bank(K, c["M"], D, c["seed"] + 1)

        def new_bank():
            mb = cs.MemoryBank(K, c["M"], D, with_shadow=tensor).to(dev)
            for k in _BANK_NAMES:
                getattr(mb, k).copy_(b0[k])
            if tensor:
                mb.sync_shadow()
            return mb
        bank = new_bank()
        bank_e = new_bank() if c["bank"] == "enqueue" else bank
        kw = dict(segment_queue=bank.segment_queue, pixel_queue=bank.pixel_queue, bank_shadow=bank.shadow)
        kw_e = dict(segment_queue=bank_e.segment_queue, pixel_queue=bank_e.pixel_queue, bank_shadow=bank_e.shadow)
        if c["bank"] == "enqueue":
            enq = dict(network_stride=c["stride"], pixel_update_freq=c["freq"], seed=c["seed"] % 997)
    opts = cs.ContrastOptions(temperature=T, base_temperature=bT, max_samples=ms, max_views=mv, seed=c["seed"] % 1000,
                              num_classes=K, normalize=c["normalize"], nan_safe=c["nan_safe"], precision=c["precision"])
    mk = lambda e, q: cs.GraphedContrastStep(e, labels, seg=seg, predict=pred, options=opts, grad_scale=scale,   # noqa: E731
                                             overlap_zero_fill=c["overlap"], fused=c["fused"],
                                             sparse_reset=c["sparse"], enqueue=q, **kw)
    # the twin reads the bank before the step under test writes it (same state as the eager loss reads)
    twin = mk(embed32, None) if half else None
    step = mk(embed, dict(enq, bank=bank) if enq else None)
    want_fused = tensor and c["bank"] == "none" and not c["normalize"] and c["fused"] is None
    if step.fused != want_fused or (twin is not None and twin.fused != step.fused):
        return [f"fused = {step.fused}, expected {want_fused}: {desc}"]
    ref = twin if half else step                 # the fp32 step checked against the eager step and float64
    steps = [s for s in (twin, step) if s is not None]
    for s in steps:
        if s.sparse_reset:                       # nothing else may write a sparse-reset buffer: poison, then reset
            s.grad.fill_(float("nan"))
            s.reset_grad()
    reached = {"half embed": half, "bank": bank is not None, "bank + enqueue": enq is not None,
               "fused full-fill": step.fused and not step.sparse_reset, "fused sparse": step.sparse_reset,
               "streaming bf16": tensor and not step.fused, "exact fp32": not tensor,
               "non-integer label ratio": c["himg"] % h != 0 or c["wimg"] % w != 0}
    scored, prev_A = 0, None
    for r in range(n_rep):
        why = f"replay {r}: {desc}"
        if r:
            d = draw(r)
            embed.copy_(src(d).to(embed.dtype))
            if half:
                embed32.copy_(embed.float())
            labels.copy_(d["target"])
            if seg is not None:
                seg.copy_(d["seg"].to(seg.dtype))
            else:
                pred.copy_(d["seg"].argmax(1))
        for s in steps:
            if not s.sparse_reset:               # a full fill must cover the whole buffer
                s.grad.fill_(float("nan"))
        q_before = torch.cat((bank.segment_queue, bank.pixel_queue), 1).double().cpu() if bank is not None else None
        for s in steps:
            s.replay()
        _sync(dev)
        meta = ref.ws.anchor_meta.clone()
        TC, V, A = ref.ws.plan_header()[:3]
        # eager step with counter r + 1 (trainer order with an enqueue: loss -> enqueue -> backward)
        Fn._step_counter[0] = r
        bank_mod._enqueue_counter[0] = r
        e = embed32.clone().requires_grad_(True)
        l2 = cs.pixel_contrast_loss(e, labels, seg=seg, predict=pred, options=opts, **kw_e)
        ws = Fn.last_workspace(e.device)
        if enq:
            bank_e.enqueue(e.detach(), labels, network_stride=enq["network_stride"],
                           pixel_update_freq=enq["pixel_update_freq"], seed=enq["seed"])
        l2.backward(torch.full((), scale, device=dev))
        _sync(dev)
        lv, gv = ref.loss.item(), ref.grad
        if not torch.equal(ws.anchor_meta, meta):
            return [f"anchors differ from the eager step: {why}"]
        le = l2.item()
        if step.fused:                           # the one-kernel InfoNCE against the streaming sweeps: summation order
            ok_l = (math.isnan(le) and math.isnan(lv)) or abs(le - lv) <= 2e-6 * abs(le) + 1e-6
            gfloor = abs(scale) * 1e-3 / (bT * max(A, 1))
            ok_g = math.isnan(le) or (e.grad - gv).abs().max().item() <= 2e-3 * max(e.grad.abs().max().item(), gfloor)
        else:
            ok_l = _same_bits(l2.detach(), ref.loss)
            ok_g = torch.allclose(e.grad, gv, rtol=3e-6, atol=0, equal_nan=True)
        if not (ok_l and ok_g):
            return [f"loss / gradient differ from the eager step (loss {lv} vs {le}): {why}"]
        if half and not (_same_bits(step.loss, ref.loss) and _same_bits(step.grad, ref.grad.to(embed.dtype))):
            return [f"half embed: loss or gradient differ from the fp32 twin's (rounded once): {why}"]
        if enq:
            for k in _BANK_NAMES:
                if not torch.equal(getattr(bank, k), getattr(bank_e, k)):
                    return [f"bank {k} differs from the eager trainer order: {why}"]
            if tensor and not torch.equal(bank.shadow, bank_e.shadow):
                return [f"bank shadow differs from the eager trainer order: {why}"]
        bad, A, ok, _ = score_step_replay(c, ref, step, embed32, labels, seg, pred, q_before, scale, check_sampling,
                                          cov, reached, prev_A, why)
        if bad is not None:
            return [bad]
        scored += ok
        prev_A = A
    for s in steps:
        if int(s.counter.item()) != n_rep:
            return [f"step counter {int(s.counter.item())} after {n_rep} replays: {desc}"]
        if s.fused and int(s.ws.sync.abs().sum().item()) != 0:
            return [f"the fused kernels left their counters armed: {desc}"]
    if scored:
        for k, v in reached.items():
            cov[k] = cov.get(k, 0) + int(bool(v))
    return []


def _draw_graph_case(rng, it, scale):
    """Configuration of fuzz case `it`.  The step path cycles (fused full-fill, streaming bf16, exact fp32, fused
    sparse, any) so that few cases reach all of them; the rest is drawn.  Caps: B <= 2 scale (<= 8), h, w <= 32 scale, max_samples <= 300 scale
    (<= 1024, the fused kernel's limit)."""
    path = ("fused", "streaming", "exact", "fused", "any")[it % 5]
    seq = ("edge", "empty", "random")[it % 3]
    precision = "fp32" if path == "exact" else ("bf16" if path in ("fused", "streaming") else rng.choice(["fp32", "bf16"]))
    D = 256 if precision == "bf16" else rng.choice([32, 64, 128, 256])
    bank = "none" if path == "fused" else rng.choice(["none", "shadow", "enqueue"])
    normalize = path != "fused" and rng.random() < 0.25
    fused = None if path == "fused" else rng.choice([None, False])
    if path == "streaming" and bank == "none" and not normalize:
        fused = False
    ms_cap = min(1024, 300 * scale)
    ms = rng.choice([m for m in _MS_EDGES if m <= ms_cap]) if rng.random() < 0.6 else rng.randint(1, ms_cap)
    if seq == "edge" and ms < 129:               # room for A on both sides of a tile edge
        ms = rng.choice([m for m in _MS_EDGES if 129 <= m <= ms_cap])
    B = rng.randint(1, min(8, 2 * scale))
    if seq == "edge":            # few classes of many pixels: max_views ~ max_samples / 4 still leaves classes in
        h, w, K = rng.randint(20, 32 * scale), rng.randint(20, 32 * scale), rng.randint(2, 4)
        mv = rng.randint(max(1, ms // 6), max(1, ms // 3))
    else:
        h, w, K = rng.randint(4, 32 * scale), rng.randint(4, 32 * scale), rng.randint(2, 7)
        mv = rng.randint(1, 24 * scale)
    if rng.random() < 0.5:
        st = rng.choice([1, 2, 4])
        himg, wimg = h * st, w * st
    else:                                        # nearest down-sampling with a non-integer ratio
        himg, wimg = rng.randint(h, 3 * h + 2), rng.randint(w, 3 * w + 2)
    # bank rows: mostly enough columns for every anchor's diagonal column (2 M K >= max_samples), sometimes fewer
    M = rng.randint(2, 24 * scale) if rng.random() < 0.25 else -(-ms // (2 * K)) + rng.randint(0, 8)
    # enqueue: a label grid labels[:, ::s, ::s] with no more positions than feature columns, pixel_update_freq <= M
    stride = next(s for s in range(1, 64) if -(-himg // s) * -(-wimg // s) <= h * w)
    half = (torch.bfloat16, torch.float16)
    return dict(path=path, seq=seq, precision=precision, D=D, bank=bank, normalize=normalize, fused=fused,
                sparse=it % 5 == 3 or (it % 5 == 4 and rng.random() < 0.5), overlap=rng.random() < 0.5,
                embed_dtype=rng.choice([torch.float32, *half]),
                seg_dtype=None if rng.random() < 0.2 else rng.choice([torch.float32, *half]),
                grad_scale=rng.choice([1.0, 1.0, 0.37, -0.5, -2.0, 0.0]), nan_safe=rng.random() < 0.3,
                B=B, h=h, w=w, K=K, ms=ms, mv=mv, himg=himg, wimg=wimg, M=M, stride=stride, freq=rng.randint(1, M),
                T=rng.choice([0.07, 0.1, 0.5]), bT=0.07, block=rng.choice([2, 4, 8]), ignore=rng.choice([0.0, 0.1, 0.3]),
                n_rep=rng.randint(3, 4), seed=rng.randint(0, 10 ** 6))


def fuzz_graphed_step(seed: int, n: int, check_sampling, device="cpu", scale: int = 1):
    """GraphedContrastStep over random configurations (path, bank / enqueue, dtypes, grad_scale, nan_safe, sparse reset,
    overlapped fill, normalise, non-integer label ratios, max_samples around the tile edges), several replays with the
    static inputs refilled in place between them (graphed_step_case: eager step, float64 closed form, zeros outside the
    anchors, bank).  On a CPU the emulated kernels run the launch sequence eagerly (no capture, the fill branch
    inline); on a device nothing is patched: the replays are CUDA-graph replays.  Returns (failures, coverage): how many
    cases reached each of GRAPH_CATEGORIES, "scored" and "skipped" (replays the closed form scored / could not score)."""
    from contrastiveseg_b200 import graph_step
    rng = random.Random(seed)
    bad, cov = [], {k: 0 for k in GRAPH_CATEGORIES + ("scored", "skipped")}
    G = graph_step.GraphedContrastStep
    saved = (G._capture, G._fork_zero_fill, G._join_zero_fill)
    if torch.device(device).type == "cpu":
        G._capture = lambda self, warmup: None                 # no CUDA graphs on a CPU: run eagerly
        G._fork_zero_fill = lambda self: self._side_branch(0)
        G._join_zero_fill = lambda self: None
    try:
        for it in range(n):
            c = _draw_graph_case(rng, it, scale)
            desc = "graph seed={} it={} {}".format(seed, it, " ".join(f"{k}={v}" for k, v in c.items()))
            draw = graph_step_inputs(c["B"], c["D"], c["h"], c["w"], c["K"], c["himg"], c["wimg"], c["block"],
                                     c["ignore"], c["seq"], c["seed"])
            bad += graphed_step_case(c, draw, c["n_rep"], device, check_sampling, cov, desc)
    finally:
        G._capture, G._fork_zero_fill, G._join_zero_fill = saved
    return bad, cov


# ---- the captured criterion (GraphedContrastCriterion) ---------------------------------------------------------------
CRIT_COMBOS = ("ce", "ce_lovasz", "ce_ohem", "aux_ce", "aux_rmi", "aux_ohem", "mem_ce", "mem_rmi", "mem_lovasz",
               "mem_ohem")
CRIT_CATEGORIES = CRIT_COMBOS + ("CE one-call", "CE one-call above 24 classes", "CE two-call", "fp16 head",
                                 "bf16 head with two terms", "OHEM branch flip", "Lovasz present-set change",
                                 "all-ignored replay", "A = 0 replay", "bank + enqueue", "negative grad_scale",
                                 "set_grad_scale mid-case")
_HALF_EPS = {torch.bfloat16: torch.finfo(torch.bfloat16).eps, torch.float16: torch.finfo(torch.float16).eps}


def _pooled(n, s):
    return n if s == 1 else (n + 2 * (s // 2) - s) // s + 1


def _criterion_geometry(rng, c, mode, cap):
    """h, w, H, W (and B) of geometry `mode` ("up": integer factor, "nonint", "identity", "down": a label grid smaller
    than seg in one or both dimensions), B K H W within `cap`; c["refused"]: the terms refuse it (only the seg CE takes a
    label grid smaller than seg; RMI needs a pooled map of at least radius x radius)."""
    h, w = c["h0"], c["w0"]
    while True:
        if mode == "up":
            st = rng.choice([2, 3, 4])
            H, W = h * st, w * st
        elif mode == "nonint":
            H, W = rng.randint(h + 1, 3 * h + 2), rng.randint(w + 1, 3 * w + 2)
            H, W = H + (H % h == 0), W + (W % w == 0)
        elif mode == "identity":
            H, W = h, w
        else:
            which = rng.choice(["H", "W", "both"])
            H = rng.randint(max(1, h // 2), h - 1) if which != "W" else h * rng.choice([1, 2])
            W = rng.randint(max(1, w // 2), w - 1) if which != "H" else w * rng.choice([1, 2])
        if c["K"] * H * W <= cap or h <= 4 and w <= 4:
            break
        h, w = max(4, h * 3 // 4), max(4, w * 3 // 4)
    B = max(1, min(c["B0"], cap // (c["K"] * H * W)))
    refused = mode == "down" and c["name"] not in ("ce", "aux_ce", "mem_ce")
    if c["name"].endswith("rmi"):
        r, st = c["params"]["rmi_radius"], c["params"]["rmi_pool_stride"]
        refused = refused or min(_pooled(H, st), _pooled(W, st)) < r
    # enqueue: a label grid labels[:, ::s, ::s] with no more positions than feature columns
    stride = next(s for s in range(1, 64) if -(-H // s) * -(-W // s) <= h * w)
    c.update(mode=mode, h=h, w=w, H=H, W=W, B=B, refused=refused, stride=stride)
    return c


def _draw_criterion_case(rng, it, scale, device):
    """Configuration of criterion fuzz case `it`: the wrapper x seg-term combination cycles through CRIT_COMBOS; case 0
    draws K above 24 with integer up-sampling (the one-call seg CE of several class chunks), case 5 on a device K >= 150,
    cases 3 and 4 a label grid smaller than seg (the two-call seg CE; RMI refuses it); cases 1 (bf16 seg: a bf16 head
    with two terms), 6 (fp16 seg, bank with enqueue) and 2 (negative grad_scale) pin what the categories need, the rest
    is drawn.  Caps: B <= 2 scale (<= 8), h, w <= 12 scale (<= 128), max_samples <= 96 scale (<= 1024); on a device
    case 0 takes max_samples = 1024.  The aux weight is never 1 and the grad_scale set mid-case never 0, so a
    coefficient lost on the way to a term shows."""
    cuda = torch.device(device).type == "cuda"
    name = CRIT_COMBOS[it % len(CRIT_COMBOS)]
    K = rng.randint(25, 40) if it == 0 else (rng.randint(150, 171) if it == 5 and cuda else rng.randint(2, 24))
    hw = min(128, 12 * scale) if K < 150 else 24
    ms = min(1024, 96 * scale)
    ms = rng.choice([m for m in _MS_EDGES if m <= ms]) if rng.random() < 0.5 else rng.randint(1, ms)
    if cuda and it == 0:
        ms = 1024
    half = [torch.float32, torch.bfloat16, torch.float16]
    ohem_sum = name in ("ce_ohem", "mem_ohem") and rng.random() < 0.5
    params = dict(ce_ignore_index=rng.choice([-1, 255]), rmi_radius=rng.randint(1, 4), rmi_pool_way=rng.randint(0, 1),
                  lambda_way=rng.randint(0, 1), ce_reduction="sum" if ohem_sum else "elementwise_mean")
    params["rmi_pool_stride"] = params["rmi_pool_size"] = rng.randint(1, 4)
    if rng.random() < 0.4:
        params["ce_weight"] = [round(0.5 + rng.random(), 3) for _ in range(K)]
    n_rep = rng.randint(3, 4)
    all_ignored = it in (1, 2) or rng.random() < 0.3
    c = dict(name=name, K=K, h0=rng.randint(4, hw), w0=rng.randint(4, hw), B0=rng.randint(1, min(8, 2 * scale)),
             D=rng.choice([32, 64, 256]) if cuda else 32, ms=ms, mv=rng.randint(1, min(100, 16 * scale)),
             seq=("edge", "empty", "random")[it % 3], block=rng.choice([2, 4, 8]), ignore=rng.choice([0.0, 0.1, 0.3]),
             params=params, lw={"seg_loss": rng.choice([1.0, 0.7]), "aux_loss": rng.choice([0.4, 0.25, 1.5])},
             seg_dtype=torch.bfloat16 if it == 1 else (torch.float16 if it == 6 else rng.choice(half)),
             aux_dtype=rng.choice(half), embed_dtype=rng.choice([torch.float32, torch.bfloat16]),
             bank=("enqueue" if it == 6 else rng.choice(["read", "enqueue"])) if name.startswith("mem") else "none",
             grad_scale=-0.5 if it == 2 else rng.choice([1.0, 0.37, -0.5, -2.0, 0.0]),
             scale2=rng.choice([2.0, -1.0, 0.5, -0.25]), n_rep=4 if all_ignored else n_rep,
             all_ignored=all_ignored, seed=rng.randint(0, 10 ** 6), T=None, bT=None,
             precision="fp32", normalize=False, nan_safe=False, ignore_label=params["ce_ignore_index"])
    c["r_set"] = rng.randint(1, c["n_rep"] - 1)
    c["M"] = -(-ms // (2 * K)) + rng.randint(0, 8)
    c["freq"] = rng.randint(1, c["M"])
    cap = (2 * 10 ** 6 if name.endswith("rmi") else 8 * 10 ** 6) if cuda else 8 * 10 ** 4
    mode = "up" if it == 0 else ("down" if it in (3, 4) else rng.choice(["up", "nonint", "identity", "down"]))
    return _criterion_geometry(rng, c, mode, cap), cap


def criterion_inputs(c):
    """inputs(r): the CPU (embed, target, seg, seg_aux) of replay r, on graph_step_inputs's label sequence (A = 0 on
    replay 1 of "empty", one class on the odd replays of "edge") with: replay 1 of "random" without the first labelled
    class of replay 0 (it comes back on replay 2), replay 3 with every label ignored when c["all_ignored"], and for
    OHEM three quarters of replay 1's labels ignored: with min_kept at half the count under the threshold of replay 0,
    too few pixels lie under it and the select branch runs, where the other replays take the threshold branch.  Ignored
    labels are c's ignore index."""
    ign = c["params"]["ce_ignore_index"]
    base = graph_step_inputs(c["B"], c["D"], c["h"], c["w"], c["K"], c["H"], c["W"], c["block"], c["ignore"],
                             c["seq"], c["seed"])
    gone = []

    def inputs(r):
        d = base(r)
        t = d["target"]
        if r == 0 and bool((t >= 0).any()):
            gone.append(int(t[t >= 0][0]))
        if c["seq"] == "random" and r == 1 and gone:
            t[t == gone[0]] = -1
        if c["all_ignored"] and r == 3:
            t.fill_(-1)
        if "ohem" in c["name"] and r == 1:
            t[torch.rand(t.shape, generator=torch.Generator().manual_seed(c["seed"] + 5)) < 0.75] = -1
        seg = d["seg"]
        if "ohem" in c["name"]:             # the logit range OHEM's bounds were measured on (test_gpu_ohem._inputs)
            seg = (torch.rand(seg.shape, generator=torch.Generator().manual_seed(c["seed"] + 7 * r)) * 2 - 1) * 4
        aux = seg * 0.5 + 0.3 * torch.randn(seg.shape, generator=torch.Generator().manual_seed(c["seed"] + r))
        t[t == -1] = ign
        return d["embed"], t, seg, aux
    return inputs


def _upsample_f64(s, H, W):
    """s (B, K, h, w) float64 bilinearly (align_corners=True) up-sampled to H x W at the source coordinates the fp32
    kernels sample (test_gpu_many_classes._bilinear_matrix): for non-integer ratios the exact coordinates differ by
    more than OHEM's gradient bound allows."""
    import test_gpu_many_classes as M
    my, mx = M._bilinear_matrix(s.shape[2], H, s.device), M._bilinear_matrix(s.shape[3], W, s.device)
    return torch.einsum("yh,bkhw,xw->bkyx", my, s, mx)


def _score_seg_term(t, x, target, gs, gap_frac):
    """One seg term of a replay against its float64 oracle on the values the head holds (x, fp32) and this replay's
    labels, at the term's bounds (those of its standalone tests).  t.loss / t.dseg: the engine's loss and gradient
    (times gs = grad_scale * coef).  Returns (failure or None, scored, loss_ref, gradient_ref * gs, gradient bound
    (absolute), loss bound (absolute), (B, h, w) mask of the positions the gradient bound does not cover or None,
    OHEM branch or None)."""
    from oracle.lovasz_port import footprint_mask, lovasz_loss_and_grad
    from oracle.ohem_port import ohem_loss
    from oracle.rmi_port import rmi_loss_and_grad
    import test_gpu_many_classes as M
    B, K, h, w = x.shape
    lv, d = t.loss.item(), t.dseg.double()
    unscored = (None, False, None, None, None, None, None, None)
    zero_ok = torch.count_nonzero(t.dseg).item() == 0
    mask = branch = None
    if t.kind == "ce":
        s = x.double().requires_grad_(True)
        wt = None if t.weight is None else t.weight.double()
        ref = M.seg_ce_reference(s, target, wt, t.ignore)
        lref = ref.item()
        if not bool((target != t.ignore).any()):          # every pixel ignored: NaN, zero gradient
            if not (math.isnan(lv) and zero_ok):
                return (f"seg CE, every pixel ignored: loss {lv}, {torch.count_nonzero(t.dseg).item()} gradient "
                        "elements not 0",) + unscored[1:]
            return None, True, float("nan"), torch.zeros_like(d), 0.0, 0.0, None, None
        if math.isnan(lref):
            return unscored
        ref.backward()
        gref = s.grad * gs
        gmax = gref.abs().max().item()
        gbound, lbound = 1e-5 * gmax, 2e-6 * abs(lref)
    elif t.kind == "lovasz":
        lref, gref, near = lovasz_loss_and_grad(x, target, 1.0, ignore_index=t.ignore, near_tie_ulps=64)
        lref, gref = lref.item(), gref * gs
        gmax = gref.abs().max().item()
        gbound, lbound = 1e-4 * gmax, 1e-5 * max(abs(lref), 1e-6)
        mask = footprint_mask(near, h, w)
        if gmax > 0:
            if bool(mask.float().mean() > 0.5):           # near-tie footprints cover more than half the positions
                return unscored
            fro = ((d - gref).norm() / gref.norm()).item()
            if fro > 1.7e-4:
                return (f"Lovasz gradient: relative Frobenius error {fro:.2e}",) + unscored[1:]
    elif t.kind == "ohem":
        from contrastiveseg_b200.functional import ohem_selection
        red = ("mean", "sum")[t.red]
        kw = dict(weight=t.weight, ignore_index=t.ignore, thresh=t.thresh, min_kept=t.min_kept, reduction=red)
        s = x.double().requires_grad_(True)
        dd = ohem_loss(_upsample_f64(s, *target.shape[1:]), target, details=True, **kw)
        dd["loss"].backward()
        gref = s.grad
        sel = ohem_selection(x, target, t.weight, t.ignore, t.thresh, t.min_kept, red)
        branch = sel["branch"]
        if not (sel["n"] == dd["n"] and sel["count"] == dd["count"] and torch.equal(sel["selected"], dd["selected"])):
            return (f"OHEM selection: n {sel['n']} / {dd['n']}, count {sel['count']} / {dd['count']}",) + unscored[1:]
        if gap_frac < 0.5:                                # the gap ignored more than half the counted pixels
            return unscored
        lref, gref = dd["loss"].item(), gref * gs
        if math.isnan(lref):                              # mean of an empty selection: NaN, zero gradient
            if dd["n"] == 0 or dd["count"] != 0 or red != "mean":
                return unscored
            if not (math.isnan(lv) and zero_ok):
                return (f"OHEM, empty selection: loss {lv}, gradient not 0",) + unscored[1:]
            return None, True, lref, torch.zeros_like(d), 0.0, 0.0, None, branch
        gmax = gref.abs().max().item()
        gbound, lbound = 3.8e-6 * gmax, 2.1e-7 * abs(lref)
    else:                                                 # rmi
        r_, way, st, lam, lway, lw = t.params
        kw = dict(num_classes=K, radius=r_, pool_way=way, pool_stride=st, weight_lambda=lam, lambda_way=lway,
                  loss_weight=lw)
        try:
            lref, gref = rmi_loss_and_grad(x, target, 1.0, **kw)
            _, g32 = rmi_loss_and_grad(x, target, 1.0, front=torch.float32, **kw)
        except RuntimeError:                              # a reference solve that is not positive definite
            return unscored
        lref = lref.item()
        if not math.isfinite(lref):
            return unscored
        gmax0 = gref.abs().max().item()
        if gmax0 > 0 and bool(((g32 - gref).abs() <= 1e-4 * gmax0).float().mean() < 0.5):
            return unscored                               # the reference's own spread covers most elements
        spread = (g32 - gref).abs().max().item() * abs(gs)
        gref = gref * gs
        gmax = gref.abs().max().item()
        gbound, lbound = max(1e-4 * gmax, 4 * spread), 1e-5 * max(abs(lref), 1e-3)
    if abs(lv - lref) > lbound or math.isnan(lv):
        return (f"{t.kind} loss {lv} vs float64 {lref}",) + unscored[1:]
    if gmax == 0:
        if not zero_ok:
            return (f"{t.kind}: the float64 gradient is 0, {torch.count_nonzero(t.dseg).item()} elements are not",) + \
                unscored[1:]
    else:
        err = (d - gref).abs().amax(dim=1)                # (B, h, w): worst class plane
        if mask is not None:
            err = err[~mask]
        if err.numel() and err.max().item() > gbound:
            return (f"{t.kind} gradient: max error {err.max().item():.3e}, bound {gbound:.3e}",) + unscored[1:]
    return None, True, lref, gref, gbound, lbound, mask, branch


def graphed_criterion_case(c, device, check_sampling, cov, desc):
    """One GraphedContrastCriterion (configuration `c`), c["n_rep"] replays, the target, every head and embed refilled
    in place from criterion_inputs before each replay (OHEM's target gapped first, so fp32 and float64 select the same
    pixels), grad_scale changed with set_grad_scale before replay c["r_set"].  Every replay: the loss equals the eager
    seg terms plus loss_weight times a twin GraphedContrastStep to the bit, the embed gradient is the twin's (rounded once
    for bf16 embed), each head within _close of the eager gradient, a bank written by the step equals the twin bank
    after the eager enqueue; the contrast half is scored as fuzz_graphed_step's replays (score_step_replay), each seg
    term against its float64 oracle (_score_seg_term), the total loss and each head's gradient against the float64 sums
    within the terms' bounds combined.  A replay is scored when every part of it was.  Then apply() once.
    Returns the failures, or None when the geometry is refused as expected (c["refused"]; PclError asserted)."""
    from contrastiveseg_b200 import bank as bank_mod
    from oracle.ohem_port import gap_labels
    import test_gpu_graphed_criterion as TG
    import test_gpu_ohem as TO
    dev = torch.device(device)
    name, K, D, h, w = c["name"], c["K"], c["D"], c["h"], c["w"]
    aux, mem, ohem = name.startswith("aux"), name.startswith("mem"), "ohem" in name
    heads = ["seg", "seg_aux"] if aux else ["seg"]
    dtypes = {"seg": c["seg_dtype"], "seg_aux": c["aux_dtype"]}
    ign = c["params"]["ce_ignore_index"]
    inputs = criterion_inputs(c)
    e0, t0, s0, a0 = inputs(0)
    params = dict(c["params"])
    if ohem:           # OHEM's thresh and min_kept from replay 0's logits as the head holds them: the threshold branch there
        x0, tt = s0.to(dtypes["seg"]).float().to(dev), t0.to(dev)
        thresh = TO.median_thresh(x0, tt, ign) if bool(((tt != ign)).any()) else 0.5
        params.update(ohem_thresh=thresh, ohem_minkeep=TO.branch_min_kept(x0, tt, "threshold", thresh, ign))
    crit = TG.make_criterion(name, ms=c["ms"], extra={"max_views": c["mv"]}, K=K, params=params,
                             loss_weights=c["lw"]).to(dev)
    cc = crit.contrast_criterion
    c.update(T=cc.temperature, bT=cc.base_temperature)
    lw = crit.loss_weight
    ohem_mod = None
    if ohem:
        ohem_mod = crit.seg_criterion.ohem_ce_loss if aux else crit.seg_criterion
    gap_frac = [1.0]

    def gapped(t, seg):
        """OHEM: the target with the pixels whose p_t lies near the threshold ignored (gap_labels)."""
        if not ohem:
            return t
        x = _upsample_f64(seg.to(dtypes["seg"]).to(dev).double(), *t.shape[1:])
        t = t.to(dev)
        kw = dict(weight=ohem_mod.weight, thresh=ohem_mod.thresh, min_kept=ohem_mod.min_kept,
                  reduction=ohem_mod.reduction)
        g = gap_labels(x, t, ignore_index=ign, near_ulps=TO.NEAR_ULPS, **kw)
        n0 = int(((t != ign) & (t >= 0) & (t < K)).sum())
        gap_frac[0] = int(((g != ign) & (g >= 0) & (g < K)).sum()) / max(n0, 1) if n0 else 1.0
        return g.cpu()

    target = gapped(t0, s0).to(dev)
    static = {k: v.to(dev, dtypes[k]).requires_grad_(True) for k, v in (("seg", s0), ("seg_aux", a0)) if k in heads}
    static["embed"] = e0.to(dev, c["embed_dtype"]).requires_grad_(True)
    half_e = c["embed_dtype"] != torch.float32
    embed32 = static["embed"].detach().float() if half_e else static["embed"].detach()
    bank = twin_bank = enq = None
    if mem:
        b0 = make_bank(K, c["M"], D, c["seed"] + 1)

        def new_bank():
            mb = cs.MemoryBank(K, c["M"], D).to(dev)
            for k in _BANK_NAMES:
                getattr(mb, k).copy_(b0[k])
            return mb
        bank, twin_bank = new_bank(), new_bank()
        static["segment_queue"], static["pixel_queue"] = bank.segment_queue, bank.pixel_queue
        if c["bank"] == "enqueue":
            enq = dict(bank=bank, network_stride=c["stride"], pixel_update_freq=c["freq"], seed=c["seed"] % 997)
    scale = c["grad_scale"]
    try:
        gc_ = cs.GraphedContrastCriterion(crit, static, target, grad_scale=scale, enqueue=enq)
    except _abi.PclError as ex:
        return None if c["refused"] else [f"refused ({str(ex)[:100]}): {desc}"]
    if c["refused"]:
        return [f"a geometry the terms refuse was accepted: {desc}"]
    opts = cc.options()
    opts.num_classes = K
    twin = cs.GraphedContrastStep(embed32, target, seg=static["seg"].detach(), options=opts, grad_scale=scale * lw,
                                  segment_queue=twin_bank.segment_queue if mem else None,
                                  pixel_queue=twin_bank.pixel_queue if mem else None)
    # each head's coefficient in the seg loss, from the configuration (not from the wrapper's seg_terms)
    want = {"seg": c["lw"]["seg_loss"], "seg_aux": c["lw"]["aux_loss"]} if aux else {"seg": 1.0}
    reached, branches, present, prev_A = set(), [], [], None
    for r in range(c["n_rep"]):
        why = f"replay {r}: {desc}"
        if r:
            e, t, s, a = inputs(r)
            t = gapped(t, s)
            with torch.no_grad():
                static["embed"].copy_(e)
                if half_e:
                    embed32.copy_(static["embed"].float())
                target.copy_(t)
                for k, v in (("seg", s), ("seg_aux", a)):
                    if k in heads:
                        static[k].copy_(v.to(dtypes[k]))
        if r == c["r_set"]:
            scale = c["scale2"]
            gc_.set_grad_scale(scale)
            twin.set_grad_scale(scale * lw)
        q_before = torch.cat((twin_bank.segment_queue, twin_bank.pixel_queue), 1).double().cpu() if mem else None
        loss, grads = gc_.replay()
        twin.replay()
        _sync(dev)
        # the exact checks: the eager seg terms, the twin step, the eager trainer order of a bank write
        eager = {k: static[k].detach().clone().requires_grad_(True) for k in heads}
        seg_loss = crit._seg_loss(eager, target)
        seg_loss.backward(torch.full((), scale, device=dev))
        if enq:
            bank_mod._enqueue_counter[0] = r
            twin_bank.enqueue(embed32, target, network_stride=enq["network_stride"],
                              pixel_update_freq=enq["pixel_update_freq"], seed=enq["seed"])
        _sync(dev)
        if not _same_bits(loss, seg_loss.detach() + lw * twin.loss):
            return [f"loss {loss.item()} is not the eager seg loss {seg_loss.item()} + loss_weight x the twin step's "
                    f"{twin.loss.item()}: {why}"]
        if not _same_bits(grads["embed"], twin.grad.to(grads["embed"].dtype)):
            return [f"embed gradient differs from the twin step's: {why}"]
        for k in heads:
            parts = [t.dseg for t in gc_.terms if t.head == k]
            if not (grads[k].dtype == dtypes[k] and TG._close(grads[k], eager[k].grad, parts)):
                return [f"{k} gradient differs from the eager seg terms': {why}"]
        if enq:
            for k in _BANK_NAMES:
                if not torch.equal(getattr(bank, k), getattr(twin_bank, k)):
                    return [f"bank {k} differs from the eager trainer order: {why}"]
        # the contrast half against float64
        step_cov, step_reached = {}, {}
        bad, A, ok, lo = score_step_replay(c, twin, gc_.step, embed32, target, static["seg"].detach(), None, q_before,
                                           scale * lw, check_sampling, step_cov, step_reached, prev_A, why)
        if bad is not None:
            return [bad]
        prev_A = A
        scored = ok or A == 0
        # each seg term against its float64 oracle
        terms = []
        for t in gc_.terms:
            gs = scale * want[t.head]
            out = _score_seg_term(t, static[t.head].detach().float(), target, gs, gap_frac[0])
            if out[0] is not None:
                return [f"{out[0]}: {why}"]
            scored = scored and out[1]
            terms.append((t,) + out[2:])
        if not scored:
            cov["skipped"] += 1
            continue
        # the whole criterion: total loss and each head's gradient against the float64 sums, bounds combined
        coef = lambda t: want[t.head]                                       # noqa: E731
        lref = sum(coef(t) * lr for t, lr, *_ in terms) + lw * lo
        lbound = (sum(abs(coef(t)) * lb for t, _, _, _, lb, _, _ in terms) + abs(lw) * (2e-6 * abs(lo) + 1e-6) +
                  1e-6 * (sum(abs(coef(t) * lr) for t, lr, *_ in terms if not math.isnan(lr)) + abs(lw * lo)))
        lv = loss.item()
        if not ((math.isnan(lref) and math.isnan(lv)) or abs(lv - lref) <= lbound):
            return [f"total loss {lv} vs float64 {lref} (bound {lbound:.2e}): {why}"]
        for k in heads:
            mine = [tm for tm in terms if tm[0].head == k]
            gsum = sum(tm[2] for tm in mine)
            tol = sum(tm[3] for tm in mine)
            if dtypes[k] != torch.float32:              # each term's gradient cast to the head's dtype, then added
                eps, tiny = _HALF_EPS[dtypes[k]], torch.finfo(dtypes[k]).tiny
                # one rounding per cast and per add: eps / 2 relative, and half a subnormal step below fp16's normal
                # range (the gradients of a large label grid are small)
                tol = tol * (1 + eps) + eps * sum(tm[2].abs() for tm in mine) + 2 * len(mine) * tiny * eps
            err = (grads[k].double() - gsum).abs() - tol
            for tm in mine:
                if tm[5] is not None:                   # the Lovasz near-tie footprints
                    err = err.masked_fill(tm[5][:, None], 0.0)
            if bool((err > 0).any()):
                return [f"{k} gradient vs the float64 sum of its terms: {int((err > 0).sum())} elements out of bounds: "
                        f"{why}"]
        cov["scored"] += 1
        reached.add(name)
        for t in gc_.terms:
            if t.kind == "ce":
                reached.add("CE one-call" if t.one_call else "CE two-call")
                if t.one_call and K > 24:
                    reached.add("CE one-call above 24 classes")
        for k in heads:
            if dtypes[k] == torch.float16:
                reached.add("fp16 head")
            if dtypes[k] == torch.bfloat16 and sum(t.head == k for t in gc_.terms) > 1:
                reached.add("bf16 head with two terms")
        if c["all_ignored"] and r == 3:
            reached.add("all-ignored replay")
        if A == 0:
            reached.add("A = 0 replay")
        if enq:
            reached.add("bank + enqueue")
        if scale < 0:
            reached.add("negative grad_scale")
        if r == c["r_set"]:
            reached.add("set_grad_scale mid-case")
        branches += [tm[6] for tm in terms if tm[6] is not None]
        if any(t.kind == "lovasz" for t in gc_.terms):
            present.append(set(target[(target != ign) & (target >= 0) & (target < K)].unique().tolist()))
    # OHEM's branch flipped both ways: threshold -> select -> threshold over scored replays of the case
    if any(branches[i:i + 3] == ["threshold", "select", "threshold"] for i in range(len(branches) - 2)):
        reached.add("OHEM branch flip")
    if any(cl in present[i] and cl not in present[j] and any(cl in p for p in present[j + 1:])
           for i in range(len(present)) for j in range(i + 1, len(present)) for cl in present[i]):
        reached.add("Lovasz present-set change")
    # the autograd hand-off: apply() hands the heads and embed the buffers of its replay
    gc_.set_grad_scale(1.0)
    for k in heads + ["embed"]:
        static[k].grad = None
    gc_.apply(static).backward()
    _sync(dev)
    for k in heads + ["embed"]:
        if not _same_bits(static[k].grad, grads[k]):
            return [f"apply(): the {k} gradient is not the replay's: {desc}"]
    for k in reached:
        cov[k] += 1
    return []


def fuzz_graphed_criterion(seed: int, n: int, check_sampling, device="cpu", scale: int = 1):
    """GraphedContrastCriterion over every wrapper x seg-term combination the wrappers capture, with drawn term
    parameters, class counts, geometries, head / embed dtypes, bank, grad_scale (changed once per case), 3-4 replays per
    case with the labels, the heads and embed refilled in place (a class gone and back, every label ignored, OHEM's
    branch flipped, A = 0), each replay scored against float64 (graphed_criterion_case).  On a CPU the caller patches
    the capture out (the launch sequence runs eagerly); on a device nothing is patched.  Returns (failures, coverage):
    how many cases reached each of CRIT_CATEGORIES with a scored replay, "scored" / "skipped" replays and "refused"
    geometries (refusal asserted, then drawn again)."""
    import gc
    rng = random.Random(seed)
    bad, cov = [], {k: 0 for k in CRIT_CATEGORIES + ("scored", "skipped", "refused")}
    for it in range(n):
        c, cap = _draw_criterion_case(rng, it, scale, device)
        while True:
            desc = "criterion seed={} it={} {}".format(seed, it, " ".join(f"{k}={v}" for k, v in c.items()))
            out = graphed_criterion_case(c, device, check_sampling, cov, desc)
            if out is not None:
                break
            cov["refused"] += 1
            c = _criterion_geometry(rng, c, rng.choice(["up", "nonint", "identity"]), cap)
        bad += out
        if torch.device(device).type == "cuda":        # the float64 references of a case go back to the shared GPU
            gc.collect()
            torch.cuda.empty_cache()
    return bad, cov


def fuzz_trainer_hook(seed: int, n: int):
    """The whole hook of trainer_contrastive.py:209-255 over several iterations with an evolving bank, reference RNG
    stream (rng='torch_cpu', same torch seed on both sides): loss -> enqueue -> backward.  Loss, d/d seg, d/d embed and
    the bank after every iteration against the oracle — in particular the gradient must not see the rows the enqueue
    of the same iteration writes (the reference's autograd holds a copy of the bank; the engine holds the write back)."""
    rng = random.Random(seed)
    bad = []
    names = ("segment_queue", "segment_queue_ptr", "pixel_queue", "pixel_queue_ptr")
    for it in range(n):
        B, D, h, w, K = rng.randint(1, 2), rng.choice([32, 64]), rng.randint(6, 20), rng.randint(6, 20), rng.randint(3, 7)
        st, block, M, Fq = rng.choice([1, 2]), rng.choice([2, 4, 8]), rng.randint(6, 16), rng.randint(1, 5)
        ms, mv, warm, iters, sd = rng.randint(8, 80), rng.randint(1, 6), rng.randint(0, 2), rng.randint(2, 4), rng.randint(0, 10 ** 6)
        T, lw = rng.choice([0.07, 0.1]), 0.1
        desc = f"hook seed={seed} it={it} B={B} D={D} {h}x{w} K={K} stride={st} M={M} F={Fq} ms={ms} mv={mv} warmup={warm} iters={iters}"
        cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": st},
                           "loss": {"loss_type": "mem_contrast_ce_loss", "params": {"ce_ignore_index": -1}},
                           "contrast": {"temperature": T, "base_temperature": 0.07, "max_samples": ms, "max_views": mv,
                                        "loss_weight": lw, "use_rmi": False, "use_lovasz": False, "warmup_iters": warm,
                                        "with_memory": True, "memory_size": M, "pixel_update_freq": Fq, "rng": "torch_cpu"}})
        bank = cs.MemoryBank(K, M, D)
        b0 = make_bank(K, M, D, sd)
        for k in names:
            getattr(bank, k).copy_(b0[k])
        ref = [b0[k].clone().double() if "ptr" not in k else b0[k].clone() for k in names]
        hook = cs.ContrastTrainerHook(cfg, bank)
        ok = True
        for step in range(iters):
            data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=st, block=block, seed=sd + step)
            with_embed = step >= warm
            # reference side (float64), torch RNG stream seeded
            torch.manual_seed(sd + step)
            s64, e64 = data["seg"].double().requires_grad_(True), data["embed"].double().requires_grad_(True)
            try:
                lo = P.contrast_ce_loss({"seg": s64, "embed": e64, "segment_queue": ref[0], "pixel_queue": ref[2]},
                                        data["target"], with_embed=with_embed, loss_weight=lw, temperature=T,
                                        base_temperature=0.07, max_samples=ms, max_views=mv, with_memory=True)
                P.dequeue_and_enqueue(data["embed"].double(), data["target"], *ref, network_stride=st, memory_size=M,
                                      pixel_update_freq=Fq)
                lo.backward()
            except (RuntimeError, IndexError, ValueError):
                ok = None                       # degenerate draw (no class qualifies, A > bank columns, ...): skip the case
                break
            # engine side, same stream
            torch.manual_seed(sd + step)
            seg, emb = data["seg"].clone().requires_grad_(True), data["embed"].clone().requires_grad_(True)
            out = {"seg": seg, "embed": emb, "key": emb.detach(), "lb_key": data["target"]}
            loss = hook.loss_step(out, data["target"], iters=step)
            loss.backward()
            if math.isnan(lo.item()):
                if not math.isnan(loss.item()):
                    bad.append(f"reference NaN, engine {loss.item()} at iteration {step}: {desc}")
                ok = None
                break
            ge = (emb.grad.double() - e64.grad).abs().max().item() / max(e64.grad.abs().max().item(), 1e-9)
            gs = (seg.grad.double() - s64.grad).abs().max().item() / max(s64.grad.abs().max().item(), 1e-9)
            eb = max((bank.segment_queue.double() - ref[0]).abs().max().item(), (bank.pixel_queue.double() - ref[2]).abs().max().item())
            ptr_ok = torch.equal(bank.segment_queue_ptr, ref[1]) and torch.equal(bank.pixel_queue_ptr, ref[3])
            if _rel(loss.item(), lo.item()) > 5e-6 or ge > 3e-5 or gs > 3e-5 or eb > 3e-6 or not ptr_ok:
                bad.append(f"iteration {step}: rel={_rel(loss.item(), lo.item()):.1e} d_embed={ge:.1e} d_seg={gs:.1e} bank={eb:.1e} "
                           f"ptr_ok={ptr_ok}: {desc}")
                ok = False
                break
            # fp32 bank rows drift from the float64 reference by rounding only; re-align so the drift cannot accumulate
            ref[0], ref[2] = bank.segment_queue.double().clone(), bank.pixel_queue.double().clone()
    return bad


def fuzz_wrappers(seed: int, n: int):
    """ContrastCELoss / MemContrastCELoss end to end (fused up-sample + CE kernels for the seg half, pixel contrast on the
    reference RNG stream), warm-up and post-warm-up, optional class weights: loss, d/d seg, d/d embed vs the oracle."""
    from contrastiveseg_b200 import loss as loss_mod
    rng = random.Random(seed)
    bad = []
    saved = loss_mod.ContrastCELoss._can_fuse
    loss_mod.ContrastCELoss._can_fuse = lambda self, ce, s: self.fused_seg_ce and ce.ce_loss.reduction == "mean"
    try:
        for it in range(n):
            B, D, h, w, K = rng.randint(1, 2), rng.choice([32, 64]), rng.randint(5, 18), rng.randint(5, 18), rng.randint(2, 8)
            mem, with_embed, weighted = rng.random() < 0.5, rng.random() < 0.7, rng.random() < 0.4
            ms, mv, M, sd = rng.randint(8, 90), rng.randint(1, 8), rng.randint(4, 14), rng.randint(0, 10 ** 6)
            if rng.random() < 0.5:
                st = rng.choice([2, 4])
                himg, wimg = h * st, w * st
            else:
                himg, wimg = rng.randint(h, 3 * h + 2), rng.randint(w, 3 * w + 2)
            T, lw = rng.choice([0.07, 0.1]), rng.choice([0.1, 1.0])
            desc = (f"wrapper seed={seed} it={it} B={B} D={D} {h}x{w}->{himg}x{wimg} K={K} mem={mem} with_embed={with_embed} "
                    f"weighted={weighted} ms={ms} mv={mv}")
            data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=1, block=rng.choice([2, 4, 8]), seed=sd,
                                       himg=himg, wimg=wimg)
            bank = make_bank(K, M, D, sd + 1)
            g = torch.Generator().manual_seed(sd)
            cew = (torch.rand(K, generator=g) + 0.5) if weighted else None
            params = {"ce_ignore_index": -1, "ce_reduction": "elementwise_mean"}
            if weighted:
                params["ce_weight"] = cew.tolist()
            cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": 8}, "loss": {"params": params},
                               "contrast": {"temperature": T, "base_temperature": 0.07, "max_samples": ms, "max_views": mv,
                                            "loss_weight": lw, "use_rmi": False, "use_lovasz": False, "rng": "torch_cpu"}})
            crit = (cs.MemContrastCELoss if mem else cs.ContrastCELoss)(cfg)
            extra = {"segment_queue": bank["segment_queue"], "pixel_queue": bank["pixel_queue"]} if mem else {}
            torch.manual_seed(sd)
            s64, e64 = data["seg"].double().requires_grad_(True), data["embed"].double().requires_grad_(True)
            try:
                lo = P.contrast_ce_loss(dict({"seg": s64, "embed": e64}, **{k: v.double() for k, v in extra.items()}),
                                        data["target"], with_embed=with_embed, loss_weight=lw, temperature=T, base_temperature=0.07,
                                        max_samples=ms, max_views=mv, with_memory=mem, ce_weight=cew.double() if weighted else None)
                lo.backward()
            except (RuntimeError, IndexError, ValueError):
                continue
            torch.manual_seed(sd)
            seg, emb = data["seg"].clone().requires_grad_(True), data["embed"].clone().requires_grad_(True)
            loss = crit(dict({"seg": seg, "embed": emb}, **extra), data["target"], with_embed=with_embed)
            loss.backward()
            if math.isnan(lo.item()):
                if not math.isnan(loss.item()):
                    bad.append(f"reference NaN, engine {loss.item()}: {desc}")
                continue
            ge = (emb.grad.double() - e64.grad).abs().max().item() / max(e64.grad.abs().max().item(), 1e-9)
            gs = (seg.grad.double() - s64.grad).abs().max().item() / max(s64.grad.abs().max().item(), 1e-9)
            if _rel(loss.item(), lo.item()) > 5e-6 or ge > 3e-5 or gs > 3e-5:
                bad.append(f"mismatch rel={_rel(loss.item(), lo.item()):.1e} d_embed={ge:.1e} d_seg={gs:.1e}: {desc}")
    finally:
        loss_mod.ContrastCELoss._can_fuse = saved
    return bad


# ------------------------------------------------------------------------------------------------------------------
# the fused projection head (csrc/pcl_norm.cu): every fusion level, the dense and the anchor-column backward
# ------------------------------------------------------------------------------------------------------------------
HEAD_CATEGORIES = ("plain", "bn_relu", "conv1", "fp32", "bf16", "autocast", "train", "eval", "SyncBatchNorm",
                   "a bias None", "x without grad", "dense gzn", "column hand-off", "contrast loss", "fallback",
                   "all-dead deposit", "first / last pixel column", "n_cols at a tile edge", "A = 0",
                   "A = max_samples", "Cin at a 64 edge", "Cin 255-257", "HW = 1", "clamped pixel", "dead BN channel",
                   "large-mean channel", "weights changed", "control replay")
# Cin and H x W lean on the kernels' edges: 64-wide K-blocks and wgrad tiles, 256-channel bands (the column buffers'
# Cin + 1 row, k_col_prep's c += 256 loop, conv1's one-row bands at 257 / 513), BM = 128 pixel tiles, WB = 64
_HEAD_CIN = (16, 40, 63, 64, 65, 127, 128, 129, 191, 255, 256, 257, 300, 320)
_HEAD_CIN_DEV = (511, 512, 513, 720, 1023, 1024, 2048)
_HEAD_HW = (1, 2, 7, 63, 64, 65, 127, 128, 129, 191, 255, 256, 257)
_HEAD_NCOLS = (1, 63, 64, 65, 127, 128, 129)
_FALLBACK_PATTERNS = ("other_term", "two_losses", "retain_grad", "hook")

# Per-element bound of |kernel - float64 reference| (_head_bound), built in float64 from the operand magnitudes along
# the same chain, so that it scales with the shape instead of being measured at a few.  With u = 2^-24 and u_bf = 2^-8,
# the unit roundoffs of fp32 and bf16 (24 and 8 significant bits: rounding to nearest is off by at most half an ulp, u
# of the value), and gam(n) = n u / (1 - n u) (the classical bound of an n-term fp32 sum of products relative to the
# sum of their magnitudes):
#   * a GEMM product whose two operands the kernel rounds to bf16 and the reference may keep (u or W2 in fp32):
#     _RB = (1 + u_bf)^2 - 1 of |a||b|;
#   * a computed value that kernel and reference both round to bf16 (gz before the last conv's GEMMs, g_y before
#     conv1's): their inputs differ by rounding, so the two results can land on neighbouring bf16 values, one ulp,
#     _ULP = 2 u_bf = 2^-7 of the value;
#   * a value only the kernel rounds to bf16 (the fp32 columns the reference takes rounded, the stored bf16 zn the
#     backward reads): u_bf;
#   * the forward error reaches the backward through zn and inv_norm (|d zn| <= (|dz| + |zn| <|zn|, |dz|>) inv), the
#     BN terms through k1 = sum(g_u) / N and k2 = sum(g_u x_hat) / N;
#   * an element within PB.KINK of the ReLU's kink may take the other branch: its g_u is bounded by its full magnitude;
#   * the output's own rounding: u_bf of the value for bf16, 2u for fp32.
# Every step adds the errors of its inputs through the magnitudes of the other operands.  That is first order: the
# products of two errors it leaves out are below (2^-7)^2 of the terms, negligible next to the first-order ones.
_U32 = 2. ** -24
_UBF = 2. ** -8
_RB = (1 + _UBF) ** 2 - 1
_ULP = 2 * _UBF
_OUT = {torch.float32: 2 * _U32, torch.bfloat16: _UBF}
# The Frobenius norm of the error against that of the per-element bound: rounding errors of independent terms add up
# like a random walk, the bound like a worst case, so the error stays a small fraction of it (DESIGN §4 lists the ratios
# measured on an H100).
HEAD_FROB_FRACTION = 0.25


def _gam(n):
    return n * _U32 / (1. - n * _U32)


def _head_bound(c, x, w1, b1, bn0, w2, b2, g, y_stored, kink, out_dtype, n_rows):
    """{name: float64 per-element bound} of the head's outputs (see the constants above) for one call.  bn0: (training,
    gamma, beta, running_mean, running_var, eps) as the call saw them; y_stored: conv1's y as stored (conv1 level);
    kink: the reference's ReLU-kink mask; n_rows: the length of the pixel sums (B HW, or the live column count)."""
    d64 = lambda t: t.detach().double()                                             # noqa: E731
    B, C = x.shape[:2]
    P = x[0, 0].numel()
    X = (d64(x.to(torch.bfloat16)) if c["level"] != "bn_relu" else d64(x)).reshape(B, C, P)
    W2 = d64(w2).reshape(256, C)
    aW2 = W2.abs()
    absb2 = 0. if b2 is None else d64(b2).abs().view(1, 256, 1)
    n = max(n_rows, 1)
    out = {}
    if c["level"] == "plain":
        U, Eu = X, torch.zeros_like(X)
    else:
        training, gamma, beta, rm, rv, eps = bn0
        Y = X if c["level"] == "bn_relu" else d64(y_stored).reshape(B, C, P)
        if training:
            mean, var = Y.mean((0, 2)), Y.var((0, 2), unbiased=False)
        else:
            mean, var = d64(rm), d64(rv)
        invstd = 1. / torch.sqrt(var + eps)
        sc = (d64(gamma) * invstd).view(1, C, 1)
        sh = d64(beta).view(1, C, 1) - mean.view(1, C, 1) * sc
        A = Y * sc + sh
        mask = (A > 0).double()
        U = A.clamp_min(0.)
        Ea = 8 * _U32 * ((Y * sc).abs() + sh.abs())
        Eu = Ea * (A > -Ea)                     # below -Ea the ReLU gives an exact 0 on both sides
        XH = (Y - mean.view(1, C, 1)) * invstd.view(1, C, 1)
        Exh = 8 * _U32 * (Y.abs() + mean.abs().view(1, C, 1)) * invstd.view(1, C, 1)
        K = d64(kink).reshape(B, C, P).double()
    Z = torch.einsum("nc,bcp->bnp", W2, U) + (0. if b2 is None else d64(b2).view(1, 256, 1))
    Ez = (_RB + _gam(C + 1)) * (torch.einsum("nc,bcp->bnp", aW2, U.abs()) + absb2) + \
        torch.einsum("nc,bcp->bnp", aW2, Eu)
    nz = Z.norm(dim=1, keepdim=True)
    inv = 1. / nz.clamp_min(1e-12)
    ZN = Z * inv
    aZN = ZN.abs()
    rel_inv = (aZN * Ez).sum(1, keepdim=True) * inv                 # relative error of inv_norm
    Ezn = (Ez + aZN * (aZN * Ez).sum(1, keepdim=True)) * inv + _gam(256) * aZN        # + the norm's own sum
    out["zn"] = Ezn + _OUT[out_dtype] * aZN
    Ezn_used = Ezn + (_UBF if out_dtype == torch.bfloat16 else 0.) * aZN      # the backward reads the stored zn
    G = d64(g).reshape(B, 256, P)
    aG = G.abs()
    dot = (ZN * G).sum(1, keepdim=True)
    GZ = torch.where(nz < 1e-12, G * inv, (G - ZN * dot) * inv)
    MGZ = (aG + aZN * (aZN * aG).sum(1, keepdim=True)) * inv
    # the column path takes the loss's fp32 columns, the reference their rounding to zn's dtype: one more u_bf of g
    rg = _UBF if out_dtype == torch.bfloat16 else 0.
    Egz = (_ULP + _gam(256) + rg) * MGZ + inv * (Ezn_used * dot.abs() + aZN * (Ezn_used * aG).sum(1, keepdim=True)) + \
        GZ.abs() * rel_inv
    aGZ = GZ.abs()
    sum_p = lambda t: t.sum((0, 2)) if t.dim() == 3 else t                          # noqa: E731
    out_w = lambda E, V: E + _OUT[torch.float32] * V.abs()                           # noqa: E731
    GW2 = torch.einsum("bnp,bcp->nc", GZ, U)
    Egw2 = (_RB + _gam(n)) * torch.einsum("bnp,bcp->nc", aGZ, U.abs()) + torch.einsum("bnp,bcp->nc", Egz, U.abs()) + \
        torch.einsum("bnp,bcp->nc", aGZ, Eu)
    Egb2 = _gam(n) * sum_p(aGZ) + sum_p(Egz)
    wname, bname, xname = ("gw", "gb", "gx") if c["level"] == "plain" else \
        (("gw", "gb", "gy") if c["level"] == "bn_relu" else ("gw2", "gb2", "gx"))
    out[wname] = out_w(Egw2, GW2).view(256, C)
    out[bname] = out_w(Egb2, sum_p(GZ))
    MGU = torch.einsum("nc,bnp->bcp", aW2, aGZ)
    Ed = (_RB + _gam(256)) * MGU + torch.einsum("nc,bnp->bcp", aW2, Egz)
    if c["level"] == "plain":
        GX = torch.einsum("nc,bnp->bcp", W2, GZ)
        out["gx"] = (Ed + _OUT[out_dtype] * (GX.abs() + Ed)).reshape(x.shape)
        return out
    GU = torch.einsum("nc,bnp->bcp", W2, GZ) * mask
    Egu = mask * Ed + K * MGU
    aGU = GU.abs()
    N = B * P
    Egbeta = _gam(n) * sum_p(aGU) + sum_p(Egu)
    Eggamma = (_gam(n) + 8 * _U32) * sum_p(aGU * XH.abs()) + sum_p(Egu * XH.abs()) + sum_p(aGU * Exh)
    out["gbeta"] = out_w(Egbeta, sum_p(GU))
    out["ggamma"] = out_w(Eggamma, sum_p(GU * XH))
    if training:
        k1, k2 = (sum_p(GU) / N).view(1, C, 1), (sum_p(GU * XH) / N).view(1, C, 1)
        GY = sc * (GU - k1 - XH * k2)
        Egy = sc.abs() * (Egu + (Egbeta / N).view(1, C, 1) + XH.abs() * (Eggamma / N).view(1, C, 1) +
                          Exh * k2.abs() + 8 * _U32 * (aGU + k1.abs() + (XH * k2).abs()))
    else:
        GY = sc * GU
        Egy = sc.abs() * (Egu + 4 * _U32 * aGU)
    if c["level"] == "bn_relu":
        out["gy"] = (Egy + _OUT[out_dtype] * (GY.abs() + Egy)).reshape(x.shape)
        return out
    W1 = d64(w1.to(torch.bfloat16)).reshape(C, C)
    Egy_r = Egy + _ULP * GY.abs()                                   # g_y rounded to bf16 for conv1's GEMMs
    aGY = GY.abs()
    GX = torch.einsum("nc,bnp->bcp", W1, GY)
    Egx = _gam(C) * torch.einsum("nc,bnp->bcp", W1.abs(), aGY) + torch.einsum("nc,bnp->bcp", W1.abs(), Egy_r)
    out["gx"] = (Egx + _OUT[out_dtype] * (GX.abs() + Egx)).reshape(x.shape)
    out["gw1"] = out_w(_gam(n) * torch.einsum("bnp,bcp->nc", aGY, X.abs()) +
                       torch.einsum("bnp,bcp->nc", Egy_r, X.abs()),
                       torch.einsum("bnp,bcp->nc", GY, X)).view(C, C, 1, 1)
    out["gb1"] = out_w(_gam(n) * sum_p(aGY) + sum_p(Egy_r), sum_p(GY))
    return out


def _draw_head_case(rng, it, scale, device):
    """One case of fuzz_projection_head: the head, the geometry, the incoming gradient and the adversarial value.  The
    level, gradient source and adversarial value rotate with `it`, the rest is drawn."""
    dev = torch.device(device).type == "cuda"
    level = ("bn_relu", "conv1", "plain")[it % 3]
    grad = "dense" if level == "plain" else ("cols", "loss", "fallback", "dense")[(it - (it + 1) // 3) % 4]
    adv = (None, "clamped", "dead channel", "large mean", None)[(it // 2) % 5]
    if level == "plain" and adv in ("dead channel", "large mean"):
        adv = None
    c = dict(level=level, grad=grad, adv=adv, seed=rng.randint(0, 10 ** 6))
    c["act"] = ("fp32", "bf16", "autocast")[(it // 3) % 3] if level == "conv1" else rng.choice(["fp32", "bf16"])
    c["train"] = level != "plain" and (adv == "large mean" or rng.random() < 0.7)
    if adv == "clamped" and level == "conv1":
        c["train"] = False          # conv1's y at an all-zero x column is b1: only the running statistics place it
    c["sync"] = level != "plain" and rng.random() < 0.3
    c["momentum"] = rng.choice([0.1, 0.01, 0.5, 1.0])
    c["b1"] = level == "conv1" and rng.random() < 0.75
    c["b2"] = rng.random() < 0.75 if adv != "clamped" else rng.choice([False, "tiny"])
    c["x_grad"] = level != "conv1" or rng.random() < 0.75
    cins = _HEAD_CIN + (_HEAD_CIN_DEV if dev else ())
    if level == "conv1" and rng.random() < 0.3:
        cins = (257, 513) if dev else (257,)                     # conv1's one-row bands
    Cin = rng.choice(cins)
    cap = 200 * scale * scale if Cin <= 320 else 30 * scale * scale
    if not dev and it == 4:                                      # one wide case at a small image on the emulator
        Cin, cap = 720, 12
    if dev and it == 5:
        Cin = 2048
    hws = [h for h in _HEAD_HW if h <= cap and (h > 1 or not c["train"])]
    HW = 1 if it == 2 else rng.choice(hws)
    B = rng.randint(1, max(1, min(8, cap // HW)))
    if c["train"] and B * HW < 2:
        B = 2
    divs = [d for d in range(1, HW + 1) if HW % d == 0]
    H = rng.choice(divs)
    c.update(B=B, Cin=Cin, H=H, W=HW // H)
    if grad == "cols":
        c["n_cols"] = rng.choice(_HEAD_NCOLS + (rng.randint(2, 300),))
    if grad in ("loss", "fallback"):
        K = rng.randint(2, 6)
        c.update(K=K, precision=rng.choice(["fp32", "bf16"]), bank=rng.random() < 0.3,
                 ms=rng.choice([B * K, B * K, 2 * B * K, rng.randint(2, 200)]), mv=rng.choice([2, 2, 4, 100]))
    if grad == "fallback":
        c["pattern"] = _FALLBACK_PATTERNS[(it // 12) % 4] if rng.random() < 0.5 else rng.choice(_FALLBACK_PATTERNS)
    c["n_rep"] = rng.randint(2, 4)
    c["actions"] = [rng.choice(["inputs", "weights", "both", "both", "control"]) for _ in range(c["n_rep"] - 1)]
    return c


class _Head:
    """One copy of the fuzzed head: its leaves (w1, b1, gamma, beta, w2, b2), its BatchNorm and its call."""

    def __init__(self, c, init, sparse, device):
        import torch.nn as nn
        self.c, self.sparse = c, sparse
        C = c["Cin"]
        self.bn = None
        if c["level"] != "plain":
            self.bn = (nn.SyncBatchNorm(C) if c["sync"] else nn.BatchNorm2d(C)).to(device)
            self.bn.momentum = c["momentum"]
            with torch.no_grad():
                for k in ("weight", "bias", "running_mean", "running_var"):
                    getattr(self.bn, k).copy_(init[k])
            self.bn.train(c["train"])
        if c["level"] == "conv1":
            self.mod = cs.ProjectionHead(C, 256, "convmlp", bn_type="torchsyncbn" if c["sync"] else "torchbn",
                                         fused=True, fuse_bn_relu=True, fuse_conv1=True, sparse_grad=sparse).to(device)
            self.mod.proj[1][0] = self.bn
            conv1, conv2 = self.mod.proj[0], self.mod.proj[2]
            with torch.no_grad():
                conv1.weight.copy_(init["w1"])
                conv2.weight.copy_(init["w2"])
                for conv, k in ((conv1, "b1"), (conv2, "b2")):
                    if init[k] is None:
                        conv.register_parameter("bias", None)
                    else:
                        conv.bias.copy_(init[k])
            self.w1, self.b1, self.w2, self.b2 = conv1.weight, conv1.bias, conv2.weight, conv2.bias
        else:
            self.w1 = self.b1 = None
            self.w2 = init["w2"].clone().to(device).requires_grad_(True)
            self.b2 = None if init["b2"] is None else init["b2"].clone().to(device).requires_grad_(True)

    def leaves(self):
        ps = {"w1": self.w1, "b1": self.b1, "w2": self.w2, "b2": self.b2}
        if self.bn is not None:
            ps.update(gamma=self.bn.weight, beta=self.bn.bias)
        return {k: v for k, v in ps.items() if v is not None}

    def __call__(self, x):
        c = self.c
        if c["level"] == "plain":
            return cs.project_normalize(x, self.w2, self.b2)
        if c["level"] == "bn_relu":
            return cs.bn_relu_project_normalize(x, self.bn, self.w2, self.b2, sparse_grad=self.sparse)
        with torch.autocast(x.device.type, dtype=torch.bfloat16, enabled=c["act"] == "autocast"):
            return self.mod(x)

    def grads(self, x):
        names = {"plain": {"w2": "gw", "b2": "gb"}, "bn_relu": {"w2": "gw", "b2": "gb"},
                 "conv1": {"w1": "gw1", "b1": "gb1", "w2": "gw2", "b2": "gb2"}}[self.c["level"]]
        out = {names[k]: p.grad for k, p in self.leaves().items() if k in names}
        if self.bn is not None:
            out.update(ggamma=self.bn.weight.grad, gbeta=self.bn.bias.grad)
        if x.requires_grad:
            out["gy" if self.c["level"] == "bn_relu" else "gx"] = x.grad
        return out

    def absent(self, x_grad):
        """The outputs this head has none of: the gradient of a bias that is None, x's when x needs none."""
        conv1 = self.c["level"] == "conv1"
        out = set()
        if self.b2 is None:
            out.add("gb2" if conv1 else "gb")
        if conv1 and self.b1 is None:
            out.add("gb1")
        if not x_grad:
            out.add("gy" if self.c["level"] == "bn_relu" else "gx")
        return out

    def zero_grad(self, x):
        for p in list(self.leaves().values()) + [x]:
            p.grad = None

    def buffers(self):
        return {} if self.bn is None else {k: getattr(self.bn, k).clone() for k in ("running_mean", "running_var",
                                                                                     "num_batches_tracked")}


def _head_init(c, g):
    C = c["Cin"]
    init = {"w1": torch.randn(C, C, 1, 1, generator=g) / C ** 0.5, "b1": 0.5 * torch.randn(C, generator=g),
            "weight": 1 + 0.2 * torch.randn(C, generator=g), "bias": 0.2 * torch.randn(C, generator=g),
            "running_mean": 0.3 * torch.randn(C, generator=g), "running_var": 0.5 + torch.rand(C, generator=g),
            "w2": torch.randn(256, C, 1, 1, generator=g) / C ** 0.5, "b2": 0.1 * torch.randn(256, generator=g)}
    if not c["b1"]:
        init["b1"] = None
    if c["b2"] == "tiny":           # z = b2 at the clamped pixel: |z| = 0.95 eps, F.normalize's clamped branch with
        b2 = torch.randn(256, generator=g)      # |zn| = 0.95, where projecting gzn would change its gradient
        init["b2"] = b2 * (0.95e-12 / b2.norm())
    elif not c["b2"]:
        init["b2"] = None
    if c["adv"] == "clamped":
        init["weight"] = init["weight"].abs().clamp(0.9, 1.5)
        init["bias"] = init["bias"].clamp(-0.3, 0.3)
        if c["level"] == "conv1":   # y = b1 at the all-zero x column, 4 running standard deviations below the mean
            init["b1"] = init["running_mean"] - 4 * torch.sqrt(init["running_var"] + 1e-5)
    if c["adv"] == "dead channel":
        init["bias"][0] = -1e3
    if c["adv"] == "large mean" and c["level"] == "conv1":
        if init["b1"] is None:
            init["b1"] = torch.zeros(C)
            c["b1"] = True
        init["b1"][0] = 1000.
    return init


def _head_x(c, init_bn, g, pix):
    """x for one replay (fp32, CPU), with the case's adversarial value; pix = (b, p) of the clamped pixel."""
    B, C, H, W = c["B"], c["Cin"], c["H"], c["W"]
    x = torch.randn(B, C, H, W, generator=g)
    if c["level"] == "bn_relu":
        x = x * (0.5 + torch.rand(1, C, 1, 1, generator=g)) + 0.5 * torch.randn(1, C, 1, 1, generator=g)
    if c["adv"] == "large mean" and c["level"] == "bn_relu":
        x[:, 0] += 1000.
    if c["adv"] == "clamped":
        b, p = pix
        xv = x.view(B, C, H * W)
        if c["level"] == "bn_relu":   # every BN output of the pixel below 0: 4 standard deviations under the others
            if c["train"]:
                others = torch.cat([xv[:b].transpose(0, 1).reshape(C, -1), xv[b, :, :p], xv[b, :, p + 1:],
                                    xv[b + 1:].transpose(0, 1).reshape(C, -1)], 1)
                xv[b, :, p] = others.min(1).values - 4 * (others.std(1, unbiased=False) + 1)
            else:
                xv[b, :, p] = init_bn[0] - 4 * torch.sqrt(init_bn[1] + 1e-5)
        else:
            xv[b, :, p] = 0.
    return x


def _head_cols(c, g, live, pix, n_px):
    """Static column buffers of n_cols entries: `live` distinct pixels (the clamped pixel and, when there is room, the
    first and last pixel of the batch among them) at shuffled slots, the rest dead (-1); bf16-exact values."""
    n = c["n_cols"]
    q = torch.randperm(n_px, generator=g)[:live]
    if live:
        forced = ([pix[0] * c["H"] * c["W"] + pix[1]] if c["adv"] == "clamped" else []) + [0, n_px - 1]
        forced = torch.tensor(list(dict.fromkeys(forced)))
        q = torch.cat([forced, q[~torch.isin(q, forced)]])[:live]
    col_pix = torch.full((n,), -1, dtype=torch.int32)
    slots = torch.randperm(n, generator=g)[:live]
    col_pix[slots] = q.to(torch.int32)
    cols = torch.randn(n, 256, generator=g).to(torch.bfloat16).float()
    cols[col_pix < 0] = torch.randn(int((col_pix < 0).sum()), 256, generator=g).to(torch.bfloat16).float()
    return cols, col_pix


def _head_reference(c, x, h, gzn):
    """The float64 chain of the case's level (test_gpu_projection*.py), with a bias that is None taken as zeros: the
    outputs, the BN statistics (or None) and conv1's stored y (or None)."""
    import test_gpu_projection as TP
    import test_gpu_projection_bnrelu as TPB
    import test_gpu_projection_conv1 as TPC
    z = lambda b, n: torch.zeros(n, device=x.device) if b is None else b.detach()       # noqa: E731
    w2, b2 = h.w2.detach(), z(h.b2, 256)
    if c["level"] == "plain":
        return TP._reference(x, w2, b2, gzn, True), None, None
    if c["level"] == "bn_relu":
        ref, st = TPB._reference(x, h.bn, w2, b2, gzn)
        return ref, st, None
    b1 = z(h.b1, c["Cin"])
    ref, st = TPC.head_reference(x, h.w1.detach(), b1, h.bn, w2, b2, gzn)
    return ref, st, TPC.conv1_abi(x, h.w1.detach(), b1)["y"]


def _score_head(got, ref, bound, absent, worst, where):
    """Every output within its per-element bound and the Frobenius fraction; worst[name] keeps the largest ratio.  Only
    the outputs in `absent` (a bias that is None, x without a gradient) may be missing, and those must be."""
    bad = []
    for k, b in bound.items():
        if (got.get(k) is None) != (k in absent):
            bad.append(f"{where}: {k} {'missing' if k not in absent else 'written although the case has none'}")
            continue
        if k in absent:
            continue
        d = (got[k].double().reshape(-1) - ref[k].double().reshape(-1)).abs()
        b = b.reshape(-1)
        if not bool(torch.isfinite(d).all()):
            bad.append(f"{where}: {k} not finite")
            continue
        ratio = (d / b.clamp_min(1e-300)).max().item()
        frob = (d.norm() / b.norm().clamp_min(1e-300)).item()
        worst[k] = max(worst.get(k, 0.), ratio)
        worst["frob " + k] = max(worst.get("frob " + k, 0.), frob)
        if ratio > 1. or frob > HEAD_FROB_FRACTION:
            bad.append(f"{where}: {k} error/bound {ratio:.3g} (Frobenius {frob:.3g})")
    return bad


def _loss_options(c, r, k=0):
    g = torch.Generator().manual_seed(c["seed"] + 1000 * r + k)
    return cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=c["ms"], max_views=c["mv"],
                              precision=c["precision"], rng="torch_cpu", num_classes=c["K"], nan_safe=True,
                              perm_fn=lambda n: torch.randperm(n, generator=g))


def _head_loss(c, zn, lab, r):
    """The contrast loss on zn (c), or the case's fallback consumer pattern (d)."""
    target, seg, bank = lab
    kw = dict(seg=seg, segment_queue=bank[0], pixel_queue=bank[1]) if bank else dict(seg=seg)
    pat = c.get("pattern") if c["grad"] == "fallback" else None
    if pat == "retain_grad":
        zn.retain_grad()
    if pat == "hook":
        zn.register_hook(lambda g: g * 1.0)
    loss = cs.pixel_contrast_loss(zn, target, options=_loss_options(c, r), **kw)
    if pat == "other_term":
        loss = loss + (zn.float() ** 2).mean()
    if pat == "two_losses":
        loss = loss + 0.5 * cs.pixel_contrast_loss(zn, target, options=_loss_options(c, r, 1), **kw)
    return loss


def head_case(c, device, cov, worst, desc, calls):
    """One case of fuzz_projection_head: n_rep replays with inputs and weights changed in place between them, each
    scored against float64 (_head_bound), the column path against the dense head fed the same gradient, the fallbacks
    against the dense head bit for bit, and on a device the captured forward + backward of (a) / (b) against eager
    calls bit for bit.  calls: the wrapper's record of _bn_head_backward_cols calls."""
    dev = torch.device(device).type == "cuda"
    g = torch.Generator().manual_seed(c["seed"])
    init = _head_init(c, g)
    B, C, H, W = c["B"], c["Cin"], c["H"], c["W"]
    n_px = B * H * W
    xdt = torch.bfloat16 if c["act"] == "bf16" else torch.float32
    zdt = torch.float32 if c["act"] == "fp32" else torch.bfloat16
    sparse = c["grad"] != "dense"
    E = _Head(c, init, sparse, device)
    D = _Head(c, init, False, device) if sparse else None
    Gh = _Head(c, init, sparse, device) if dev and c["grad"] in ("dense", "cols") else None
    pix = (int(torch.randint(B, (1,), generator=g)), int(torch.randint(H * W, (1,), generator=g)))
    n_rep = c["n_rep"]
    actions = ["inputs"] + list(c["actions"])
    if c["grad"] in ("cols", "loss") and actions[-1] in ("weights", "control"):
        actions[-1] = "both"                            # the last replay: every column dead / A = 0
    bank = None
    if c["grad"] in ("loss", "fallback") and c["bank"]:
        bk = make_bank(c["K"], 12, 256, c["seed"] + 7)
        bank = (bk["segment_queue"].to(device), bk["pixel_queue"].to(device))
    heads = [h for h in (E, D, Gh) if h is not None]
    graph = x_s = gzn_s = cols_s = pix_s = zn_g = None
    lab = None
    bad = []
    reached = set()
    for r in range(n_rep):
        act = actions[r]
        where = f"replay {r} ({act}): {desc}"
        if act in ("inputs", "both"):
            x_new = _head_x(c, (init["running_mean"], init["running_var"]), g, pix).to(device=device, dtype=xdt)
            if c["grad"] == "dense":
                gzn_new = torch.randn(B, 256, H, W, generator=g).to(device=device, dtype=zdt)
            if c["grad"] == "cols":
                last = r == n_rep - 1
                live = 0 if last else int(torch.randint(1, min(c["n_cols"], n_px) + 1, (1,), generator=g))
                cols_new, pix_new = _head_cols(c, g, live, pix, n_px)
                cols_new, pix_new = cols_new.to(device), pix_new.to(device)
            if c["grad"] in ("loss", "fallback"):
                data = make_contrast_batch(B=B, D=8, h=H, w=W, num_classes=c["K"], img_stride=1,
                                           block=int(torch.randint(1, 5, (1,), generator=g)), seed=c["seed"] + r)
                target = data["target"].clone()
                if c["grad"] == "loss" and r == n_rep - 1:
                    target.fill_(-1)                            # no class qualifies: A = 0
                lab = (target.to(device), data["seg"].to(device), bank)
            if x_s is None:
                x_s = x_new.clone().requires_grad_(c["x_grad"])
                gzn_s = gzn_new.clone() if c["grad"] == "dense" else None
                if c["grad"] == "cols":
                    cols_s, pix_s = cols_new.clone(), pix_new.clone()
            else:
                with torch.no_grad():
                    x_s.copy_(x_new)
                    if c["grad"] == "dense":
                        gzn_s.copy_(gzn_new)
                    if c["grad"] == "cols":
                        cols_s.copy_(cols_new)
                        pix_s.copy_(pix_new)
        if act in ("weights", "both"):
            reached.add("weights changed")
            with torch.no_grad():                               # an optimizer step, the same on every copy
                for k, p in E.leaves().items():
                    step = 0.05 * torch.randn(p.shape, generator=g).to(device) * p.detach().abs().mean()
                    for h in heads:
                        h.leaves()[k].add_(step)
        if act == "control":
            reached.add("control replay")
        if Gh is not None and graph is None:                    # warm up on a side stream, then capture
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for h in (Gh, E):
                    xw = x_s.detach().clone().requires_grad_(c["x_grad"])
                    zw = h(xw)
                    zw.backward(gzn_s if c["grad"] == "dense" else Fn._sink_of(zw).deposit(cols_s, pix_s, zw.shape))
                    h.zero_grad(xw)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            if D is not None and D.bn is not None:              # the dense twin starts from the warmed-up buffers
                for k, v in E.buffers().items():
                    getattr(D.bn, k).copy_(v)
            Gh.zero_grad(x_s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                zn_g = Gh(x_s)
                zn_g.backward(gzn_s if c["grad"] == "dense" else Fn._sink_of(zn_g).deposit(cols_s, pix_s, zn_g.shape))
        # the eager call (and the reference, from the state the call starts from)
        bn0 = None if E.bn is None else (E.bn.training, E.bn.weight.detach().clone(), E.bn.bias.detach().clone(),
                                          E.bn.running_mean.clone(), E.bn.running_var.clone(), E.bn.eps)
        nbt0 = None if E.bn is None else int(E.bn.num_batches_tracked.item())
        x_ref = x_s.detach().to(torch.bfloat16) if c["act"] == "autocast" else x_s.detach()
        xe = x_s.detach().clone().requires_grad_(c["x_grad"])
        n_calls = len(calls)
        zn = E(xe)
        loss = None
        if c["grad"] == "dense":
            gref = gzn_s
            zn.backward(gzn_s)
        elif c["grad"] == "cols":
            zn.backward(Fn._sink_of(zn).deposit(cols_s, pix_s, zn.shape))
        else:
            loss = _head_loss(c, zn, lab, r)
            if c["grad"] == "loss":
                A = int(Fn.last_workspace(zn.device).plan[_abi.PLAN_A].item())
                reached.add("A = 0" if A == 0 else ("A = max_samples" if A == c["ms"] else "contrast loss"))
            loss.backward()
        _sync(device)
        took_cols = len(calls) - n_calls
        want = 1 if c["grad"] in ("cols", "loss") else 0
        if took_cols != want:
            bad.append(f"{where}: the column path ran {took_cols} times, expected {want}")
            break
        got = E.grads(xe)
        got["zn"] = zn.detach()
        if c["grad"] in ("cols", "loss"):
            cols, cpix = calls[-1]
            live = cpix[cpix >= 0].long()
            if live.numel() == 0:
                reached.add("all-dead deposit")
            if live.numel() and (int(live.min()) == 0 or int(live.max()) == n_px - 1):
                reached.add("first / last pixel column")
            gref = Fn._with_deposits(torch.zeros(zn.shape, dtype=zdt, device=device), [(cols, cpix)], zdt)
        if c["grad"] == "fallback":
            gref = torch.zeros(zn.shape, dtype=zdt, device=device)      # the BN buffers only
        ref, st, y_st = _head_reference(c, x_ref, _Snapshot(E, bn0), gref)
        if c["grad"] != "fallback":
            bound = _head_bound(c, x_ref, E.w1, E.b1, bn0, E.w2, E.b2, gref, y_st,
                                None if st is None else st["kink"], zdt, n_px)
            bad += _score_head(got, ref, bound, E.absent(c["x_grad"]), worst, where)
        if E.bn is not None:
            import test_gpu_projection_bnrelu as TPB
            for k in ("running_mean", "running_var"):
                rb = st[k]
                if (getattr(E.bn, k).double() - rb).abs().max().item() > TPB.STATS_REL * rb.abs().max().item():
                    bad.append(f"{where}: {k} off the float64 update")
            if int(E.bn.num_batches_tracked.item()) != nbt0 + int(c["train"]):
                bad.append(f"{where}: num_batches_tracked {int(E.bn.num_batches_tracked.item())}, expected "
                           f"{nbt0 + int(c['train'])}")
        if D is not None:                                       # the dense head, same inputs
            xd = x_s.detach().clone().requires_grad_(c["x_grad"])
            zd = D(xd)
            if c["grad"] == "fallback":
                ld = _head_loss(c, zd, lab, r)
                ld.backward()
            else:
                if loss is not None:
                    ld = cs.pixel_contrast_loss(zd.detach(), lab[0], seg=lab[1], options=_loss_options(c, r),
                                                **(dict(segment_queue=bank[0], pixel_queue=bank[1]) if bank else {}))
                zd.backward(gref)
            _sync(device)
            dg = D.grads(xd)
            if not _same_bits(zd.detach(), got["zn"]):
                bad.append(f"{where}: zn differs from the dense head's")
            if loss is not None and not _same_bits(ld.detach(), loss.detach()):
                bad.append(f"{where}: loss differs from the dense head's")
            for k, v in E.buffers().items():
                if not torch.equal(v, D.buffers()[k]):
                    bad.append(f"{where}: {k} differs from the dense head's")
            for k, v in dg.items():
                if c["grad"] == "fallback":
                    if not _same_bits(got[k], v):
                        bad.append(f"{where}: {k} differs from the dense head's ({c['pattern']})")
                elif k in bound:
                    d = (got[k].double() - v.double()).abs().reshape(-1)
                    if not bool((d <= 2 * bound[k].reshape(-1)).all()):
                        bad.append(f"{where}: {k} of the column path off the dense head's by more than the bound")
            if c.get("pattern") == "retain_grad" and not _same_bits(zn.grad, zd.grad):
                bad.append(f"{where}: zn.grad differs from the dense head's")
        if graph is not None:
            graph.replay()
            torch.cuda.synchronize()
            gg = Gh.grads(x_s)
            gg["zn"] = zn_g.detach()
            for k, v in got.items():
                if v is not None and not _same_bits(gg[k], v):
                    bad.append(f"{where}: graph replay {k} differs from the eager call")
        for h in heads:
            if h is not Gh:
                h.zero_grad(xe)
        Fn.clear_workspaces()
        if bad:
            break
    if graph is not None and not bad:
        for k, v in E.buffers().items():
            if not torch.equal(v, Gh.buffers()[k]):
                bad.append(f"after the replays: {k} of the graph differs from the eager sequence: {desc}")
    if not bad:
        reached |= {c["level"], c["act"], "train" if c["train"] else "eval"}
        reached |= {{"dense": "dense gzn", "cols": "column hand-off", "loss": "contrast loss",
                     "fallback": "fallback"}[c["grad"]]}
        if c["sync"]:
            reached.add("SyncBatchNorm")
        if (c["level"] == "conv1" and not c["b1"]) or not c["b2"]:
            reached.add("a bias None")
        if not c["x_grad"]:
            reached.add("x without grad")
        if c["grad"] == "cols" and c["n_cols"] in _HEAD_NCOLS:
            reached.add("n_cols at a tile edge")
        if C % 64 in (63, 0, 1):
            reached.add("Cin at a 64 edge")
        if 255 <= C <= 257:
            reached.add("Cin 255-257")
        if H * W == 1:
            reached.add("HW = 1")
        if c["adv"]:
            reached.add({"clamped": "clamped pixel", "dead channel": "dead BN channel",
                         "large mean": "large-mean channel"}[c["adv"]])
        for k in reached & set(HEAD_CATEGORIES):
            cov[k] += 1
    return bad


class _Snapshot:
    """A head's leaves with its BatchNorm as it was before a call (bn0): what the float64 reference starts from."""

    def __init__(self, h, bn0):
        import copy
        self.w1, self.b1, self.w2, self.b2 = h.w1, h.b1, h.w2, h.b2
        self.bn = None
        if bn0 is not None:
            self.bn = copy.deepcopy(h.bn)
            with torch.no_grad():
                self.bn.weight.copy_(bn0[1])
                self.bn.bias.copy_(bn0[2])
                self.bn.running_mean.copy_(bn0[3])
                self.bn.running_var.copy_(bn0[4])


def fuzz_projection_head(seed: int, n: int, device="cpu", scale: int = 1):
    """The fused projection head (project_normalize, bn_relu_project_normalize, conv_bn_relu_project_normalize /
    ProjectionHead) over drawn fusion levels, activation dtypes (autocast included), BatchNorm modes, biases and
    geometries at the kernels' edges, with a dense gzn, a column hand-off, the real contrast loss or a fallback consumer
    pattern, and adversarial values (a clamped pixel, a dead BN channel, a large-mean channel).  Each case runs 2-4
    replays with x, the gradient or the columns, and the weights changed in place between them (head_case).  On a
    device (a) and (b) are captured as one CUDA graph and replayed for real.  Returns (failures, coverage): how many
    clean cases reached each of HEAD_CATEGORIES, and coverage["worst"], the largest error / bound ratio per output."""
    rng = random.Random(seed)
    return run_head_cases([_draw_head_case(rng, it, scale, device) for it in range(n)], device, f"seed={seed}")


def run_head_cases(cases, device="cpu", tag=""):
    """head_case over `cases` with _bn_head_backward_cols wrapped to record its calls; (failures, coverage)."""
    import gc
    bad, cov = [], {k: 0 for k in HEAD_CATEGORIES}
    cov["worst"] = {}
    calls = []
    orig = Fn._bn_head_backward_cols

    def counted(lib, yc, dt, zn, inv, w2, state, cols, col_pix, *a):
        calls.append((cols.clone(), col_pix.clone()))
        return orig(lib, yc, dt, zn, inv, w2, state, cols, col_pix, *a)
    Fn._bn_head_backward_cols = counted
    try:
        for it, c in enumerate(cases):
            desc = "head {} it={} {}".format(tag, it, " ".join(f"{k}={v}" for k, v in c.items()))
            bad += head_case(c, device, cov, cov["worst"], desc, calls)
            calls.clear()
            if torch.device(device).type == "cuda":
                gc.collect()
                torch.cuda.empty_cache()
    finally:
        Fn._bn_head_backward_cols = orig
    return bad, cov


def edge_cases():
    """Constructed cases for what a short random draw may miss: the column path at Cin = 300 (k_col_prep's channel loop
    past 256) with a clamped anchor whose |z| is just under eps, and bf16 fallbacks whose deposits add to another
    gradient term (each deposit rounded to zn's dtype before the sum, as the loss's dense gradient would be)."""
    base = dict(adv=None, seed=9, act="fp32", train=True, sync=False, momentum=0.1, b1=False, b2=True, x_grad=True,
                B=2, Cin=40, H=5, W=4, n_rep=2, actions=["both"])
    cols = dict(base, level="bn_relu", grad="cols", adv="clamped", b2="tiny", Cin=300, n_cols=65)
    fb = [dict(base, level="bn_relu", grad="fallback", act="bf16", pattern=p, K=3, precision="fp32", bank=False,
               ms=12, mv=2) for p in ("other_term", "two_losses")]
    return [cols] + fb


def width_one_case(grad, Cin=64, B=2, H=9):
    """The constructed case of the fuzzer's finding: a feature map one pixel wide, the gradient a column hand-off or the
    contrast loss.  The placeholder's last dimension (W = 1) keeps stride 1 under expand(); the column path must run."""
    c = dict(level="bn_relu", grad=grad, adv=None, seed=5, act="fp32", train=True, sync=False, momentum=0.1, b1=False,
             b2=True, x_grad=True, B=B, Cin=Cin, H=H, W=1, n_rep=2, actions=["both"])
    if grad == "cols":
        c["n_cols"] = 7
    else:
        c.update(K=3, precision="fp32", bank=False, ms=6, mv=2)
    return c
