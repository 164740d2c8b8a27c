"""Column mode of the captured contrast step and criterion (GraphedContrastStep(grad="cols"),
GraphedContrastCriterion(embed_grad="cols")) as real graph replays: labels, seg and embed are refilled in place between
replays so that classes vanish and A varies down to 0.  Against a dense-mode twin on the same inputs (the same seed and
replay index draw the same anchors in both modes): the loss bit for bit, the dense gradient built from the columns bit
for bit, rows >= A marked unused, the bank written by a one-rank enqueue step, the eager capture=False sequence bit for
bit, and a sparse_grad projection head fed through apply() against the dense step + the head's dense backward.
test_emu_graphed_cols.py runs the check functions at small shapes on the emulated kernels (DEV = "cpu")."""
import copy

import pytest
import torch

import contrastiveseg_b200 as cs
import test_gpu_graphed_criterion as T
import test_gpu_sparse_head as S
from contrastiveseg_b200 import _abi, functional as Fn
from contrastiveseg_b200.synth import make_bank, make_contrast_batch

DEV = "cuda:0"
BF = torch.bfloat16
G = cs.GraphedContrastStep

# step configurations: ContrastOptions entries, plus fused= (GraphedContrastStep) and bank= ("read" / "enqueue")
MODES = {
    "fused": dict(precision="bf16"),
    "simt": dict(),
    "tensor": dict(precision="bf16", fused=False),
    "normalize": dict(normalize=True),
    "topk": dict(topk_negatives=5),
    "bank_simt": dict(bank="read"),
    "bank_tensor": dict(precision="bf16", bank="read"),
    "bank_enqueue": dict(bank="enqueue"),
}
SCALES = [0.5, 0.5, -1.25, 0.0, 2.0, 0.75]


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _draw(r, B, D, h, w, K, seed):
    """Replay r's inputs: r = 1 drops two classes, r = 2 keeps one class in one image, r = 3 ignores every pixel
    (A = 0), the others are fresh batches."""
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=2, block=3, seed=seed + r)
    target = data["target"]
    if r == 1:
        target[(target == 0) | (target == 1)] = -1
    elif r == 2:
        keep = target == int(target[0].max())
        keep[1:] = False
        target[~keep] = -1
    elif r == 3:
        target.fill_(-1)
    return data["embed"], target, data["seg"]


def _banks(K, M, D, tensor, n):
    init = make_bank(K, M, D, 42)
    out = []
    for _ in range(n):
        b = cs.MemoryBank(K, M, D, with_shadow=tensor).to(DEV)
        for k in ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr"):
            getattr(b, k).copy_(init[k])
        if tensor:
            b.sync_shadow()
        out.append(b)
    return out


def check_step(mode, dtype=torch.float32, B=2, D=64, h=12, w=10, K=5, ms=96, replays=6, eager_twin=True, mv=8):
    kw = dict(MODES[mode])
    bank, fused = kw.pop("bank", None), kw.pop("fused", None)
    tensor = kw.get("precision") == "bf16"
    D = 256 if tensor else D
    e0, t0, s0 = _draw(0, B, D, h, w, K, 61)
    embed, target, seg = e0.to(DEV, dtype).contiguous(), t0.to(DEV), s0.to(DEV)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, seed=9, **kw)
    banks = _banks(K, 12, D, tensor, 3) if bank else [None] * 3

    def make(i, grad, capture=True):
        b = banks[i]
        extra = {}
        if b is not None:
            extra = dict(segment_queue=b.segment_queue, pixel_queue=b.pixel_queue, bank_shadow=b.shadow)
            if bank == "enqueue":
                extra["enqueue"] = dict(bank=b, network_stride=2, pixel_update_freq=3, seed=5)
        return G(embed, target, seg=seg, options=opts, grad_scale=SCALES[0], fused=fused, grad=grad, capture=capture,
                 **extra)
    dense, cols = make(0, "dense"), make(1, "cols")
    eager = make(2, "cols", capture=False) if eager_twin else None
    assert cols.grad is None and dense.fused == cols.fused == (mode == "fused")
    As = []
    for r in range(replays):
        if r:
            e, t, s = _draw(r % 5, B, D, h, w, K, 61 + 7 * (r // 5))
            embed.copy_(e.to(dtype)), target.copy_(t), seg.copy_(s)
            for st in (dense, cols, eager):
                if st is not None:
                    st.set_grad_scale(SCALES[r])
        ld, gd = dense.replay()
        lc, (c, p) = cols.replay()
        assert c.data_ptr() == cols.cols.data_ptr() and p.data_ptr() == cols.col_pix.data_ptr()   # static buffers
        _sync()
        A = int(cols.ws.plan[_abi.PLAN_A].item())
        As.append(A)
        why = (mode, dtype, r, A)
        assert torch.equal(dense.ws.anchor_meta, cols.ws.anchor_meta), why             # the same anchors
        assert torch.equal(_bits(lc), _bits(ld)), why
        assert bool((p[A:] == -1).all()) and bool((_bits(c[A:]) == 0).all()), why       # unused rows, every replay
        assert bool((p[:A] >= 0).all()), why
        assert torch.equal(_bits(cols.dense_grad()), _bits(gd)), why                    # bit for bit
        if eager is not None:
            le, (ce, pe) = eager.replay()
            _sync()
            assert torch.equal(_bits(le), _bits(lc)) and torch.equal(_bits(ce), _bits(c)) and torch.equal(pe, p), why
        if bank == "enqueue":
            for k in ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr"):
                assert torch.equal(getattr(banks[0], k), getattr(banks[1], k)), (why, k)
    assert 0 in As and len(set(As)) >= 3, As
    # apply() with no sparse head behind embed: the dense gradient, bit for bit the dense step's
    cols.set_grad_scale(1.0), dense.set_grad_scale(1.0)
    ec = embed.detach().requires_grad_(True)
    cols.apply(ec).backward()
    _, gd = dense.replay()
    _sync()
    assert torch.equal(_bits(ec.grad), _bits(gd)), mode
    with pytest.raises(_abi.PclError):                  # the columns are handed over once
        loss = cols.apply(embed.detach().requires_grad_(True))
        loss.backward(retain_graph=True)
        loss.backward()
    return As


def check_fused_splits(dtype=torch.float32, B=2, h=16, w=16, K=5, ms=1024, mv=32, replays=6, eager_twin=True):
    """The fused step's column writer past one 256-column split of the InfoNCE kernel (max_samples up to 1024: up to
    four splits): the kernel writes only the live splits' partials, so after a replay with A > 256 the partials of the
    dropped splits are stale and a later replay with A <= 256 must not sum them.  Columns against the dense twin, bit
    for bit, on a sequence where A rises above 256, then falls below it and to 0."""
    As = check_step("fused", dtype, B=B, h=h, w=w, K=K, ms=ms, mv=mv, replays=replays, eager_twin=eager_twin)
    big = [i for i, a in enumerate(As) if a > 256]
    assert big and any(0 < a <= 256 for a in As[big[0] + 1:]), As


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_captured_fused_cols_past_one_split(dtype):
    check_fused_splits(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_captured_cols_step_matches_the_dense_step(mode):
    check_step(mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fused", "simt", "bank_tensor"])
def test_captured_cols_step_with_a_bf16_embed(mode):
    check_step(mode, BF)


def check_criterion(name, dtype=torch.float32, B=2, D=64, h=16, w=16, replays=4):
    crit = T.make_criterion(name).to(DEV)
    heads = ["seg"] + (["seg_aux"] if isinstance(crit, cs.ContrastAuxCELoss) else [])
    first, target = T._batch(100, B, D, h, w, len(heads) > 1)
    target = target.to(DEV)
    static = {k: first[k].to(DEV).to(dtype).requires_grad_(True) for k in heads}
    static["embed"] = first["embed"].to(DEV).requires_grad_(True)
    if crit.with_memory:
        init = make_bank(T.K_CRIT, 40, D, seed=7)
        static["segment_queue"], static["pixel_queue"] = init["segment_queue"].to(DEV), init["pixel_queue"].to(DEV)
    dense = cs.GraphedContrastCriterion(crit, static, target)
    cols = cs.GraphedContrastCriterion(crit, static, target, embed_grad="cols")
    As = []
    for r in range(replays):
        if r:
            nxt, t = T._batch(100 + r, B, D, h, w, len(heads) > 1)
            if r == 2:
                t.fill_(-1)                                  # every pixel ignored: A = 0
            with torch.no_grad():
                for k in heads + ["embed"]:
                    static[k].copy_(nxt[k].to(DEV).to(static[k].dtype))
            target.copy_(t)
        if r == replays - 1:
            dense.set_grad_scale(-0.5), cols.set_grad_scale(-0.5)
        ld, gd = dense.replay()
        gd = {k: v.clone() for k, v in gd.items()}
        lc, gc_ = cols.replay()
        _sync()
        A = int(cols.step.ws.plan[_abi.PLAN_A].item())
        As.append(A)
        c, p = gc_["embed"]
        assert torch.equal(_bits(lc), _bits(ld)) and torch.equal(_bits(cols.step.loss), _bits(dense.step.loss)), (name, r)
        assert bool((p[A:] == -1).all()), (name, r)
        assert torch.equal(_bits(cols.step.dense_grad()), _bits(gd["embed"])), (name, r)
        for k in heads:                                  # the seg backward adds with atomics: not bit-reproducible
            assert T._close(gc_[k], gd[k]), (name, k, r)
    assert 0 in As, As
    dense.set_grad_scale(1.0), cols.set_grad_scale(1.0)
    for k in heads + ["embed"]:
        static[k].grad = None
    cols.apply(static).backward()
    _, gd = dense.replay()
    _sync()
    assert torch.equal(_bits(static["embed"].grad), _bits(gd["embed"])), name
    for k in heads:
        assert T._close(static[k].grad, gd[k]), (name, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ce", "aux_ohem", "mem_rmi"])
def test_captured_cols_criterion_matches_the_dense_criterion(name):
    check_criterion(name)


# ------------------------------------------------------------------------------------------------------------------
# the sparse projection head behind apply()
# ------------------------------------------------------------------------------------------------------------------
def _count_column_backwards():
    """Wraps the head's column backward; returns the list its calls are appended to and the restore function."""
    calls, orig = [], Fn._bn_head_backward_cols

    def wrapped(*a, **k):
        calls.append(1)
        return orig(*a, **k)
    Fn._bn_head_backward_cols = wrapped
    return calls, lambda: setattr(Fn, "_bn_head_backward_cols", orig)


def check_head_apply(conv1, dtype=torch.float32, B=2, Cin=40, h=12, w=10, K=5, ms=64, replays=4, criterion=False):
    """zn = head(x, out=step.embed) -> step.apply(zn) (or the criterion's apply) -> backward, for a sparse_grad head and
    a column step against the same head without sparse_grad and a dense step: loss and BN buffers bit for bit, every
    gradient within the sparse-head bounds, and the column backward ran once per replay."""
    dense_head, sparse_head = S._heads(Cin, conv1)
    x0, t0, s0 = S._e2e_inputs(B, Cin, h, w, K)
    target, seg = t0.clone(), s0.clone()
    zdt = BF if dtype == BF else torch.float32
    bufs = [torch.zeros(B, 256, h, w, dtype=zdt, device=DEV) for _ in range(2)]
    if criterion:
        crit = cs.ContrastCELoss(S._cfg(K, precision="bf16", rng="device")).to(DEV)
        objs = [cs.GraphedContrastCriterion(crit, {"seg": seg, "embed": bufs[i]}, target, embed_grad=g)
                for i, g in enumerate(("dense", "cols"))]
        run = lambda o, zn: o.apply({"seg": seg, "embed": zn})                                    # noqa: E731
    else:
        opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=8,
                                  precision="bf16", seed=3)
        objs = [G(bufs[i], target, seg=seg, options=opts, grad_scale=0.1, grad=g) for i, g in
                enumerate(("dense", "cols"))]
        run = lambda o, zn: o.apply(zn)                                                          # noqa: E731
    calls, restore = _count_column_backwards()
    try:
        for r in range(replays):
            x, t, s = S._e2e_inputs(B, Cin, h, w, K, seed=21 + r)
            if r == 2:
                t[1:] = -1
            target.copy_(t), seg.copy_(s)
            out = []
            for head, o, buf in ((dense_head, objs[0], bufs[0]), (sparse_head, objs[1], bufs[1])):
                xx = x.clone().requires_grad_(True)
                head.zero_grad(set_to_none=True)
                with torch.autocast("cuda" if str(DEV).startswith("cuda") else "cpu", dtype=BF, enabled=dtype == BF):
                    zn = head(xx, out=buf)
                    assert zn.data_ptr() == buf.data_ptr()
                    loss = run(o, zn)
                loss.backward()
                _sync()
                res = {"loss": loss.detach().clone(), "gx": xx.grad}
                res.update({n: p.grad for n, p in head.named_parameters()})
                bn = head.proj[1][0]
                res.update({k: getattr(bn, k).clone() for k in ("running_mean", "running_var", "num_batches_tracked")})
                out.append(res)
            S._compare(out[1], out[0])
            assert len(calls) == r + 1, (r, len(calls))
    finally:
        restore()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("conv1", [False, True], ids=["bn_relu", "conv1"])
def test_sparse_head_through_the_captured_cols_step(conv1, dtype):
    check_head_apply(conv1, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("conv1", [False, True], ids=["bn_relu", "conv1"])
def test_sparse_head_through_the_captured_cols_criterion(conv1):
    check_head_apply(conv1, criterion=True)


def check_retain_grad_falls_back(B=2, Cin=40, h=12, w=10, K=5):
    """zn.retain_grad(): the sink refuses, apply() returns the dense gradient built from the columns and the head runs
    its dense backward (INTEGRATION §1)."""
    _, head = S._heads(Cin, False)
    x, target, seg = S._e2e_inputs(B, Cin, h, w, K)
    buf = torch.zeros(B, 256, h, w, device=DEV)
    opts = cs.ContrastOptions(max_samples=64, max_views=8, precision="bf16", seed=3)
    step = G(buf, target, seg=seg, options=opts, grad="cols")
    calls, restore = _count_column_backwards()
    try:
        zn = head(x.clone().requires_grad_(True), out=buf)
        zn.retain_grad()
        step.apply(zn).backward()
        _sync()
        assert not calls
        assert torch.equal(zn.grad, step.dense_grad())
    finally:
        restore()


@pytest.mark.gpu
def test_retain_grad_falls_back_to_the_dense_gradient():
    check_retain_grad_falls_back()


# ------------------------------------------------------------------------------------------------------------------
# memory at S1
# ------------------------------------------------------------------------------------------------------------------
def _step_peak(grad, B=8, h=128, w=256, K=19):
    data = make_contrast_batch(B=B, D=256, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=5)
    embed, target, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    opts = cs.ContrastOptions(max_samples=1024, max_views=100, precision="bf16")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step = G(embed, target, seg=seg, options=opts, grad=grad)
    for _ in range(3):
        step.replay()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del step
    return peak, embed.numel() * 4


@pytest.mark.gpu
def test_cols_step_peak_memory_stays_far_below_one_dense_gradient():
    peak_cols, dense_bytes = _step_peak("cols")
    peak_dense, _ = _step_peak("dense")
    assert peak_dense >= dense_bytes, (peak_dense, dense_bytes)
    assert peak_cols < dense_bytes // 8, (peak_cols, dense_bytes)


def check_refusals():
    data = make_contrast_batch(B=1, D=64, h=8, w=8, num_classes=3, img_stride=2, block=3, seed=1)
    embed, target, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    opts = cs.ContrastOptions(max_samples=16, max_views=4)
    with pytest.raises(_abi.PclError):
        G(embed, target, seg=seg, options=opts, grad="sparse", capture=False)
    with pytest.raises(_abi.PclError):
        G(embed, target, seg=seg, options=opts, grad="cols", sparse_reset=True, capture=False)
    dense_head, sparse_head = S._heads(40, False)
    x, _, _ = S._e2e_inputs(1, 40, 8, 8, 3)
    for bad in (torch.zeros(1, 256, 8, 8, dtype=BF, device=DEV), torch.zeros(1, 256, 8, 9, device=DEV),
                torch.zeros(1, 8, 8, 256, device=DEV).permute(0, 3, 1, 2),
                torch.zeros(1, 256, 8, 8, device=DEV, requires_grad=True)):
        with pytest.raises(_abi.PclError):
            sparse_head(x, out=bad)
    plain = cs.ProjectionHead(40, 256, "convmlp", bn_type="torchbn", fused=True).to(DEV)
    with pytest.raises(_abi.PclError):
        plain(x, out=torch.zeros(1, 256, 8, 8, device=DEV))
    # without out= nothing changes: the same values in a fresh tensor
    buf = torch.full((1, 256, 8, 8), float("nan"), device=DEV)
    h2 = copy.deepcopy(dense_head)
    z_out = h2(x, out=buf)
    z_ref = dense_head(x)
    _sync()
    assert z_out.data_ptr() == buf.data_ptr() and torch.equal(z_out, z_ref)


@pytest.mark.gpu
def test_refusals_and_out():
    check_refusals()
