"""GPU tests of the deferred bank write and the CUDA-graph step (the file sorts last among the GPU tests on purpose: it
contains the CUDA-graph capture).  The three fp32 cases once failed ONLY when they ran after tests/test_gpu_topk.py: a
D=64 top-k call lowered the dynamic-shared-memory opt-in of k_sweep<POS> below the D=256 size (cudaErrorInvalidValue at
the next D=256 launch) — fixed
by the per-device one-time opt-in to the kernel's maximum (PCL_SMEM_OPT_IN, csrc/pcl_common.cuh);
`test_smem_opt_in_survives_a_smaller_launch` below pins it."""
import os

import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import functional as Fn
from contrastiveseg_b200.synth import make_bank, make_contrast_batch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda:0"


def _cfg(K, precision="fp32", **extra):
    c = {"temperature": 0.07, "base_temperature": 0.07, "max_samples": 128, "max_views": 8, "loss_weight": 0.1,
         "precision": precision}
    c.update(extra)
    return cs.Configer({"data": {"num_classes": K}, "contrast": c, "loss": {"params": {"ce_ignore_index": -1}},
                        "network": {"stride": 4}})


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_enqueue_between_loss_and_backward_does_not_change_the_gradient(precision):
    """Trainer order loss -> enqueue -> backward (trainer_contrastive.py:241-255): the reference's autograd holds a
    copy of the bank, the engine re-reads it in the backward sweep, so the in-place write is held back until after
    that backward.  Property: the gradient is bit-identical to the run without an enqueue, and the bank afterwards is
    bit-identical to an immediate enqueue."""
    K, D, M = 6, 256, 32
    data = make_contrast_batch(B=2, D=D, h=16, w=32, num_classes=K, img_stride=4, block=16, seed=5)
    tgt, seg = data["target"].to(DEV), data["seg"].to(DEV)
    banks = []
    grads = []
    for with_enqueue in (False, True):
        torch.manual_seed(0)
        bank = cs.MemoryBank(K, M, D, with_shadow=(precision == "bf16")).to(DEV)
        if precision == "bf16":
            bank.sync_shadow()
        crit = cs.PixelContrastLoss(_cfg(K, precision, seed=11))
        Fn._step_counter[0] = 0                                   # same device-RNG stream in both runs
        embed = data["embed"].to(DEV).requires_grad_(True)
        loss = crit(embed, tgt, seg=seg, queue=(bank.segment_queue, bank.pixel_queue), bank_shadow=bank.shadow)
        before = bank.pixel_queue.clone()
        if with_enqueue:
            bank.enqueue(embed.detach(), tgt, network_stride=4, pixel_update_freq=5, seed=3)
            assert torch.equal(bank.pixel_queue, before)          # held back: a backward that reads the bank is pending
        loss.backward()
        if with_enqueue:
            assert not torch.equal(bank.pixel_queue, before)      # ... and written right after it
        grads.append(embed.grad.clone())
        banks.append(bank)
    assert torch.equal(grads[0], grads[1])
    # the deferred write equals an immediate one on a fresh copy of the initial bank
    torch.manual_seed(0)
    ref = cs.MemoryBank(K, M, D, with_shadow=(precision == "bf16")).to(DEV)
    if precision == "bf16":
        ref.sync_shadow()
    from contrastiveseg_b200 import bank as bank_mod
    bank_mod._enqueue_counter[0] -= 1                             # replay the same enqueue seed
    ref.enqueue(data["embed"].to(DEV), tgt, network_stride=4, pixel_update_freq=5, seed=3)
    for name in ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr"):
        assert torch.equal(getattr(ref, name), getattr(banks[1], name)), name
    if precision == "bf16":
        assert torch.equal(ref.shadow, banks[1].shadow)


@pytest.mark.parametrize("overlap", [False, True])
@pytest.mark.parametrize("precision,mem", [("bf16", False), ("fp32", False), ("bf16", True)])
def test_graphed_step_equals_eager_step(precision, mem, overlap):
    """GraphedContrastStep: replay r samples like the eager step with counter r+1 (same keyed bijection), so anchors,
    loss and dense gradient are bit-identical; successive replays draw different anchors; grad_scale scales the gradient.
    To confirm on hardware: capture of the whole C-ABI sequence (no illegal call under capture)."""
    K, D, M = 7, 256, 48
    data = make_contrast_batch(B=2, D=D, h=32, w=32, num_classes=K, img_stride=4, block=16, seed=21)
    embed, tgt, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    bank = None
    kw = {}
    if mem:
        bank = cs.MemoryBank(K, M, D, with_shadow=True).to(DEV)
        bank.sync_shadow()
        kw = dict(segment_queue=bank.segment_queue, pixel_queue=bank.pixel_queue, bank_shadow=bank.shadow)
    opts = cs.ContrastOptions(temperature=0.07, base_temperature=0.07, max_samples=128, max_views=8, seed=5,
                              precision=precision, num_classes=K)
    step = cs.GraphedContrastStep(embed, tgt, seg=seg, options=opts, overlap_zero_fill=overlap, fused=False, **kw)
    metas, losses, grads = [], [], []
    for r in range(3):
        loss, grad = step.replay()
        torch.cuda.synchronize()
        metas.append(step.ws.anchor_meta.clone()); losses.append(loss.clone()); grads.append(grad.clone())
    assert int(step.counter.item()) == 3
    assert not torch.equal(metas[0], metas[1]) and not torch.equal(metas[1], metas[2])
    for r in range(3):
        Fn._step_counter[0] = r                                   # the eager call pre-increments: counter r+1
        e = embed.clone().requires_grad_(True)
        l = cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts, **{k: v for k, v in kw.items()})
        ws = Fn.last_workspace(e.device)
        l.backward()
        torch.cuda.synchronize()
        assert torch.equal(ws.anchor_meta, metas[r])
        assert torch.equal(l.detach(), losses[r])
        if overlap:    # rows reduced by the sweep's own reduction kernel instead of the fused writer: same sum order
            assert torch.allclose(e.grad, grads[r], rtol=2e-6, atol=0)
        else:
            assert torch.equal(e.grad, grads[r])
    step.set_grad_scale(0.25)
    step.counter.fill_(1)
    _, g = step.replay()
    torch.cuda.synchronize()
    assert torch.allclose(g, 0.25 * grads[1], rtol=1e-6, atol=0)
    # autograd hand-off
    e = embed.clone().requires_grad_(True)
    step2 = cs.GraphedContrastStep(e, tgt, seg=seg, options=opts, **kw)
    out = step2.apply(e)
    out.backward()
    assert torch.equal(e.grad, step2.grad)


@pytest.mark.parametrize("geom", [dict(B=2, h=32, w=32, K=7, ms=128, mv=8), dict(B=3, h=32, w=48, K=9, ms=700, mv=40),
                                  dict(B=4, h=64, w=64, K=19, ms=1024, mv=100)])
def test_fused_small_anchor_step_matches_the_streaming_path_and_the_oracle(geom):
    """The fused step (scan+plan | selection | ONE kernel for InfoNCE forward+backward with the logits in tensor memory |
    scatter; csrc/pcl_infonce_fused.cu) draws the same anchors as the eager step with the same counter (bit-exact
    anchor_meta) and computes the same loss / gradient as the streaming tensor sweeps up to summation order (loss 2e-6
    rel, gradient 2e-3 max|g|: bf16 rounding of the gradient tile flips on last-bit differences of its fp32 inputs), and
    the float64 oracle's within the tensor-path tolerances (loss 1e-4, gradient 4e-3 max|g|).  Covers 1 (128 anchors),
    partial (A < max_samples, several row/column tiles) and 8 x 4 tiles."""
    from oracle import ref_port as P
    B, h, w, K, ms, mv = (geom[k] for k in ("B", "h", "w", "K", "ms", "mv"))
    D = 256
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=33)
    embed, tgt, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, seed=5,
                              precision="bf16", num_classes=K)
    step = cs.GraphedContrastStep(embed, tgt, seg=seg, options=opts, grad_scale=0.5)
    assert step.fused
    for r in range(3):
        loss, grad = step.replay()
        torch.cuda.synchronize()
        meta, loss, grad = step.ws.anchor_meta.clone(), loss.clone(), grad.clone()
        A = int(step.ws.plan[2].item())
        assert A > 0 and (ms < 1024 or A >= 512)
        Fn._step_counter[0] = r
        e = embed.clone().requires_grad_(True)
        l = cs.pixel_contrast_loss(e, tgt, seg=seg, options=opts)
        ws = Fn.last_workspace(e.device)
        l.backward()
        torch.cuda.synchronize()
        assert torch.equal(ws.anchor_meta, meta)
        assert abs(l.item() - loss.item()) <= 2e-6 * abs(l.item())
        gmax = e.grad.abs().max().item()
        assert (0.5 * e.grad - grad).abs().max().item() <= 2e-3 * 0.5 * gmax
        # float64 oracle on the anchors the step drew (self-contrast, class-sorted rows: diagonal = own row)
        m = meta.view(4, ms)[:, :A].long().cpu()
        rows = data["embed"].permute(0, 2, 3, 1).reshape(B, h * w, D)[m[1], m[0]].double()
        cf = P.infonce_closed_form(rows, m[2].double(), rows, m[2].double(), 0.1, 0.07, True)
        assert abs(loss.item() - cf["loss"].item()) <= 1e-4 * abs(cf["loss"].item())
        g_rows = grad.permute(0, 2, 3, 1).reshape(B, h * w, D)[m[1].to(DEV), m[0].to(DEV)].double().cpu() / 0.5
        assert (g_rows - cf["dA"]).abs().max().item() <= 4e-3 * cf["dA"].abs().max().item()
        assert int((grad != 0).sum().item()) <= A * D
    assert int(step.counter.item()) == 3
    assert int(step.ws.sync.abs().sum().item()) == 0             # the kernels re-armed their counters


def test_fused_step_sparse_reset_equals_full_fill():
    """sparse_reset=True: the dense gradient persists between replays and only the entries of the previous replay are
    cleared.  Bit-identical to the full-fill step on every replay (different anchors every time), also after inputs
    change, and after reset_grad() following an outside write."""
    D, K = 256, 9
    data = make_contrast_batch(B=3, D=D, h=32, w=48, num_classes=K, img_stride=4, block=16, seed=33)
    tgt, seg = data["target"].to(DEV), data["seg"].to(DEV)
    e1, e2 = data["embed"].to(DEV), data["embed"].to(DEV).clone()
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=700, max_views=40, seed=5,
                              precision="bf16", num_classes=K)
    full = cs.GraphedContrastStep(e1, tgt, seg=seg, options=opts)
    sparse = cs.GraphedContrastStep(e2, tgt, seg=seg, options=opts, sparse_reset=True)
    assert full.fused and sparse.sparse_reset
    for r in range(5):
        if r == 3:                                             # new inputs in the static buffers
            nxt = make_contrast_batch(B=3, D=D, h=32, w=48, num_classes=K, img_stride=4, block=16, seed=77)
            for e in (e1, e2):
                e.copy_(nxt["embed"].to(DEV))
            tgt.copy_(nxt["target"].to(DEV)); seg.copy_(nxt["seg"].to(DEV))
        lf, gf = full.replay()
        ls, gs = sparse.replay()
        torch.cuda.synchronize()
        assert torch.equal(full.ws.anchor_meta, sparse.ws.anchor_meta)
        assert torch.equal(lf, ls) and torch.equal(gf, gs), r
    sparse.grad.add_(1.0)                                      # somebody wrote into the buffer ...
    sparse.reset_grad()                                        # ... and said so
    lf, gf = full.replay()
    ls, gs = sparse.replay()
    torch.cuda.synchronize()
    assert torch.equal(lf, ls) and torch.equal(gf, gs)


def test_fused_step_with_no_qualifying_class_gives_zero_loss():
    """TC == 0 (every class has <= max_views pixels): zero loss, zero gradient, no hang of the inter-CTA barriers."""
    data = make_contrast_batch(B=2, D=256, h=16, w=16, num_classes=5, img_stride=4, block=16, seed=3)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=64, max_views=100000, seed=5,
                              precision="bf16", num_classes=5)
    step = cs.GraphedContrastStep(data["embed"].to(DEV), data["target"].to(DEV), seg=data["seg"].to(DEV), options=opts)
    assert step.fused
    loss, grad = step.replay()
    torch.cuda.synchronize()
    assert loss.item() == 0.0 and float(grad.abs().sum().item()) == 0.0


def test_smem_opt_in_survives_a_smaller_launch():
    """Regression (round-1 hidden failure): a small-D launch of a sweep kernel must not lower the shared-memory opt-in a
    later D=256 launch needs — exact fp32 loss at D=256, then the top-k path (which launches k_sweep<POS>) at D=64, then
    D=256 again."""
    def run(D, topk=None):
        K = 5
        data = make_contrast_batch(B=2, D=D, h=16, w=32, num_classes=K, img_stride=4, block=16, seed=9)
        e = data["embed"].to(DEV).requires_grad_(True)
        opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=64, max_views=4, seed=1,
                                  precision="fp32", num_classes=K, topk_negatives=topk)
        Fn._step_counter[0] = 0
        l = cs.pixel_contrast_loss(e, data["target"].to(DEV), seg=data["seg"].to(DEV), options=opts)
        l.backward()
        torch.cuda.synchronize()
        return l.detach().clone(), e.grad.clone()
    l0, g0 = run(256)
    run(64, topk=3)
    run(64)
    l1, g1 = run(256)
    assert torch.equal(l0, l1) and torch.equal(g0, g1)


def test_second_backward_is_refused_and_state_dict_flushes_the_pending_write():
    """ADVICE r1: (a) the engine keeps no copy of the forward's scratch, so a second backward through the same node
    (retain_graph=True) must raise instead of returning a gradient computed from overwritten scratch; (b) a checkpoint
    taken between loss_step and backward must contain the rows enqueued in that window."""
    from contrastiveseg_b200._abi import PclError
    K, D, M = 6, 64, 32
    data = make_contrast_batch(B=2, D=D, h=16, w=32, num_classes=K, img_stride=4, block=16, seed=5)
    tgt, seg = data["target"].to(DEV), data["seg"].to(DEV)
    bank = cs.MemoryBank(K, M, D).to(DEV)
    crit = cs.PixelContrastLoss(_cfg(K, "fp32", seed=11))
    embed = data["embed"].to(DEV).requires_grad_(True)
    loss = crit(embed, tgt, seg=seg, queue=(bank.segment_queue, bank.pixel_queue))
    before = bank.pixel_queue.clone()
    bank.enqueue(embed.detach(), tgt, network_stride=4, pixel_update_freq=5, seed=3)
    assert torch.equal(bank.pixel_queue, before)                 # held back
    sd = bank.state_dict()
    assert not torch.equal(sd["pixel_queue"], before)            # state_dict() flushed the pending write
    loss.backward(retain_graph=True)
    with pytest.raises(PclError, match="backward ran twice"):
        loss.backward()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_graphed_bank_step_with_enqueue_equals_the_trainer_order(precision):
    """Bank step as ONE graph (world 1): stats -> ranks -> forward -> enqueue packet -> backward -> bank write.  Replay r
    must equal the eager trainer order (loss -> enqueue -> backward, trainer_contrastive.py:241-255) with counters r+1:
    same loss bits, same gradient, bit-identical bank (rows, pointers, bf16 shadow) after every step."""
    from contrastiveseg_b200 import bank as bank_mod
    K, D, M = 7, 256, 48
    data = make_contrast_batch(B=2, D=D, h=32, w=32, num_classes=K, img_stride=4, block=16, seed=21)
    embed, tgt, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    shadow = precision == "bf16"
    torch.manual_seed(0)
    bank_g = cs.MemoryBank(K, M, D, with_shadow=shadow).to(DEV)
    bank_e = cs.MemoryBank(K, M, D, with_shadow=shadow).to(DEV)
    bank_e.load_state_dict(bank_g.state_dict())
    if shadow:
        bank_g.sync_shadow(); bank_e.sync_shadow()
    opts = cs.ContrastOptions(temperature=0.07, base_temperature=0.07, max_samples=128, max_views=8, seed=5,
                              precision=precision, num_classes=K)
    step = cs.GraphedContrastStep(embed, tgt, seg=seg, segment_queue=bank_g.segment_queue, pixel_queue=bank_g.pixel_queue,
                                  bank_shadow=bank_g.shadow, options=opts,
                                  enqueue=dict(bank=bank_g, network_stride=4, pixel_update_freq=5, seed=3))
    names = ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr")
    for name in names:                                           # warm-up runs of the capture left no trace in the bank
        assert torch.equal(getattr(bank_g, name), getattr(bank_e, name)), name
    for r in range(3):
        loss, grad = step.replay()
        torch.cuda.synchronize()
        Fn._step_counter[0] = r
        bank_mod._enqueue_counter[0] = r
        e = embed.clone().requires_grad_(True)
        l = cs.pixel_contrast_loss(e, tgt, seg=seg, segment_queue=bank_e.segment_queue, pixel_queue=bank_e.pixel_queue,
                                   bank_shadow=bank_e.shadow, options=opts)
        bank_e.enqueue(e.detach(), tgt, network_stride=4, pixel_update_freq=5, seed=3)
        l.backward()
        torch.cuda.synchronize()
        assert torch.equal(l.detach(), loss)
        assert torch.allclose(e.grad, grad, rtol=2e-6, atol=0)
        for name in names:
            assert torch.equal(getattr(bank_g, name), getattr(bank_e, name)), (r, name)
        if shadow:
            assert torch.equal(bank_g.shadow, bank_e.shadow)
    assert not torch.equal(bank_g.pixel_queue_ptr, torch.zeros_like(bank_g.pixel_queue_ptr))


@pytest.mark.gpu
@pytest.mark.parametrize("world,M,B", [(5, 4, 2), (8, 7, 3), (3, 40, 2)])
def test_bank_apply_of_many_ranks_equals_the_sequential_reference(monkeypatch, world, M, B):
    """pcl_bank_apply writes every row once, by its LAST writer (thread 0 replays the pointer arithmetic of all slots,
    csrc/pcl_bank.cu k_bank_apply).  world * B slots per class with a tiny ring: the segment ring wraps inside one apply
    and the pixel windows overlap (Q4) — must equal the reference applied image by image, rank-major
    (trainer_contrastive.py:96-139 after its all-gather)."""
    from contrastiveseg_b200 import bank as bank_mod
    from contrastiveseg_b200.synth import make_bank, make_contrast_batch
    from oracle import ref_port as P
    dev = torch.device(DEV)
    K, D, Fq, stride = 6, 32, 3, 2
    names = ("segment_queue", "segment_queue_ptr", "pixel_queue", "pixel_queue_ptr")
    b0 = make_bank(K, M, D, 5)
    ref = [b0[k].clone() for k in names]
    mine = [b0[k].clone().to(dev) for k in names]
    for step in range(3):
        datas = [make_contrast_batch(B=B, D=D, h=12, w=14, num_classes=K, img_stride=2, block=4, seed=31 * step + r)
                 for r in range(world)]
        perms, packets = [], []
        for r in range(world):
            rec = P.PermRecorder(torch.Generator().manual_seed(9 * step + r))
            P.dequeue_and_enqueue(datas[r]["embed"], datas[r]["target"], *ref, network_stride=stride, memory_size=M,
                                  pixel_update_freq=Fq, perm_fn=rec)
            perms.append(rec.draws)
        # every rank's packet, computed on a throw-away bank ...
        for r in range(world):
            monkeypatch.setattr(bank_mod, "gather_packets", lambda pk, group=None, out=None: (packets.append(pk.clone()),
                                                                                                pk.view(1, -1))[1])
            monkeypatch.setattr(bank_mod, "world_size", lambda group=None: 1)
            scratch = [b0[k].clone().to(dev) for k in names]
            cs.dequeue_and_enqueue(datas[r]["embed"].to(dev), datas[r]["target"].to(dev), *scratch,
                                   network_stride=stride, memory_size=M, pixel_update_freq=Fq,
                                   perm_fn=P.PermReplay(perms[r]))
        # ... then one apply of the rank-major stack on the bank under test
        stack = torch.stack([p.view(-1) for p in packets])
        monkeypatch.setattr(bank_mod, "gather_packets", lambda pk, group=None, out=None: stack)
        monkeypatch.setattr(bank_mod, "world_size", lambda group=None: world)
        cs.dequeue_and_enqueue(datas[0]["embed"].to(dev), datas[0]["target"].to(dev), *mine, network_stride=stride,
                               memory_size=M, pixel_update_freq=Fq, perm_fn=P.PermReplay(perms[0]))
    torch.cuda.synchronize()
    assert torch.equal(mine[1].cpu(), ref[1]) and torch.equal(mine[3].cpu(), ref[3])
    assert (mine[0].cpu() - ref[0]).abs().max().item() <= 2e-6
    assert (mine[2].cpu() - ref[2]).abs().max().item() <= 2e-7
