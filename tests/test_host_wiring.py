"""Host-side wiring of the autograd entry points, checked on CPU: the real library answers the size queries (pure
host code), every compute entry point is replaced by a recorder that returns PCL_OK.  Verifies the call sequence and
the pointer / scalar arguments the Python layer hands to the C ABI (no arithmetic runs; outputs are uninitialised)."""
import ctypes as C

import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi, functional as Fn

HOST_ONLY = {"pcl_version", "pcl_strerror", "pcl_last_cuda_error", "pcl_abi_sizeof", "pcl_select_sizes",
             "pcl_sweep_sizes", "pcl_tc_sizes", "pcl_topk_scratch_u32", "pcl_seg_ce_scratch_floats",
             "pcl_bank_packet_floats", "pcl_bank_scratch_floats", "pcl_step_fused_supported", "pcl_launch_count",
             "pcl_tc_topk_scratch_u32"}


class RecordingLib:
    def __init__(self, real):
        self._real = real
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name in HOST_ONLY:
            return fn

        def rec(*args):
            snap = []
            for a in args:
                obj = getattr(a, "_obj", None)          # ctypes.byref(struct) -> copy of the struct at call time
                if obj is not None:
                    cp = type(obj)()
                    C.memmove(C.byref(cp), C.byref(obj), C.sizeof(obj))
                    snap.append(cp)
                else:
                    snap.append(a)
            self.calls.append((name, snap))
            return 0
        return rec


class _NoCtx:
    def __init__(self, *a):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


@pytest.fixture
def rec(monkeypatch):
    lib = RecordingLib(_abi.load(build_if_missing=True))
    monkeypatch.setattr(Fn._abi, "load", lambda *a, **k: lib)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, name: None)
    monkeypatch.setattr(Fn, "_stream_ptr", lambda device: 0x5EED)
    monkeypatch.setattr(Fn, "_on_device", _NoCtx)
    from contrastiveseg_b200 import bank as bank_mod
    monkeypatch.setattr(bank_mod, "_is_cuda", lambda t: True)
    Fn.clear_workspaces()
    Fn._BANK_READERS.clear()
    yield lib
    Fn.clear_workspaces()
    Fn._BANK_READERS.clear()


def _inputs(B=2, D=32, h=8, w=8, K=5, s=2):
    g = torch.Generator().manual_seed(0)
    embed = torch.randn(B, D, h, w, generator=g).requires_grad_(True)
    labels = torch.randint(0, K, (B, h * s, w * s), generator=g)
    seg = torch.randn(B, K, h, w, generator=g)
    return embed, labels, seg


def test_default_step_call_sequence(rec):
    embed, labels, seg = _inputs()
    opts = cs.ContrastOptions(max_samples=64, max_views=4, temperature=0.2, base_temperature=0.1)
    loss = cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
    assert loss.shape == () and loss.requires_grad
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_forward"]
    d = rec.calls[1][1][0]
    ws = Fn.last_workspace(embed.device)
    assert (d.g.B, d.g.D, d.g.h, d.g.w, d.g.Himg, d.g.Wimg, d.g.K) == (2, 32, 8, 8, 16, 16, 5)
    assert (d.g.max_samples, d.g.max_views, d.g.ignore_label) == (64, 4, -1)
    assert d.embed == embed.data_ptr() and d.labels == labels.data_ptr() and d.seg == seg.data_ptr()
    assert d.predict is None and d.ranks is None and d.mode == 0 and d.precision == 0
    assert d.loss == loss.data_ptr()
    assert abs(d.temperature - 0.2) < 1e-7 and abs(d.base_temperature - 0.1) < 1e-7
    for name in ("keys", "chunk_pref", "counts", "plan", "anchor_meta", "anchors_f32", "anchors_bf16", "inv_norm",
                 "partials", "rowstats", "dpartials", "dA", "row_m2"):
        assert getattr(d, name) == getattr(ws, name).data_ptr(), name
    assert rec.calls[1][1][1] == 0x5EED
    assert ws.busy
    loss.backward()
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_forward", "pcl_step_backward"]
    db = rec.calls[2][1][0]
    assert db.grad_embed == embed.grad.data_ptr() and embed.grad.shape == embed.shape
    assert not ws.busy                                    # workspace handed back by the backward


def test_pending_graphs_get_distinct_workspaces(rec):
    """A workspace holds the row statistics its backward needs: a second forward before the first backward must not
    reuse it; dropping a graph without backward hands the workspace back (weakref finalizer)."""
    embed, labels, seg = _inputs()
    opts = cs.ContrastOptions(max_samples=64, max_views=4)
    l1 = cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
    w1 = Fn.last_workspace(embed.device)
    l2 = cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
    w2 = Fn.last_workspace(embed.device)
    assert w1 is not w2 and w1.busy and w2.busy
    d1, d2 = rec.calls[1][1][0], rec.calls[3][1][0]
    assert d1.rowstats != d2.rowstats and d1.partials != d2.partials
    l1.backward()
    assert not w1.busy and w2.busy
    assert rec.calls[-1][1][0].rowstats == w1.rowstats.data_ptr()      # l1's backward read l1's statistics
    l2.backward()
    assert not w2.busy
    assert rec.calls[-1][1][0].rowstats == w2.rowstats.data_ptr()
    seen = set()
    for _ in range(6):                                    # logged only: no backward
        loss = cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
        seen.add(id(Fn.last_workspace(embed.device)))
        del loss
    assert len(seen) <= 2
    with torch.no_grad():
        cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
    assert not Fn.last_workspace(embed.device).busy


def test_bank_step_passes_queues_and_seed_changes(rec):
    embed, labels, seg = _inputs()
    segq, pixq = torch.randn(5, 6, 32), torch.randn(5, 6, 32)
    opts = cs.ContrastOptions(max_samples=64, max_views=4)
    for _ in range(2):
        cs.pixel_contrast_loss(embed.detach(), labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    d0, d1 = rec.calls[1][1][0], rec.calls[3][1][0]
    assert d0.mode == 1 and (d0.bank_K, d0.bank_M0, d0.bank_M1) == (5, 6, 6)
    assert d0.segment_queue == segq.data_ptr() and d0.pixel_queue == pixq.data_ptr()
    assert d0.seed != d1.seed                             # a fresh sampling stream every call
    assert not Fn.last_workspace(embed.device).busy       # no grad requested: workspace never locked


def test_topk_step_call_sequence(rec):
    embed, labels, seg = _inputs()
    opts = cs.ContrastOptions(max_samples=64, max_views=4, topk_negatives=7, normalize=True)
    loss = cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
    names = [c[0] for c in rec.calls]
    assert names == ["pcl_step_stats", "pcl_select_gather", "pcl_infonce_topk_fwd"]
    ws = Fn.last_workspace(embed.device)
    ms = 64
    sg = rec.calls[1][1]
    assert sg[1] == embed.data_ptr() and sg[2] == ws.keys.data_ptr() and sg[3] == ws.chunk_pref.data_ptr()
    assert sg[4] == ws.plan.data_ptr() and sg[5] is None and sg[7] == 1            # ranks NULL (device rng), normalize
    assert sg[8] == ws.anchor_meta.data_ptr() and sg[9] == ws.anchors_f32.data_ptr() and sg[-1] == 0x5EED
    sw, k, scratch = rec.calls[2][1][0], rec.calls[2][1][1], rec.calls[2][1][2]
    assert k == 7 and scratch == ws.topk_scratch.data_ptr()
    assert sw.anchors == ws.anchors_f32.data_ptr() and sw.plan == ws.plan.data_ptr()
    assert sw.anchor_cls == ws.anchor_meta.data_ptr() + 4 * 2 * ms          # class column of anchor_meta (int32)
    assert sw.diag_col == ws.anchor_meta.data_ptr() + 4 * 3 * ms            # reference row index (Q1)
    assert (sw.a_rows, sw.D, sw.mode) == (ms, 32, 0)
    assert ws.topk_scratch.numel() == 64 * 2048 + 4 * ms
    assert rec.calls[2][1][3] == ws.partials.data_ptr() and rec.calls[2][1][4] == ws.rowstats.data_ptr()
    assert rec.calls[2][1][5] == loss.data_ptr()
    loss.backward()
    names = [c[0] for c in rec.calls]
    assert names[3:] == ["pcl_infonce_topk_bwd", "pcl_scatter_grad"]
    bw = rec.calls[3][1]
    assert bw[1] == 7 and bw[2] == ws.topk_scratch.data_ptr() and bw[3] == ws.rowstats.data_ptr()
    assert bw[5] == ws.dpartials.data_ptr() and bw[6] == ws.dA.data_ptr()
    sc = rec.calls[4][1]
    assert sc[1] == ws.plan.data_ptr() and sc[3] == ws.dA.data_ptr() and sc[6] == 1 and sc[7] == embed.grad.data_ptr()


def test_topk_on_the_tensor_path_call_sequence_and_bad_k(rec):
    """precision='bf16' + topk_negatives: selection, then the tensor-path top-k forward (radix select in the wgmma sweep's
    epilogue) and its backward with the SAME scratch (selection state)."""
    embed, labels, seg = _inputs(D=256)
    loss = cs.pixel_contrast_loss(embed, labels, seg=seg,
                                  options=cs.ContrastOptions(max_samples=64, max_views=4, topk_negatives=3, precision="bf16"))
    ws = Fn.last_workspace(embed.device)
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_select_gather", "pcl_infonce_tc_topk_fwd"]
    fw = rec.calls[2][1]
    assert fw[1] == 3 and fw[2] == ws.topk_scratch.data_ptr() and fw[3] == ws.row_m2.data_ptr()
    assert fw[0].anchors_bf16 == ws.anchors_bf16.data_ptr() and fw[0].mode == 0 and fw[0].a_rows == 64
    loss.backward()
    assert [c[0] for c in rec.calls][3:] == ["pcl_infonce_tc_topk_bwd", "pcl_scatter_grad"]
    assert rec.calls[3][1][1] == 3 and rec.calls[3][1][2] == ws.topk_scratch.data_ptr()
    rec.calls.clear()
    with pytest.raises(_abi.PclError):
        cs.pixel_contrast_loss(embed, labels, seg=seg,
                               options=cs.ContrastOptions(max_samples=64, max_views=4, topk_negatives=-2))


def test_loss_module_reads_topk_key():
    cfg = cs.Configer(cs.cityscapes_contrast_config())
    assert cs.PixelContrastLoss(cfg).options().topk_negatives is None
    cfg.add(["contrast", "topk_negatives"], 32)
    assert cs.PixelContrastLoss(cfg).options().topk_negatives == 32


def test_workspace_cache_is_bounded(rec, monkeypatch):
    """Varying geometries (multi-scale training) must not pile up scratch buffers: idle geometries beyond the bound
    are dropped oldest first, busy ones survive."""
    monkeypatch.setattr(Fn, "_WS_CACHE_MAX", 3)
    opts = cs.ContrastOptions(max_samples=64, max_views=4)
    held = None
    for i, hw in enumerate((8, 10, 12, 14, 16, 18)):
        embed, labels, seg = _inputs(h=hw, w=hw)
        loss = cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
        if i == 0:
            held, held_ws = loss, Fn.last_workspace(embed.device)      # pending graph: its workspace must survive
        else:
            loss.backward()
        assert len(Fn._WS_CACHE) <= 3 + 1
    assert any(held_ws in lst for lst in Fn._WS_CACHE.values())
    held.backward()
    assert not held_ws.busy
    embed, labels, seg = _inputs(h=20, w=20)
    cs.pixel_contrast_loss(embed, labels, seg=seg, options=opts)
    assert len(Fn._WS_CACHE) <= 3


def test_fused_graphed_step_launch_sequence(rec):
    """No bank, precision bf16, D = 256, max_samples <= 1024: the step takes the fused path — zero-fill on the side
    stream, pcl_step_fused_loss (scan+plan, selection seeded from the device counter, one InfoNCE fwd+bwd kernel), then
    the reducing scatter that advances the counter."""
    embed, labels, seg = _inputs(D=256)
    opts = cs.ContrastOptions(max_samples=64, max_views=4, seed=77, precision="bf16")
    step = cs.GraphedContrastStep(embed.detach(), labels, seg=seg, options=opts, grad_scale=0.1, capture=False)
    assert step.fused
    step._fork_zero_fill = lambda: rec.calls.append(("fill", []))
    step._join_zero_fill = lambda: rec.calls.append(("join", []))
    loss, grad = step.replay()
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_fused_select", "fill", "pcl_step_fused_loss", "join",
                                         "pcl_step_fused_scatter"]
    d = rec.calls[1][1][0]
    assert d.sync == step.ws.sync.data_ptr() and d.precision == 1 and d.mode == 0 and d.seed == 77
    assert rec.calls[1][1][1] == step.counter.data_ptr() and rec.calls[1][1][2] is None
    sc = rec.calls[5][1]
    assert sc[1] == step.scale.data_ptr() and sc[2] == step.counter.data_ptr()
    assert sc[0].grad_embed == grad.data_ptr() and sc[0].loss == loss.data_ptr()
    # sparse reset: no fill at all, the previous step's rows travel from the scatter to the next selection
    rec.calls.clear()
    sp = cs.GraphedContrastStep(embed.detach(), labels, seg=seg, options=opts, capture=False, sparse_reset=True)
    sp.replay()
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_fused_select", "pcl_step_fused_loss", "pcl_step_fused_scatter"]
    assert rec.calls[1][1][2] == sp.prev_rows.data_ptr() == rec.calls[3][1][3]
    # a bank, fp32 sweeps or fused=False keep the streaming path
    assert not cs.GraphedContrastStep(embed.detach(), labels, seg=seg, options=opts, capture=False, fused=False).fused
    o32 = cs.ContrastOptions(max_samples=64, max_views=4, precision="fp32")
    assert not cs.GraphedContrastStep(embed.detach(), labels, seg=seg, options=o32, capture=False).fused


def test_graphed_step_launch_sequence(rec):
    """GraphedContrastStep (capture=False: the same launch sequence, eagerly): stats -> device rank draw -> forward
    -> backward on static buffers, the upstream gradient as a device scalar, the rank table wired into the step."""
    embed, labels, seg = _inputs()
    opts = cs.ContrastOptions(max_samples=64, max_views=4, seed=77)
    step = cs.GraphedContrastStep(embed.detach(), labels, seg=seg, options=opts, grad_scale=0.1, capture=False,
                                  overlap_zero_fill=False)
    loss, grad = step.replay()
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_forward_ctr", "pcl_step_backward"]
    d = rec.calls[1][1][0]
    assert d.seed == 77
    assert d.loss == loss.data_ptr() and d.grad_embed == grad.data_ptr() and grad.shape == embed.shape
    assert d.embed == embed.data_ptr() and d.labels == labels.data_ptr() and d.seg == seg.data_ptr()
    assert rec.calls[1][1][1] == step.counter.data_ptr()
    assert rec.calls[2][1][1] == step.scale.data_ptr() and abs(step.scale.item() - 0.1) < 1e-7
    l2, g2 = step.replay()
    assert l2.data_ptr() == loss.data_ptr() and g2.data_ptr() == grad.data_ptr() and step.replays == 2
    # autograd hand-off: the static gradient comes back for the captured tensor only
    e = embed.detach().requires_grad_(True)
    with pytest.raises(_abi.PclError):
        step.apply(torch.zeros_like(e))
    step2 = cs.GraphedContrastStep(e, labels, seg=seg, options=opts, capture=False, overlap_zero_fill=False)
    out = step2.apply(e)
    out.backward()
    assert e.grad.shape == e.shape
    with pytest.raises(_abi.PclError):
        cs.GraphedContrastStep(embed.detach(), labels, seg=seg, capture=False,
                               options=cs.ContrastOptions(max_samples=64, max_views=4, rng="torch_cpu"))
    with pytest.raises(_abi.PclError):
        cs.GraphedContrastStep(embed.detach(), labels.to(torch.int32), seg=seg, options=opts, capture=False)
    # overlapped zero-fill: fork before the first kernel, join before the scatter-only backward
    rec.calls.clear()
    step3 = cs.GraphedContrastStep(embed.detach(), labels, seg=seg, options=opts, capture=False)
    step3._fork_zero_fill = lambda: rec.calls.append(("fork", []))
    step3._join_zero_fill = lambda: rec.calls.append(("join", []))
    step3.replay()
    assert _names(rec) == ["fork", "pcl_step_stats", "pcl_step_forward_ctr", "join", "pcl_step_backward_prezeroed"]
    assert rec.calls[-1][1][0].grad_embed == step3.grad.data_ptr() and rec.calls[-1][1][1] == step3.scale.data_ptr()


def _bank(K=5, M=6, D=32):
    return (torch.randn(K, M, D), torch.zeros(K, dtype=torch.long), torch.randn(K, M, D), torch.zeros(K, dtype=torch.long))


def _names(rec):
    return [c[0] for c in rec.calls]


def test_bank_write_waits_for_the_pending_backward(rec):
    """Trainer order (trainer_contrastive.py:241-255): loss -> enqueue -> backward.  The engine's backward re-reads the
    bank, so the in-place write must land after it; without a pending reader it is immediate."""
    embed, labels, seg = _inputs()
    segq, sp, pixq, pp = _bank()
    opts = cs.ContrastOptions(max_samples=64, max_views=4)
    kw = dict(network_stride=2, memory_size=6, pixel_update_freq=3, distributed=False)
    cs.dequeue_and_enqueue(embed.detach(), labels, segq, sp, pixq, pp, **kw)
    assert _names(rec) == ["pcl_bank_packet", "pcl_bank_apply"]                 # nobody is reading: write at once
    rec.calls.clear()
    loss = cs.pixel_contrast_loss(embed, labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    ws = Fn.last_workspace(embed.device)
    assert Fn.bank_reader(embed.device.index, segq.data_ptr()) is ws
    cs.dequeue_and_enqueue(embed.detach(), labels, segq, sp, pixq, pp, **kw)
    assert _names(rec) == ["pcl_step_stats", "pcl_step_forward", "pcl_bank_packet"] and len(ws.deferred) == 1
    loss.backward()
    assert _names(rec)[3:] == ["pcl_step_backward", "pcl_bank_apply"]
    ap = rec.calls[-1][1]
    assert ap[3] == segq.data_ptr() and ap[4] == sp.data_ptr() and ap[5] == pixq.data_ptr() and ap[6] == pp.data_ptr()
    assert not ws.deferred and ws.bank_key is None and not ws.busy and not Fn._BANK_READERS
    # a different bank is not held back by this reader
    rec.calls.clear()
    loss = cs.pixel_contrast_loss(embed, labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    other = _bank()
    cs.dequeue_and_enqueue(embed.detach(), labels, *other, **kw)
    assert _names(rec)[-2:] == ["pcl_bank_packet", "pcl_bank_apply"]
    # opt-out writes immediately
    cs.dequeue_and_enqueue(embed.detach(), labels, segq, sp, pixq, pp, defer_to_backward=False, **kw)
    assert _names(rec)[-1] == "pcl_bank_apply"
    loss.backward()
    assert not Fn._BANK_READERS


def test_held_back_bank_write_is_never_lost(rec):
    embed, labels, seg = _inputs()
    segq, sp, pixq, pp = _bank()
    opts = cs.ContrastOptions(max_samples=64, max_views=4)
    kw = dict(network_stride=2, memory_size=6, pixel_update_freq=3, distributed=False)
    # graph dropped without backward: the write lands when the graph dies
    loss = cs.pixel_contrast_loss(embed, labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    cs.dequeue_and_enqueue(embed.detach(), labels, segq, sp, pixq, pp, **kw)
    assert "pcl_bank_apply" not in _names(rec)
    del loss
    assert _names(rec)[-1] == "pcl_bank_apply" and not Fn._BANK_READERS
    # a new forward on the same bank first lets the held-back write in (it must see the updated bank)
    rec.calls.clear()
    l1 = cs.pixel_contrast_loss(embed, labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    cs.dequeue_and_enqueue(embed.detach(), labels, segq, sp, pixq, pp, **kw)
    l2 = cs.pixel_contrast_loss(embed, labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    assert _names(rec) == ["pcl_step_stats", "pcl_step_forward", "pcl_bank_packet", "pcl_bank_apply",
                           "pcl_step_stats", "pcl_step_forward"]
    l1.backward(); l2.backward()
    assert _names(rec).count("pcl_bank_apply") == 1 and not Fn._BANK_READERS
    # evaluation (no grad): nothing pending, immediate
    rec.calls.clear()
    with torch.no_grad():
        cs.pixel_contrast_loss(embed, labels, seg=seg, segment_queue=segq, pixel_queue=pixq, options=opts)
    cs.dequeue_and_enqueue(embed.detach(), labels, segq, sp, pixq, pp, **kw)
    assert _names(rec)[-1] == "pcl_bank_apply"


def test_trainer_hook_order_with_bank(rec):
    """ContrastTrainerHook.loss_step + backward: loss (fused seg CE + contrast on the bank), packet build at the
    reference's point of the iteration, bank write right after the contrast backward."""
    K, D = 5, 32
    cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": 2},
                       "loss": {"loss_type": "mem_contrast_ce_loss", "params": {"ce_ignore_index": -1}},
                       "contrast": {"temperature": 0.07, "base_temperature": 0.07, "max_samples": 64, "max_views": 4,
                                    "loss_weight": 0.1, "use_rmi": False, "use_lovasz": False, "warmup_iters": 0,
                                    "with_memory": True, "memory_size": 6, "pixel_update_freq": 3,
                                    "fused_seg_ce": False}})
    bank = cs.MemoryBank(K, 6, D)
    hook = cs.ContrastTrainerHook(cfg, bank)
    embed, labels, seg = _inputs()
    seg = seg.requires_grad_(True)
    out = {"seg": seg, "embed": embed, "key": embed.detach(), "lb_key": labels}
    loss = hook.loss_step(out, labels, iters=3, distributed=True)
    assert _names(rec) == ["pcl_step_stats", "pcl_step_forward", "pcl_bank_packet"]
    loss.backward()
    assert _names(rec)[3:] == ["pcl_step_backward", "pcl_bank_apply"]
    assert rec.calls[-1][1][3] == bank.segment_queue.data_ptr()
    assert seg.grad is not None and embed.grad is not None


def test_fused_seg_ce_wiring(rec):
    g = torch.Generator().manual_seed(1)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(-1, 5, (2, 16, 16), generator=g)
    weight = torch.rand(5, generator=g)
    loss = cs.upsample_cross_entropy(seg, target, weight, ignore_index=-1)
    assert _names(rec) == ["pcl_seg_ce_fwd"]
    a = rec.calls[0][1]
    assert a[0] == seg.data_ptr() and a[1] == target.data_ptr() and a[2] == weight.data_ptr()
    assert tuple(a[3:10]) == (2, 5, 8, 8, 16, 16, -1) and a[11] == loss.data_ptr() and a[12] == 0x5EED
    loss.backward()
    b = rec.calls[1][1]
    assert rec.calls[1][0] == "pcl_seg_ce_bwd" and b[0] == seg.data_ptr() and b[10] == a[10]      # same scratch
    assert b[12] == seg.grad.data_ptr() and seg.grad.shape == seg.shape
    # the wrapper takes the fused path for the reference's plain CE configuration
    cfg = cs.Configer(cs.cityscapes_contrast_config())
    crit = cs.ContrastCELoss(cfg)
    rec.calls.clear()
    import unittest.mock as um
    with um.patch.object(type(crit), "_can_fuse", lambda self, ce, s: self.fused_seg_ce):
        embed, labels, sg = _inputs(K=19)
        out = crit({"seg": sg.requires_grad_(True), "embed": embed}, labels, with_embed=True)
    assert _names(rec) == ["pcl_seg_ce_fwd", "pcl_step_stats", "pcl_step_forward"]
    out.backward()
    assert sorted(_names(rec)[3:]) == ["pcl_seg_ce_bwd", "pcl_step_backward"]


def test_explicit_operand_entry_points(rec, monkeypatch):
    """infonce_forward / infonce_backward on explicit operands, stock and top-k variants (torch.cuda.device stubbed)."""
    monkeypatch.setattr(torch.cuda, "device", _NoCtx)
    g = torch.Generator().manual_seed(2)
    a, c = torch.randn(70, 32, generator=g), torch.randn(200, 32, generator=g)
    ya, yc = torch.randint(0, 4, (70,), generator=g), torch.randint(0, 4, (200,), generator=g)
    loss, rowstats, st = Fn.infonce_forward(a, ya, contrast=c, contrast_cls=yc, temperature=0.1, base_temperature=0.07)
    assert _names(rec) == ["pcl_infonce_fwd"] and rowstats.shape == (6, 70) and len(st) == 3
    sw = rec.calls[0][1][0]
    assert (sw.a_rows, sw.D, sw.mode, sw.n_cols) == (70, 32, 2, 200)
    dA = Fn.infonce_backward(st, rowstats)
    assert _names(rec)[-1] == "pcl_infonce_bwd" and dA.shape == (70, 32)
    rec.calls.clear()
    loss, rowstats, st = Fn.infonce_forward(a, ya, contrast=c, contrast_cls=yc, topk=9)
    assert _names(rec) == ["pcl_infonce_topk_fwd"] and len(st) == 5 and rec.calls[0][1][1] == 9
    scratch = st[4]
    assert scratch.numel() == 128 * 2048 + 4 * 70 and rec.calls[0][1][2] == scratch.data_ptr()
    key, tw, G, E = Fn.topk_selection(st, 70)
    assert key.shape == tw.shape == G.shape == E.shape == (70,)
    dA = Fn.infonce_backward(st, rowstats)
    bw = rec.calls[-1]
    assert bw[0] == "pcl_infonce_topk_bwd" and bw[1][1] == 9 and bw[1][2] == scratch.data_ptr() and dA.shape == (70, 32)
    # self-contrast and bank modes build the descriptor they claim
    rec.calls.clear()
    Fn.infonce_forward(a, ya)
    assert rec.calls[0][1][0].mode == 0
    segq, pixq = torch.randn(4, 6, 32), torch.randn(4, 6, 32)
    Fn.infonce_forward(a, ya, queues=(segq, pixq))
    d = rec.calls[1][1][0]
    assert d.mode == 1 and (d.bank_K, d.bank_M0, d.bank_M1) == (4, 6, 6)


def test_loss_step_timer_never_blocks(rec, monkeypatch):
    """LossStepTimer: events recorded around loss_step, read() only reports steps whose events have completed."""
    clock = {"t": 0.0}

    class FakeEvent:
        done_after = 2                                   # becomes 'complete' two queries after it was recorded

        def __init__(self, enable_timing=False):
            self.t, self.q = None, 0

        def record(self):
            clock["t"] += 1.5
            self.t = clock["t"]

        def query(self):
            self.q += 1
            return self.q >= FakeEvent.done_after

        def elapsed_time(self, other):
            return other.t - self.t

    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    timer = cs.LossStepTimer(depth=3)
    cfg = cs.Configer(cs.cityscapes_contrast_config())
    cfg.add(["contrast", "warmup_iters"], 0)
    cfg.add(["contrast", "fused_seg_ce"], False)
    hook = cs.ContrastTrainerHook(cfg, timer=timer)
    embed, labels, seg = _inputs(K=19)
    assert timer.read() is None
    hook.loss_step({"seg": seg.requires_grad_(True), "embed": embed}, labels, iters=1)
    assert timer.read() is None                          # recorded, not complete yet: no value, no waiting
    assert timer.read() == 1.5                           # complete now
    hook.loss_step({"seg": seg, "embed": embed}, labels, iters=2)
    assert timer.read() == 1.5                           # the newest step is still in flight: last completed value


def test_three_graph_replay_order_of_the_bank_step_on_several_ranks(monkeypatch):
    """world > 1 (graph_step.GraphedContrastStep.replay): graph A (forward + packet) -> the all_gather on ITS OWN stream,
    ordered after A -> graph B (backward sweep) on the caller's stream, not waiting for the all_gather -> the caller's
    stream waits for the all_gather -> graph C (bank write).  PCL_GATHER_OVERLAP=0 / no third graph: A, all_gather, B."""
    from contrastiveseg_b200 import graph_step
    log = []

    class FakeGraph:
        def __init__(self, name): self.name = name
        def replay(self): log.append(f"replay {self.name} on {cur_name[0]}")

    class FakeStream:
        def __init__(self, name): self.name = name
        def wait_stream(self, other): log.append(f"{self.name} waits for {other.name}")

    class Ctx:
        def __init__(self, s): self.s = s
        def __enter__(self): self.prev = cur_name[0]; cur_name[0] = self.s.name
        def __exit__(self, *a): cur_name[0] = self.prev

    cur_name = ["main"]
    main, side = FakeStream("main"), FakeStream("gather")
    monkeypatch.setattr(graph_step.torch.cuda, "current_stream", lambda dev=None: main)
    monkeypatch.setattr(graph_step.torch.cuda, "stream", lambda s: Ctx(s))
    st = object.__new__(graph_step.GraphedContrastStep)
    st.device, st.replays, st.loss, st.grad = None, 0, "loss", "grad"
    st.graph, st.graph_b, st.graph_c, st._gather_stream = FakeGraph("A"), FakeGraph("B"), FakeGraph("C"), side
    st._gather = lambda: log.append(f"all_gather on {cur_name[0]}")
    assert st.replay() == ("loss", "grad")
    assert log == ["replay A on main", "gather waits for main", "all_gather on gather", "replay B on main",
                   "main waits for gather", "replay C on main"]
    del log[:]
    st.graph_c = None
    st.replay()
    assert log == ["replay A on main", "all_gather on main", "replay B on main"]
    assert st.replays == 2
