"""Host wiring of the captured step's column mode on the recording library (test_host_wiring.RecordingLib): column mode
never calls a dense-gradient writer or the zero-fill, hands the column writers the step's static buffers and the device
scalars, and dense mode keeps its call sequence."""
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi
from test_host_wiring import _inputs, rec  # noqa: F401  (rec: the recording-library fixture)

DENSE_WRITERS = {"pcl_step_backward", "pcl_step_backward_prezeroed", "pcl_step_fused_scatter", "pcl_step_fused_fill",
                 "pcl_fill_zero"}


def _step(rec, grad, **kw):  # noqa: F811
    step = cs.GraphedContrastStep(kw.pop("embed"), kw.pop("labels"), seg=kw.pop("seg"), capture=False, grad=grad, **kw)
    step._fork_zero_fill = lambda: rec.calls.append(("fill", []))
    step._join_zero_fill = lambda: rec.calls.append(("join", []))
    return step


def test_fused_cols_step_launch_sequence(rec):  # noqa: F811
    embed, labels, seg = _inputs(D=256)
    opts = cs.ContrastOptions(max_samples=64, max_views=4, seed=77, precision="bf16")
    step = _step(rec, "cols", embed=embed.detach(), labels=labels, seg=seg, options=opts, grad_scale=0.1)
    assert step.fused and step.grad is None
    loss, (cols, col_pix) = step.replay()
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_fused_select", "pcl_step_fused_loss",
                                         "pcl_step_fused_cols"]
    d, scale, ctr, c_ptr, p_ptr = rec.calls[3][1][:5]
    assert d.grad_embed is None and d.loss == loss.data_ptr()
    assert scale == step.scale.data_ptr() and ctr == step.counter.data_ptr()
    assert c_ptr == cols.data_ptr() and p_ptr == col_pix.data_ptr()
    assert tuple(cols.shape) == (64, 256) and cols.dtype == torch.float32 and col_pix.dtype == torch.int32
    assert rec.calls[1][1][2] is None                                  # no sparse reset rows
    # dense mode: unchanged
    rec.calls.clear()
    _step(rec, "dense", embed=embed.detach(), labels=labels, seg=seg, options=opts).replay()
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_fused_select", "fill", "pcl_step_fused_loss",
                                         "join", "pcl_step_fused_scatter"]


@pytest.mark.parametrize("kw", [dict(), dict(precision="bf16"), dict(topk_negatives=3), dict(normalize=True)],
                         ids=["simt", "tensor", "topk", "normalize"])
def test_streaming_cols_step_launch_sequence(rec, kw):  # noqa: F811
    embed, labels, seg = _inputs(D=256 if kw.get("precision") else 64)
    opts = cs.ContrastOptions(max_samples=64, max_views=4, seed=5, **kw)
    step = _step(rec, "cols", embed=embed.detach(), labels=labels, seg=seg, options=opts, fused=False)
    assert not step.overlap_zero_fill
    _, (cols, col_pix) = step.replay()
    names = [c[0] for c in rec.calls]
    assert names == ["pcl_step_stats", "pcl_step_forward_ctr", "pcl_step_backward_cols"], names
    d, scale, c_ptr, p_ptr = rec.calls[2][1][:4]
    assert d.grad_embed is None and scale == step.scale.data_ptr()
    assert c_ptr == cols.data_ptr() and p_ptr == col_pix.data_ptr()
    assert not DENSE_WRITERS & set(names)
    rec.calls.clear()
    _step(rec, "dense", embed=embed.detach(), labels=labels, seg=seg, options=opts, fused=False).replay()
    want = (["pcl_step_stats", "pcl_step_forward_ctr", "pcl_step_backward"] if kw.get("topk_negatives") else
            ["fill", "pcl_step_stats", "pcl_step_forward_ctr", "join", "pcl_step_backward_prezeroed"])
    assert [c[0] for c in rec.calls] == want


def test_cols_mode_refusals(rec):  # noqa: F811
    embed, labels, seg = _inputs(D=256)
    opts = cs.ContrastOptions(max_samples=64, max_views=4, precision="bf16")
    with pytest.raises(_abi.PclError):
        _step(rec, "cols", embed=embed.detach(), labels=labels, seg=seg, options=opts, sparse_reset=True)
    with pytest.raises(_abi.PclError):
        _step(rec, "columns", embed=embed.detach(), labels=labels, seg=seg, options=opts)
    assert not rec.calls


@pytest.mark.parametrize("enqueue", [False, True], ids=["bank", "bank_enqueue"])
def test_bank_cols_step_launch_sequence(rec, enqueue):  # noqa: F811
    """Bank steps: the side branch still forks for the enqueue packet, but column mode puts no fill on it and writes
    the columns where dense mode writes the gradient; the bank write keeps its place after the backward."""
    embed, labels, seg = _inputs(D=64)
    K = seg.shape[1]
    bank = cs.MemoryBank(K, 6, 64)
    opts = cs.ContrastOptions(max_samples=64, max_views=4, seed=5, num_classes=K)
    kw = dict(embed=embed.detach(), labels=labels, seg=seg, options=opts, segment_queue=bank.segment_queue,
              pixel_queue=bank.pixel_queue)
    if enqueue:
        kw["enqueue"] = dict(bank=bank, network_stride=2, pixel_update_freq=3)
    seqs = {}
    for grad in ("cols", "dense"):
        rec.calls.clear()
        step = _step(rec, grad, **dict(kw))
        step._fork_zero_fill = lambda s=step: (rec.calls.append(("fork", [])), s._side_branch(0))
        if grad == "cols":
            assert step.grad is None and not step.overlap_zero_fill
        step.replay()
        seqs[grad] = [c[0] for c in rec.calls]
    tail = ["pcl_bank_apply_ctr"] if enqueue else []
    side = ["fork", "pcl_bank_packet_dev"] if enqueue else []
    assert seqs["cols"] == side + ["pcl_step_stats", "pcl_step_forward_ctr"] + (["join"] if enqueue else []) + \
        ["pcl_step_backward_cols"] + tail, seqs["cols"]
    assert not DENSE_WRITERS & set(seqs["cols"])
    assert seqs["dense"] == ["fork"] + side[1:] + ["pcl_step_stats", "pcl_step_forward_ctr", "join",
                                                    "pcl_step_backward_prezeroed"] + tail, seqs["dense"]


def test_cols_to_dense_stores_every_live_column_and_nothing_else():
    """cols_to_dense (the dense fallback of a column-mode apply()): live columns stored with their bits (a -0 entry
    stays -0), +0 everywhere else, unused rows ignored whatever pixel value they carry, each dtype rounded once."""
    from contrastiveseg_b200 import functional as Fn
    g = torch.Generator().manual_seed(3)
    B, D, h, w, n = 2, 32, 5, 7, 9
    cols = torch.randn(n + 3, D, generator=g)
    cols[2, 5] = -0.0
    cols[n:] = 0.
    pix = torch.randperm(B * h * w, generator=g)[:n].to(torch.int32)
    col_pix = torch.cat([pix, torch.full((3,), -1, dtype=torch.int32)])
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        got = Fn.cols_to_dense(cols, col_pix, (B, D, h, w), dt)
        want = torch.zeros(B, D, h * w, dtype=dt)
        for s in range(n):
            q = int(pix[s])
            want[q // (h * w), :, q % (h * w)] = cols[s].to(dt)
        assert got.shape == (B, D, h, w) and got.is_contiguous()
        bits = torch.int32 if dt == torch.float32 else torch.int16
        assert torch.equal(got.view(bits), want.view(B, D, h, w).view(bits)), dt
