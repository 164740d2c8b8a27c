"""Host wiring of ProjectionHead(..., sparse_grad=True) on CPU with the recording library of test_host_wiring.py: the
hand-off calls pcl_step_backward_cols and the head's column entry points and never the dense writer, the dense head
backward or a fill; each fallback calls today's sequence."""
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import functional as Fn
from test_host_wiring import rec  # noqa: F401  (fixture)

DENSE = ["pcl_step_backward", "pcl_proj_bn_bwd_dt", "pcl_proj_bn_input_grad_dt"]
COLS = ["pcl_step_backward_cols", "pcl_proj_bn_bwd_cols_dt", "pcl_proj_bn_input_grad_cols_dt"]


def _head_and_inputs(conv1=False, sparse=True, B=2, C=40, h=8, w=8, K=5):
    head = cs.ProjectionHead(C, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True, fuse_conv1=conv1,
                             sparse_grad=sparse)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, C, h, w, generator=g).requires_grad_(True)
    labels = torch.randint(0, K, (B, 2 * h, 2 * w), generator=g)
    seg = torch.randn(B, K, h, w, generator=g)
    return head, x, labels, seg


def _backward_calls(rec, loss):
    n = len(rec.calls)
    loss.backward()
    return [c for c in rec.calls[n:] if c[0].startswith(("pcl_step_backward", "pcl_proj_bn_bwd", "pcl_proj_bn_input",
                                                          "pcl_fill_zero", "pcl_proj_conv1_bwd"))]


@pytest.mark.parametrize("conv1", [False, True], ids=["bn_relu", "conv1"])
def test_sparse_path_calls_the_column_entry_points(rec, conv1):
    head, x, labels, seg = _head_and_inputs(conv1)
    opts = cs.ContrastOptions(max_samples=64, max_views=4)
    loss = cs.pixel_contrast_loss(head(x), labels, seg=seg, options=opts)
    calls = _backward_calls(rec, loss)
    names = [c[0] for c in calls]
    assert names == COLS + (["pcl_proj_conv1_bwd_dt"] if conv1 else [])
    (_, step), (_, bwd), (_, ig) = calls[:3]
    cols, col_pix = step[2], step[3]
    assert bwd[5] == cols and bwd[6] == col_pix and bwd[7] == 64                 # the loss's columns, max_samples of them
    assert ig[4] == bwd[12] and ig[5] == col_pix and ig[6] == 64                 # the same scratch and pixels
    assert x.grad is not None and x.grad.shape == x.shape
    assert not Fn._SINKS or all(not s.deposits for s in Fn._SINKS.values())      # every deposit consumed


@pytest.mark.parametrize("case", ["retain_grad", "hook", "no_loss", "dense_head", "warmup_skip"])
def test_fallbacks_call_the_dense_sequence(rec, case):
    head, x, labels, seg = _head_and_inputs(sparse=case != "dense_head")
    zn = head(x)
    if case == "retain_grad":
        zn.retain_grad()
    if case == "hook":
        zn.register_hook(lambda g: g)
    if case == "no_loss":
        loss = zn.sum()
    elif case == "warmup_skip":
        cfg = cs.Configer({"data": {"num_classes": 5}, "network": {"stride": 2},
                           "loss": {"params": {"ce_ignore_index": -1}},
                           "contrast": {"temperature": 0.1, "base_temperature": 0.07, "max_samples": 64,
                                        "max_views": 4, "loss_weight": 0.1, "skip_warmup_contrast": True,
                                        "fused_seg_ce": False}})
        loss = cs.ContrastCELoss(cfg)({"seg": seg.requires_grad_(True), "embed": zn}, labels)
    else:
        loss = cs.pixel_contrast_loss(zn, labels, seg=seg, options=cs.ContrastOptions(max_samples=64, max_views=4))
    names = [c[0] for c in _backward_calls(rec, loss)]
    expect = DENSE if case in ("retain_grad", "hook", "dense_head") else DENSE[1:]
    assert names == expect
