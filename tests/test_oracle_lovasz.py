"""The float64 Lovasz restatement (oracle/lovasz_port.py) against the reference's own FSCELOVASZLoss and memory wrapper:
the goldens written by tests/golden/make_golden_lovasz.py."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ref_port as P
from oracle.lovasz_port import lovasz_loss

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", ["lovasz_identity", "lovasz_up4", "lovasz_nonint"])
def test_oracle_matches_lovasz_goldens(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    seg, target = torch.from_numpy(z["seg"]), torch.from_numpy(z["target"])
    t0 = target.clone()
    assert abs(lovasz_loss(seg, target, front=torch.float32).item() - float(z["lovasz"])) <= 1e-5 * float(z["lovasz"])
    assert torch.equal(target, t0)
    s = seg.double().requires_grad_(True)
    up = F.interpolate(s, size=target.shape[1:], mode="bilinear", align_corners=True)
    loss = F.cross_entropy(up, target, ignore_index=-1) + lovasz_loss(s, target)
    loss.backward()
    assert abs(loss.item() - float(z["loss"])) <= 1e-5 * abs(float(z["loss"]))
    # the reference's J_i - J_{i-1} in fp32 cancels: its gradient carries ~1e-7 / (1/U) relative noise
    g = z["grad_seg"]
    assert np.abs(s.grad.numpy() - g).max() <= 1e-4 * np.abs(g).max()


def test_oracle_composes_the_wrapper_golden():
    """CE(up(seg)) + Lovasz(seg) + 0.1 * the bank contrast term with the recorded draws."""
    z = np.load(os.path.join(GOLDEN, "lovasz_wrapper_mem.npz"))
    seg, target = torch.from_numpy(z["seg"]), torch.from_numpy(z["target"])
    up = F.interpolate(seg, size=target.shape[1:], mode="bilinear", align_corners=True)
    seg_loss = F.cross_entropy(up, target, ignore_index=-1).item() + lovasz_loss(seg, target, front=torch.float32).item()
    draws = np.split(z["perm_flat"], np.cumsum(z["perm_lens"])[:-1]) if len(z["perm_lens"]) else []
    queue = torch.cat((torch.from_numpy(z["segment_queue"]), torch.from_numpy(z["pixel_queue"])), 1).double()
    contrast = P.pixel_contrast_loss(torch.from_numpy(z["embed"]).double(), target, seg.argmax(1), temperature=0.1,
                                     base_temperature=0.07, max_samples=48, max_views=5, queue=queue,
                                     perm_fn=P.PermReplay([torch.from_numpy(d) for d in draws])).item()
    expect = seg_loss + 0.1 * contrast
    assert abs(expect - float(z["loss"])) <= 1e-5 * abs(float(z["loss"])), (expect, float(z["loss"]))
