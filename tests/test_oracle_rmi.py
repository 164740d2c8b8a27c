"""The float64 RMI restatement (oracle/rmi_port.py) against the reference's own RMILoss: the goldens written by
tests/golden/make_golden_rmi.py and, where the reference tree is reachable, the live module."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
from oracle.ref_loader import DictConfiger, reference_root
from oracle.rmi_port import rmi_loss

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LOSS_CASES = ["rmi_up4_r3_max", "rmi_nonint_r2_avg", "rmi_identity_r1", "rmi_up3_r4_max_s4"]


def _kw(params):
    K, radius, way, stride, lam, lambda_way, lw = params[:7]
    return dict(num_classes=int(K), radius=int(radius), pool_way=int(way), pool_stride=int(stride),
                weight_lambda=float(lam), lambda_way=int(lambda_way), loss_weight=float(lw))


@pytest.mark.parametrize("name", LOSS_CASES)
def test_oracle_matches_rmi_goldens(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    seg, target = torch.from_numpy(z["seg"]), torch.from_numpy(z["target"])
    t0 = target.clone()
    # the reference's precisions (fp32 front end, float64 moments): its float64 log-dets agree to 1e-10
    loss32, rmi_bc, _ = rmi_loss(seg, target, front=torch.float32, parts=True, **_kw(z["params"]))
    np.testing.assert_allclose(rmi_bc.numpy(), z["rmi_bc"], rtol=1e-10, atol=1e-12)
    assert abs(loss32.item() - float(z["loss"])) <= 1e-6 * abs(float(z["loss"]))
    assert torch.equal(target, t0)
    # float64 front end: loss and gradient
    s = seg.double().requires_grad_(True)
    loss = rmi_loss(s, target, **_kw(z["params"]))
    loss.backward()
    assert abs(loss.item() - float(z["loss"])) <= 1e-5 * abs(float(z["loss"]))
    g = z["grad_seg"]
    assert np.abs(s.grad.numpy() - g).max() <= 1e-4 * np.abs(g).max()


@pytest.mark.skipif(reference_root() is None, reason="reference tree not reachable")
@pytest.mark.parametrize("name", LOSS_CASES)
def test_oracle_matches_live_reference(name):
    from oracle.ref_loader import load_reference
    load_reference()
    torch.cuda.DoubleTensor = torch.DoubleTensor if not torch.cuda.is_available() else torch.cuda.DoubleTensor
    import lib.loss.rmi_loss as rmi_mod
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    kw = _kw(z["params"])
    seg, target = torch.from_numpy(z["seg"]), torch.from_numpy(z["target"])
    params = {"use_sigmoid": True, "num_classes": kw["num_classes"], "rmi_radius": kw["radius"],
              "rmi_pool_way": kw["pool_way"], "rmi_pool_size": kw["pool_stride"], "rmi_pool_stride": kw["pool_stride"],
              "loss_weight_lambda": kw["weight_lambda"], "loss_weight": kw["loss_weight"], "lambda_way": kw["lambda_way"]}
    up = F.interpolate(seg, size=target.shape[1:], mode="bilinear", align_corners=True)
    ref = rmi_mod.RMILoss(DictConfiger({"loss": {"params": params}}))(up, target.clone()).item()
    ours = rmi_loss(seg, target, front=torch.float32, **kw).item()
    assert abs(ours - ref) <= 1e-6 * abs(ref)


def golden_wrapper_loss(name, dev):
    """(engine wrapper loss, reference wrapper loss) of a use_rmi wrapper golden (with_embed=False: the seg
    composition; the contrast term enters with weight 0)."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    K, radius, way, stride, lam, lambda_way, lw, w_seg, w_aux, mem = z["params"]
    mem = bool(mem)
    d = cs.cityscapes_contrast_config(with_memory=mem)
    d["data"]["num_classes"] = int(K)
    d["contrast"].update(use_rmi=True, max_samples=48, max_views=5, loss_weight=0.1, rng="torch_cpu")
    d["loss"]["params"].update(use_sigmoid=True, num_classes=int(K), rmi_radius=int(radius), rmi_pool_way=int(way),
                               rmi_pool_size=int(stride), rmi_pool_stride=int(stride), loss_weight_lambda=float(lam),
                               loss_weight=float(lw), lambda_way=int(lambda_way))
    d["network"]["loss_weights"] = {"seg_loss": float(w_seg), "aux_loss": float(w_aux)}
    cfg = cs.Configer(d)
    crit = cs.MemContrastCELoss(cfg) if mem else cs.ContrastAuxCELoss(cfg)
    preds = {"seg": torch.from_numpy(z["seg"]).to(dev), "embed": torch.from_numpy(z["embed"]).to(dev)}
    if not mem:
        preds["seg_aux"] = torch.from_numpy(z["seg_aux"]).to(dev)
    got = crit(preds, torch.from_numpy(z["target"]).to(dev), with_embed=False).item()
    return got, float(z["loss"])


@pytest.mark.parametrize("name", ["rmi_wrapper_aux", "rmi_wrapper_mem"])
def test_oracle_composes_the_wrapper_goldens(name):
    """The wrappers' seg terms: RMI(seg) (+ 0.4 CE(seg_aux) for the aux wrapper) from the oracle."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    K, radius, way, stride, lam, lambda_way, lw, w_seg, w_aux, mem = z["params"]
    target = torch.from_numpy(z["target"])
    kw = _kw(z["params"])
    expect = w_seg * rmi_loss(torch.from_numpy(z["seg"]), target, front=torch.float32, **kw).item()
    if not mem:
        aux = F.interpolate(torch.from_numpy(z["seg_aux"]), size=target.shape[1:], mode="bilinear", align_corners=True)
        expect += w_aux * F.cross_entropy(aux, target, ignore_index=-1).item()
    assert abs(expect - float(z["loss"])) <= 1e-6 * abs(float(z["loss"]))
