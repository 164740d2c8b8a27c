"""The float64 OHEM CE restatement (oracle/ohem_port.py) against the reference's own FSOhemCELoss and FSAuxOhemCELoss:
the goldens written by tests/golden/make_golden_ohem.py, and the live reference where its tree is importable."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.ohem_port import ohem_loss, ohem_loss_and_grad
from oracle.ref_loader import DictConfiger, load_reference, reference_root

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["ohem_thresh_branch", "ohem_minkept_branch", "ohem_minkeep_ge_n", "ohem_weight", "ohem_sum", "ohem_ignore255",
         "ohem_bilinear"]


def _load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    kw = {"thresh": float(z["thresh"]), "min_kept": int(z["min_kept"]), "reduction": str(z["reduction"]),
          "ignore_index": int(z["ignore_index"]),
          "weight": torch.from_numpy(z["weight"]) if z["weight"].size else None}
    return z, torch.from_numpy(z["seg"]), torch.from_numpy(z["target"]), kw


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_ohem_goldens(name):
    z, seg, target, kw = _load(name)
    t0 = target.clone()
    ref = float(z["loss"])
    assert abs(ohem_loss(seg, target, front=torch.float32, **kw).item() - ref) <= 2e-6 * abs(ref)
    assert torch.equal(target, t0)
    d, g = ohem_loss_and_grad(seg, target, **kw)
    assert abs(d["loss"].item() - ref) <= 1e-5 * abs(ref)
    gr = z["grad_seg"]
    assert np.abs(g.numpy() - gr).max() <= 1e-5 * np.abs(gr).max()


def test_goldens_cover_both_branches_and_min_kept_above_n():
    def branch(name):
        z, seg, target, kw = _load(name)
        d = ohem_loss(seg, target, details=True, **kw)
        return d, kw
    d, kw = branch("ohem_thresh_branch")
    assert d["threshold"] == float(np.float32(kw["thresh"]))                # kth < thresh: thresh decides
    d, kw = branch("ohem_minkept_branch")
    assert d["threshold"] > float(np.float32(kw["thresh"])) and d["count"] == kw["min_kept"]
    d, kw = branch("ohem_minkeep_ge_n")
    assert kw["min_kept"] >= d["n"] and d["count"] == d["n"] - 1            # m = n - 1: all but the largest p_t


def test_oracle_composes_the_aux_golden():
    z = np.load(os.path.join(GOLDEN, "ohem_aux_bilinear.npz"))
    seg, aux, target = (torch.from_numpy(z[k]).double().requires_grad_(True) for k in ("seg", "aux", "target"))
    target = target.detach().long()
    H, W = target.shape[1:]
    up_aux = F.interpolate(aux, size=(H, W), mode="bilinear", align_corners=True)
    loss = (float(z["seg_w"]) * ohem_loss(seg, target, thresh=float(z["thresh"]), min_kept=int(z["min_kept"])) +
            float(z["aux_w"]) * F.cross_entropy(up_aux, target, ignore_index=-1))
    loss.backward()
    assert abs(loss.item() - float(z["loss"])) <= 1e-5 * abs(float(z["loss"]))
    for g, key in ((seg.grad, "grad_seg"), (aux.grad, "grad_aux")):
        assert np.abs(g.numpy() - z[key]).max() <= 1e-5 * np.abs(z[key]).max()


def test_oracle_edge_definitions():
    g = torch.Generator().manual_seed(3)
    seg = torch.randn(1, 4, 6, 7, generator=g)
    none = torch.full((1, 6, 7), -1, dtype=torch.int64)
    d, grad = ohem_loss_and_grad(seg, none)
    assert d["loss"].item() == 0.0 and d["n"] == 0 and torch.count_nonzero(grad) == 0
    one = none.clone()
    one[0, 2, 3] = 1                                          # n = 1: m = 0, threshold = max(its p_t, thresh)
    d, grad = ohem_loss_and_grad(seg, one, thresh=0.0)
    assert np.isnan(d["loss"].item()) and d["count"] == 0 and torch.count_nonzero(grad) == 0
    assert ohem_loss(seg, one, thresh=0.0, reduction="sum").item() == 0.0
    assert ohem_loss(seg, one, thresh=1.0, details=True)["count"] == 1
    with pytest.raises(NotImplementedError):
        ohem_loss(seg, one, reduction="none")


needs_ref = pytest.mark.skipif(reference_root() is None, reason="reference tree not reachable")


@needs_ref
@pytest.mark.parametrize("reduction,weight", [("elementwise_mean", None), ("sum", [0.5, 1.0, 2.0, 1.5, 0.8])])
def test_oracle_matches_live_reference(reduction, weight):
    load_reference()
    import lib.loss.loss_helper as lh
    from oracle.ohem_port import gap_labels
    g = torch.Generator().manual_seed(11)
    seg = (torch.rand(2, 5, 14, 16, generator=g) * 2 - 1) * 3
    target = torch.randint(0, 5, (2, 14, 16), generator=g)
    target[torch.rand(2, 14, 16, generator=g) < 0.1] = -1
    params = {"ohem_thresh": 0.45, "ohem_minkeep": 150, "ce_reduction": reduction, "ce_ignore_index": -1}
    if weight is not None:
        params["ce_weight"] = weight
    wt = torch.tensor(weight) if weight is not None else None
    target = gap_labels(seg, target, weight=wt, thresh=0.45, min_kept=150, reduction=reduction)
    x = seg.clone().requires_grad_(True)
    ref = lh.FSOhemCELoss(DictConfiger({"loss": {"params": params}}))(x, target.clone())
    ref.backward()
    d, grad = ohem_loss_and_grad(seg, target, weight=wt, thresh=0.45, min_kept=150, reduction=reduction)
    assert abs(d["loss"].item() - ref.item()) <= 1e-5 * abs(ref.item())
    assert (grad - x.grad.double()).abs().max().item() <= 1e-5 * x.grad.abs().max().item()
