"""The fused RMI seg loss (csrc/pcl_segce.cu, second part) on the emulated kernels (tests/emu: the real .cu sources compiled for
host threads) at reduced sizes, against the float64 oracle: radius 1-4, pool ways 0 and 1, strides 1-4, label grids
the stride does not divide, K = 1, 19 and 171; and the host wiring of the autograd function and the wrappers."""
import ctypes as C
import unittest.mock as um

import pytest
import torch

import contrastiveseg_b200 as cs
import emu_harness
import test_gpu_rmi as G
from contrastiveseg_b200 import _abi, functional as Fn


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return lib


@pytest.mark.parametrize("radius", [1, 2, 3, 4])
@pytest.mark.parametrize("way", [0, 1])
@pytest.mark.parametrize("stride", [1, 2, 3, 4])
def test_rmi_radius_pool_way_stride_on_emulation(emu, radius, way, stride):
    # 23 x 29 labels: no stride divides either side; 5 x 7 logits up-sampled non-integrally
    G.check_rmi(1, 3, 5, 7, 23, 29, radius=radius, way=way, stride=stride, lambda_way=stride % 2,
                seed=radius * 10 + stride + 100 * way)


@pytest.mark.parametrize("K,h,w,H,W", [(1, 4, 5, 14, 17), (19, 6, 7, 22, 26), (171, 3, 4, 12, 14), (19, 10, 12, 10, 12)])
def test_rmi_classes_and_geometries_on_emulation(emu, K, h, w, H, W):
    G.check_rmi(2, K, h, w, H, W, seed=K)


def test_rmi_label_edge_cases_on_emulation(emu):
    B, K, h, w, H, W = 3, 4, 5, 6, 16, 19
    seg, target = G._inputs(B, K, h, w, H, W, seed=3)
    target[0] = 2
    target[1][target[1] == 3] = 0
    G.check_rmi(B, K, h, w, H, W, seg=seg, target=target)


def test_rmi_every_pixel_ignored_on_emulation(emu):
    G.test_rmi_every_pixel_ignored()


def test_rmi_refusals_on_emulation(emu):
    G.test_rmi_refusals()


def test_rmi_wrapper_goldens_on_emulation(emu, monkeypatch):
    from test_oracle_rmi import golden_wrapper_loss
    monkeypatch.setattr(cs.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)   # fused seg CE on CPU
    for name in ("rmi_wrapper_aux", "rmi_wrapper_mem"):
        got, ref = golden_wrapper_loss(name, "cpu")
        assert abs(got - ref) <= 1e-5 * abs(ref), (name, got, ref)


# ---- host wiring ----------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, real):
        self._real, self.calls = real, []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name in ("pcl_rmi_scratch_bytes", "pcl_strerror", "pcl_last_cuda_error", "pcl_seg_ce_scratch_floats"):
            return fn

        def rec(*args):
            self.calls.append((name, list(args)))
            return 0
        return rec


@pytest.fixture
def rec(monkeypatch):
    lib = _Recorder(_abi.load(build_if_missing=True))
    monkeypatch.setattr(Fn._abi, "load", lambda *a, **k: lib)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, name: None)
    monkeypatch.setattr(Fn, "_stream_ptr", lambda device: 0x5EED)
    monkeypatch.setattr(Fn, "_on_device", emu_harness._NoCtx)
    return lib


def test_rmi_call_order_and_arguments(rec):
    g = torch.Generator().manual_seed(1)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(-1, 5, (2, 30, 31), generator=g)
    t0 = target.clone()
    loss = cs.upsample_rmi_loss(seg, target, num_classes=5, radius=2, pool_way=1, pool_stride=4, weight_lambda=0.25,
                                lambda_way=0, loss_weight=2.0)
    assert [c[0] for c in rec.calls] == ["pcl_rmi_fwd"]
    a = rec.calls[0][1]
    assert a[0] == seg.data_ptr() and a[1] == target.data_ptr()
    assert tuple(a[2:11]) == (2, 5, 8, 8, 30, 31, 2, 1, 4) and a[11] == 0.25 and a[12] == 0 and a[13] == 2.0
    assert a[15] == loss.data_ptr() and a[16] == 0x5EED
    loss.backward()
    b = rec.calls[1][1]
    assert rec.calls[1][0] == "pcl_rmi_bwd" and b[0] == seg.data_ptr() and tuple(b[2:14]) == tuple(a[2:14])
    assert b[14] == a[14] and b[16] == seg.grad.data_ptr() and b[17] == 0x5EED          # same scratch
    assert torch.equal(target, t0)


def test_rmi_bf16_gradient_comes_back_in_bf16(rec):
    seg = torch.randn(1, 3, 6, 6).bfloat16().requires_grad_(True)
    target = torch.randint(0, 3, (1, 12, 12))
    cs.upsample_rmi_loss(seg, target, num_classes=3).backward()
    assert seg.grad.dtype == torch.bfloat16
    assert rec.calls[0][1][0] != seg.data_ptr()                     # read as an fp32 copy


def _cfg(loss_type, use_rmi=True, use_lovasz=False, fused=True):
    d = G._rmi_config(with_memory=loss_type == "mem_contrast_ce_loss")
    d["loss"]["loss_type"] = loss_type
    d["contrast"].update(use_rmi=use_rmi, use_lovasz=use_lovasz, fused_seg_ce=fused)
    d["loss"]["params"]["num_classes"] = 5
    d["data"]["num_classes"] = 5
    return cs.Configer(d)


@pytest.mark.parametrize("fused", [True, False])
def test_rmi_wrapper_wiring(rec, fused):
    g = torch.Generator().manual_seed(2)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(0, 5, (2, 32, 32), generator=g)
    crit = cs.get_seg_loss(_cfg("mem_contrast_ce_loss", use_lovasz=True, fused=fused))      # use_rmi wins
    crit({"seg": seg, "embed": torch.randn(2, 16, 8, 8)}, target)
    assert [c[0] for c in rec.calls] == ["pcl_rmi_fwd"]
    a = rec.calls[0][1]
    assert tuple(a[2:8]) == ((2, 5, 8, 8, 32, 32) if fused else (2, 5, 32, 32, 32, 32))
    assert (a[0] == seg.data_ptr()) == fused
    rec.calls.clear()
    aux = torch.randn(2, 5, 8, 8, generator=g)
    crit = cs.get_seg_loss(_cfg("contrast_auxce_loss", fused=fused))
    with um.patch.object(type(crit), "_can_fuse", lambda self, ce, s: self.fused_seg_ce):
        crit({"seg": seg, "seg_aux": aux, "embed": torch.randn(2, 16, 8, 8)}, target)
    names = [c[0] for c in rec.calls]
    expect = ["pcl_seg_ce_fwd", "pcl_rmi_fwd"] if fused else ["pcl_rmi_fwd"]     # unfused: the aux CE runs in torch
    assert names[:len(expect)] == expect
    # seg_criterion= still overrides everything
    rec.calls.clear()
    mod = torch.nn.Module()
    mod.forward = lambda p, t: p.sum() * 0
    crit = cs.MemContrastCELoss(_cfg("mem_contrast_ce_loss"), seg_criterion=mod)
    crit({"seg": seg, "embed": torch.randn(2, 16, 8, 8)}, target)
    assert "pcl_rmi_fwd" not in [c[0] for c in rec.calls]


def test_rmi_refused_configurations():
    with pytest.raises(NotImplementedError, match="batch"):
        cs.ContrastCELoss(_cfg("contrast_ce_loss"))
    with pytest.raises(NotImplementedError, match="Lovasz"):
        cs.MemContrastCELoss(_cfg("mem_contrast_ce_loss", use_rmi=False, use_lovasz=True))
    with pytest.raises(_abi.PclError):
        cs.upsample_rmi_loss(torch.randn(1, 3, 8, 8), torch.zeros(1, 16, 16, dtype=torch.int64), num_classes=3)   # CPU
