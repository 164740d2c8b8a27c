"""The fused Lovasz-softmax seg loss (csrc/pcl_segce.cu, third part) on the emulated kernels (tests/emu: the real
.cu sources compiled for host threads) at reduced sizes, against the float64 oracle: up-sampling and identity geometries, class counts that
take several staged chunks and several sort chunks, label counts across the sort tile, exact ties; and the host wiring
of the autograd function, FSCELOVASZLoss and the contrast wrappers."""
import unittest.mock as um

import pytest
import torch

import contrastiveseg_b200 as cs
import emu_harness
import test_gpu_lovasz as G
from contrastiveseg_b200 import _abi, functional as Fn


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return lib


@pytest.mark.parametrize("B,K,h,w,H,W", [(2, 5, 6, 7, 22, 26), (1, 4, 9, 11, 9, 11), (1, 19, 5, 6, 17, 20),
                                         (1, 40, 4, 5, 12, 14), (1, 3, 1, 40, 1, 2100)])
def test_lovasz_geometries_on_emulation(emu, B, K, h, w, H, W):
    seg, target = G._inputs(B, K, h, w, H, W, seed=K + H)
    G.check_lovasz(seg, target)


def test_lovasz_label_edge_cases_on_emulation(emu):
    B, K, h, w, H, W = 2, 6, 5, 6, 16, 19
    seg, target = G._inputs(B, K, h, w, H, W, seed=3, ignore_index=255)
    target[target == 3] = 0
    target[1, 4, 5] = 3                                     # class 3: a single pixel
    target[0, :2] = 9                                       # out of range: ignored
    G.check_lovasz(seg, target, ignore_index=255)


def test_lovasz_exact_ties_on_emulation(emu):
    G.test_lovasz_exact_ties_follow_the_stable_order()


def test_lovasz_every_pixel_ignored_on_emulation(emu):
    G.test_lovasz_every_pixel_ignored()


def test_lovasz_refusals_on_emulation(emu):
    seg, target = G._inputs(1, 3, 8, 8, 20, 20, seed=5)
    with pytest.raises(_abi.PclError):
        cs.upsample_lovasz_softmax(seg, target[:, :6, :6].contiguous())                # down-sampling
    with pytest.raises(_abi.PclError):
        cs.upsample_lovasz_softmax(torch.zeros(1, 257, 4, 4), torch.zeros(1, 4, 4, dtype=torch.int64))
    lib = emu_harness.emu_library()
    assert lib.pcl_lovasz_scratch_bytes(1, 3, 8, 8, 6, 6) == -3
    assert lib.pcl_lovasz_scratch_bytes(1, 257, 4, 4, 4, 4) == -3
    assert lib.pcl_lovasz_scratch_bytes(2, 3, 8, 8, 32768, 32768) == -3               # N = 2^31
    assert lib.pcl_lovasz_scratch_bytes(0, 3, 8, 8, 8, 8) == -1


def test_fscelovasz_module_on_emulation(emu):
    B, K, H, W = 2, 5, 12, 14
    seg, target = G._inputs(B, K, H, W, H, W, seed=8)
    wts = [1.0, 0.5, 2.0, 1.5, 0.75]
    crit = cs.FSCELOVASZLoss(cs.Configer(G._lovasz_config(ce_weight=wts)))
    loss = crit(seg, target)
    ce = torch.nn.functional.cross_entropy(seg.double(), target, weight=torch.tensor(wts, dtype=torch.float64),
                                           ignore_index=-1)
    expect = ce.item() + G.lovasz_loss(seg, target).item()
    assert abs(loss.item() - expect) <= 1e-5 * abs(expect)


# ---- host wiring ----------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, real):
        self._real, self.calls = real, []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name in ("pcl_lovasz_scratch_bytes", "pcl_strerror", "pcl_last_cuda_error", "pcl_seg_ce_scratch_floats"):
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


def test_lovasz_call_order_and_arguments(rec):
    g = torch.Generator().manual_seed(1)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(-1, 5, (2, 30, 31), generator=g)
    t0 = target.clone()
    loss = cs.upsample_lovasz_softmax(seg, target, ignore_index=4)
    assert [c[0] for c in rec.calls] == ["pcl_lovasz_fwd"]
    a = rec.calls[0][1]
    assert a[0] == seg.data_ptr() and a[1] == target.data_ptr()
    assert tuple(a[2:9]) == (2, 5, 8, 8, 30, 31, 4)
    assert a[10] == loss.data_ptr() and a[11] == 0x5EED
    loss.backward()
    b = rec.calls[1][1]
    assert rec.calls[1][0] == "pcl_lovasz_bwd" and b[0] == seg.data_ptr() and tuple(b[1:9]) == tuple(a[1:9])
    assert b[9] == a[9] and b[11] == seg.grad.data_ptr() and b[12] == 0x5EED          # same scratch
    assert torch.equal(target, t0)


def test_lovasz_bf16_gradient_comes_back_in_bf16(rec):
    seg = torch.randn(1, 3, 6, 6).bfloat16().requires_grad_(True)
    target = torch.randint(0, 3, (1, 12, 12))
    cs.upsample_lovasz_softmax(seg, target).backward()
    assert seg.grad.dtype == torch.bfloat16
    assert rec.calls[0][1][0] != seg.data_ptr()                     # read as an fp32 copy


def _cfg(fused=True, with_memory=True):
    d = G._lovasz_config(with_memory=with_memory)
    d["contrast"]["fused_seg_ce"] = fused
    d["data"]["num_classes"] = 5
    return cs.Configer(d)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("wrapper", ["MemContrastCELoss", "ContrastCELoss"])
def test_lovasz_wrapper_routes(rec, fused, wrapper):
    g = torch.Generator().manual_seed(2)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(0, 5, (2, 32, 32), generator=g)
    cfg = _cfg(fused, with_memory=wrapper == "MemContrastCELoss")
    crit = getattr(cs, wrapper)(cfg, seg_criterion=cs.FSCELOVASZLoss(cfg))
    with um.patch.object(type(crit), "_can_fuse", lambda self, ce, s: self.fused_seg_ce):
        crit({"seg": seg, "embed": torch.randn(2, 16, 8, 8)}, target)
    names = [c[0] for c in rec.calls]
    lov = [c[1] for c in rec.calls if c[0] == "pcl_lovasz_fwd"]
    assert len(lov) == 1
    if fused:
        assert names[:2] == ["pcl_seg_ce_fwd", "pcl_lovasz_fwd"]
        assert tuple(lov[0][2:9]) == (2, 5, 8, 8, 32, 32, -1) and lov[0][0] == seg.data_ptr()
    else:                                                           # F.interpolate first, the CE in torch
        assert "pcl_seg_ce_fwd" not in names
        assert tuple(lov[0][2:9]) == (2, 5, 32, 32, 32, 32, -1)


def test_use_lovasz_still_refused_without_seg_criterion():
    with pytest.raises(NotImplementedError, match="FSCELOVASZLoss"):
        cs.MemContrastCELoss(_cfg())
    with pytest.raises(_abi.PclError):
        cs.upsample_lovasz_softmax(torch.randn(1, 3, 8, 8), torch.zeros(1, 16, 16, dtype=torch.int64))   # CPU
