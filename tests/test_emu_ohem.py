"""The fused OHEM CE (csrc/pcl_segce.cu, fourth part) on the emulated kernels (tests/emu: the real .cu sources compiled
for host threads) at reduced sizes, against the float64 oracle: both branches, up-sampling and identity geometries,
class counts that take several staged chunks (K = 40, 171), exact ties at the kth value, min_kept >= n, n = 0 and
n = 1, weights and 'sum'; the loss bits under shuffled schedules and poisoned buffers; and the host wiring of the
autograd function, FSOhemCELoss, FSAuxOhemCELoss and the three contrast wrappers."""
import os
import subprocess
import sys
import unittest.mock as um

import pytest
import torch

import contrastiveseg_b200 as cs
import emu_harness
import test_gpu_ohem as G
from contrastiveseg_b200 import _abi, functional as Fn


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return lib


@pytest.mark.parametrize("branch", ["threshold", "select"])
@pytest.mark.parametrize("B,K,h,w,H,W", [(2, 5, 6, 7, 22, 26), (1, 4, 9, 11, 9, 11), (1, 19, 5, 6, 17, 20),
                                         (1, 40, 4, 5, 12, 14), (1, 171, 3, 4, 9, 10)])
def test_ohem_geometries_on_emulation(emu, B, K, h, w, H, W, branch):
    seg, target = G._inputs(B, K, h, w, H, W, seed=K + H)
    thresh = G.median_thresh(seg, target)
    mk = G.branch_min_kept(seg, target, branch, thresh)
    G.check_ohem(seg, target, thresh=thresh, min_kept=mk, branch=branch)


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_weights_and_reductions_on_emulation(emu, reduction):
    seg, target = G._inputs(2, 6, 5, 6, 16, 19, seed=3, ignore_index=255)
    target[0, :2] = 9                                       # out of range: ignored
    weight = torch.tensor([0.5, 1.0, 1.5, 2.0, 0.75, 1.25])
    for branch in ("threshold", "select"):
        mk = G.branch_min_kept(seg, target, branch, 0.4, ignore_index=255)
        G.check_ohem(seg, target, weight=weight, ignore_index=255, thresh=0.4, min_kept=mk, reduction=reduction,
                     branch=branch)


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_exact_ties_on_emulation(emu, reduction):
    G.test_ohem_exact_ties_are_in_or_out_together(reduction)


def test_ohem_min_kept_at_least_n_on_emulation(emu):
    seg, target = G._inputs(1, 5, 6, 7, 15, 18, seed=12)
    G.check_ohem(seg, target, thresh=0.5, min_kept=10 ** 9, branch="select")


@pytest.mark.parametrize("reduction", ["mean", "sum"])
def test_ohem_no_labelled_pixel_and_empty_selection_on_emulation(emu, reduction):
    G.test_ohem_no_labelled_pixel_gives_zero(reduction)
    G.test_ohem_empty_selection(reduction)


def test_ohem_single_pixel_selected_on_emulation(emu):
    seg, _ = G._inputs(1, 5, 6, 7, 15, 18, seed=13)
    one = torch.full((1, 15, 18), -1, dtype=torch.int64)
    one[0, 7, 9] = 2                                        # n = 1 with thresh above its p_t: selected by thresh
    G.check_ohem(seg, one, thresh=1.0, min_kept=100, branch="threshold", gap=False)


def test_ohem_refusals_on_emulation(emu):
    seg, target = G._inputs(1, 3, 8, 8, 20, 20, seed=5)
    with pytest.raises(_abi.PclError):
        cs.upsample_ohem_cross_entropy(seg, target[:, :6, :6].contiguous())                # down-sampling
    with pytest.raises(_abi.PclError):
        cs.upsample_ohem_cross_entropy(torch.zeros(1, 257, 4, 4), torch.zeros(1, 4, 4, dtype=torch.int64))
    with pytest.raises(NotImplementedError):
        cs.upsample_ohem_cross_entropy(seg, target, reduction="none")
    lib = emu_harness.emu_library()
    assert lib.pcl_ohem_ce_scratch_bytes(1, 3, 8, 8, 6, 6) == -3
    assert lib.pcl_ohem_ce_scratch_bytes(1, 257, 4, 4, 4, 4) == -3
    assert lib.pcl_ohem_ce_scratch_bytes(2, 3, 8, 8, 32768, 32768) == -3               # N = 2^31
    assert lib.pcl_ohem_ce_scratch_bytes(0, 3, 8, 8, 8, 8) == -1


def test_ohem_loss_bits_on_emulation(emu, capsys):
    """Prints the loss bits of both branches; the test below compares them across schedules and poisoned buffers."""
    seg, target = G._inputs(2, 19, 5, 6, 17, 20, seed=21)
    for branch in ("threshold", "select"):
        mk = G.branch_min_kept(seg, target, branch, 0.3)
        sel = Fn.ohem_selection(seg, target, thresh=0.3, min_kept=mk)
        assert sel["branch"] == branch
        with capsys.disabled():
            print(f"\nLOSSBITS {branch} {sel['loss'].item().hex()} {sel['count']}")


def test_results_do_not_depend_on_the_schedule_or_uninitialised_memory():
    """The emulated cases again with reversed and shuffled thread / block orders, and with every torch.empty buffer
    poisoned: the tests pass and the loss is bit-identical to the default schedule's."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    bits = []
    for extra in ({}, {"PCL_EMU_SCHED": "reverse"}, {"PCL_EMU_SCHED": "random:5", "PCL_EMU_POISON": "1"},
                  {"PCL_EMU_POISON": "1"}):
        env = dict(os.environ, **extra)
        r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-s",
                            "-p", "no:cacheprovider", "-k", "on_emulation"], env=env, capture_output=True, text=True,
                           cwd=root)
        assert r.returncode == 0, (extra, r.stdout[-3000:] + r.stderr[-2000:])
        bits.append(sorted(line for line in r.stdout.splitlines() if line.startswith("LOSSBITS")))
        assert len(bits[-1]) == 2, r.stdout[-2000:]
    assert all(b == bits[0] for b in bits), bits


# ---- host wiring ----------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, real):
        self._real, self.calls = real, []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name in ("pcl_ohem_ce_scratch_bytes", "pcl_strerror", "pcl_last_cuda_error", "pcl_seg_ce_scratch_floats"):
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


def test_ohem_call_order_and_arguments(rec):
    g = torch.Generator().manual_seed(1)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(-1, 5, (2, 30, 31), generator=g)
    weight = torch.rand(5, generator=g)
    t0 = target.clone()
    loss = cs.upsample_ohem_cross_entropy(seg, target, weight, ignore_index=4, thresh=0.9, min_kept=0, reduction="sum")
    assert [c[0] for c in rec.calls] == ["pcl_ohem_ce_fwd"]
    a = rec.calls[0][1]
    assert a[0] == seg.data_ptr() and a[1] == target.data_ptr() and a[2] == weight.data_ptr()
    assert tuple(a[3:10]) == (2, 5, 8, 8, 30, 31, 4)
    assert a[10] == 0.9 and a[11] == 1 and a[12] == 1                 # min_kept = max(1, 0); 'sum'
    assert a[14] == loss.data_ptr() and a[15] == 0x5EED
    loss.backward()
    b = rec.calls[1][1]
    assert rec.calls[1][0] == "pcl_ohem_ce_bwd" and tuple(b[:10]) == tuple(a[:10])
    assert b[10] == a[13] and b[12] == seg.grad.data_ptr() and b[13] == 0x5EED      # same scratch
    assert torch.equal(target, t0)
    for red, code in (("mean", 0), ("elementwise_mean", 0)):
        cs.upsample_ohem_cross_entropy(seg, target, reduction=red)
        assert rec.calls[-1][1][12] == code


def test_ohem_bf16_gradient_comes_back_in_bf16(rec):
    seg = torch.randn(1, 3, 6, 6).bfloat16().requires_grad_(True)
    target = torch.randint(0, 3, (1, 12, 12))
    cs.upsample_ohem_cross_entropy(seg, target).backward()
    assert seg.grad.dtype == torch.bfloat16
    assert rec.calls[0][1][0] != seg.data_ptr()                     # read as an fp32 copy


def _cfg(fused=True, with_memory=False, **params):
    d = G._ohem_config(with_memory=with_memory, thresh=0.8, min_kept=123)
    d["loss"]["params"].update(params)
    d["contrast"]["fused_seg_ce"] = fused
    d["data"]["num_classes"] = 5
    return cs.Configer(d)


def test_ohem_modules_read_the_config(rec):
    crit = cs.FSOhemCELoss(_cfg(ce_weight=[1.0, 2.0, 3.0, 4.0, 5.0], ce_reduction="sum", ce_ignore_index=255,
                                ohem_minkeep=-5))
    assert crit.thresh == 0.8 and crit.min_kept == 1 and crit.reduction == "sum" and crit.ignore_label == 255
    assert torch.equal(crit.weight, torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0]))
    seg = torch.randn(1, 5, 6, 6)
    crit(seg, torch.randint(0, 5, (1, 6, 6)))
    a = rec.calls[-1][1]
    assert tuple(a[3:10]) == (1, 5, 6, 6, 6, 6, 255) and a[11] == 1 and a[12] == 1
    aux = cs.FSAuxOhemCELoss(_cfg())                       # no loss_type assertion
    assert isinstance(aux.ohem_ce_loss, cs.FSOhemCELoss)
    with pytest.raises(NotImplementedError):
        cs.FSOhemCELoss(_cfg(ce_reduction="none"))(seg, torch.randint(0, 5, (1, 6, 6)))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("wrapper", ["ContrastCELoss", "MemContrastCELoss"])
def test_ohem_wrapper_routes(rec, fused, wrapper):
    g = torch.Generator().manual_seed(2)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(0, 5, (2, 32, 32), generator=g)
    cfg = _cfg(fused, with_memory=wrapper == "MemContrastCELoss")
    crit = getattr(cs, wrapper)(cfg, seg_criterion=cs.FSOhemCELoss(cfg))
    crit({"seg": seg, "embed": torch.randn(2, 16, 8, 8)}, target)
    names = [c[0] for c in rec.calls]
    ohem = [c[1] for c in rec.calls if c[0] == "pcl_ohem_ce_fwd"]
    assert len(ohem) == 1 and "pcl_seg_ce_fwd" not in names
    assert ohem[0][10] == pytest.approx(0.8) and ohem[0][11] == 123
    if fused:
        assert tuple(ohem[0][3:10]) == (2, 5, 8, 8, 32, 32, -1) and ohem[0][0] == seg.data_ptr()
    else:                                                           # F.interpolate first, the identity geometry
        assert tuple(ohem[0][3:10]) == (2, 5, 32, 32, 32, 32, -1)


@pytest.mark.parametrize("fused", [True, False])
def test_ohem_aux_wrapper_route(rec, fused):
    g = torch.Generator().manual_seed(3)
    seg = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    aux = torch.randn(2, 5, 8, 8, generator=g).requires_grad_(True)
    target = torch.randint(0, 5, (2, 32, 32), generator=g)
    cfg = _cfg(fused)
    crit = cs.ContrastAuxCELoss(cfg, seg_criterion=cs.FSAuxOhemCELoss(cfg))
    with um.patch.object(type(crit), "_can_fuse", lambda self, ce, s: self.fused_seg_ce):
        crit({"seg": seg, "seg_aux": aux, "embed": torch.randn(2, 16, 8, 8)}, target)
    names = [c[0] for c in rec.calls]
    ohem = [c[1] for c in rec.calls if c[0] == "pcl_ohem_ce_fwd"]
    assert len(ohem) == 1
    if fused:                                                       # aux CE on the fused seg CE, OHEM on the seg logits
        ce = [c[1] for c in rec.calls if c[0] == "pcl_seg_ce_fwd"]
        assert len(ce) == 1 and ce[0][0] == aux.data_ptr()
        assert ohem[0][0] == seg.data_ptr() and tuple(ohem[0][3:10]) == (2, 5, 8, 8, 32, 32, -1)
    else:
        assert "pcl_seg_ce_fwd" not in names
        assert tuple(ohem[0][3:10]) == (2, 5, 32, 32, 32, 32, -1)
