"""bf16 activations through the fused projection head on CPU: the tests of test_gpu_projection_bf16.py at the small
shapes of test_emu_projection.py on the emulated kernels (DEV = "cpu"), once more under a shuffled thread schedule with
poisoned allocations, and the host wiring of fp32 / bf16 inputs with a recording stub."""
import os
import subprocess
import sys

import pytest
import torch

import contrastiveseg_b200 as cs
import emu_harness
import test_emu_projection as EP
import test_gpu_projection as P
import test_gpu_projection_bf16 as PB
from contrastiveseg_b200 import _abi, functional as Fn
from test_emu_mixed_precision import _NoCtx, _Recorder


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(P, "DEV", "cpu")
    monkeypatch.setattr(PB, "DEV", "cpu")
    return lib


@pytest.mark.parametrize("shape", EP.SMALL)
def test_bf16_forward_and_backward_contracts_on_emulation(emu, shape):
    PB.test_forward_is_the_fp32_forward_rounded(shape)
    PB.test_backward_is_the_fp32_backward_on_the_converted_inputs(shape)


@pytest.mark.parametrize("shape", EP.SMALL[:2])
def test_bf16_matches_fp64_on_emulation(emu, shape):
    PB.test_matches_fp64_on_bf16_activations(shape)


def test_bf16_clamped_pixel_on_emulation(emu):
    PB.test_clamped_pixel_matches_f_normalize()


def test_bf16_bit_reproducible_on_emulation(emu):
    PB.test_bit_reproducible((3, 100, 5, 7))


@pytest.mark.parametrize("proj,xdtype", [("convmlp", torch.float32), ("linear", torch.bfloat16)])
def test_bf16_head_under_cpu_autocast_on_emulation(emu, proj, xdtype):
    PB.test_fused_head_under_autocast_matches_the_unfused_head(proj, xdtype, shape=(2, 40, 6, 7))


def test_bf16_stand_in_iteration_under_cpu_autocast_on_emulation(emu, monkeypatch):
    from contrastiveseg_b200 import loss as loss_mod
    monkeypatch.setattr(loss_mod.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)   # fused seg CE on CPU
    PB.test_autocast_stand_in_iteration_matches_the_unfused_head(B=2, Cin=40, h=8, w=8)


def test_bf16_refusals_on_emulation(emu):
    PB.test_refusals()


def test_bf16_results_do_not_depend_on_the_schedule_or_uninitialised_memory():
    """The emulated bf16 cases again with a shuffled thread / block order and every torch.empty buffer poisoned (NaN):
    a missing barrier or a read of memory the kernels never wrote changes the result."""
    env = dict(os.environ, PCL_EMU_SCHED="random:1", PCL_EMU_POISON="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "on_emulation"], env=env, capture_output=True, text=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout


# ------------------------------------------------------------------------------------------------------------------
# host wiring: fp32 and bf16 inputs take the _dt entry points with PCL_DT_F32 / PCL_DT_BF16
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def rec(monkeypatch):
    lib = _Recorder(_abi.load(build_if_missing=True))
    monkeypatch.setattr(Fn._abi, "load", lambda *a, **k: lib)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, name: None)
    monkeypatch.setattr(Fn, "_stream_ptr", lambda device: 0x5EED)
    monkeypatch.setattr(Fn, "_on_device", _NoCtx)
    return lib


def _run(x, w, b, gzn):
    xx = x.clone().requires_grad_(True)
    zn = cs.project_normalize(xx, w, b)
    zn.backward(gzn)
    return xx, zn


def test_fp32_and_bf16_inputs_take_the_typed_calls_with_their_dtype_code(rec):
    B, Cin, H, W = 2, 40, 3, 5
    g = torch.Generator().manual_seed(0)
    w = torch.randn(256, Cin, 1, 1, generator=g).requires_grad_(True)
    b = torch.randn(256, generator=g).requires_grad_(True)
    x, gzn = torch.randn(B, Cin, H, W, generator=g), torch.randn(B, 256, H, W, generator=g)
    for dtype, code in ((torch.float32, _abi.DT_F32), (torch.bfloat16, _abi.DT_BF16)):
        for gdt in (torch.float32, torch.bfloat16):
            rec.calls.clear()
            xx, zn = _run(x.to(dtype), w, b, gzn.to(gdt))
            calls = [(n, a) for n, a in rec.calls if n != "pcl_proj_workspace_bytes"]
            assert [n for n, _ in calls] == ["pcl_proj_pack", "pcl_proj_fwd_dt", "pcl_proj_bwd_dt"]
            (_, pack), (_, fwd), (_, bwd) = calls
            assert zn.dtype == dtype and xx.grad.dtype == dtype
            # pcl_proj_fwd_dt(x, dtype, wpack, bias, B, Cin, HW, zn, inv_norm, stream)
            assert len(fwd) == 10 and fwd[0] == xx.data_ptr() and fwd[1] == code and fwd[2] == pack[2]
            assert fwd[4:7] == [B, Cin, H * W] and fwd[7] == zn.data_ptr() and fwd[9] == 0x5EED
            # pcl_proj_bwd_dt(x, dtype, zn, inv_norm, gzn, wpack, B, Cin, HW, scratch, gx, gw, gb, stream)
            assert len(bwd) == 14 and bwd[0] == xx.data_ptr() and bwd[1] == code
            assert bwd[2] == zn.data_ptr() and bwd[3] == fwd[8] and bwd[5] == pack[2]
            assert bwd[6:9] == [B, Cin, H * W] and bwd[10] == xx.grad.data_ptr()
