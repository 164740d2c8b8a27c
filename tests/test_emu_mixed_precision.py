"""bf16 / fp16 inputs on CPU: the tests of test_gpu_mixed_precision.py at small shapes on the emulated kernels (DEV =
"cpu"), the emulator's fp16 conversions against torch's, and the host wiring of half inputs with a recording stub."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import contrastiveseg_b200 as cs
import emu_harness
import test_gpu_mixed_precision as MP
from contrastiveseg_b200 import _abi, bank as bank_mod, functional as Fn, graph_step

SMALL = dict(B=2, h=16, w=16)
HALF_IDS = ["bf16", "fp16"]


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(MP, "DEV", "cpu")
    # no CUDA graph on a CPU: the steps run their launch sequence eagerly, the side branch inline
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_capture", lambda self, warmup: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_fork_zero_fill", lambda self: self._side_branch(0))
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_join_zero_fill", lambda self: None)
    return lib


@pytest.mark.parametrize("precision,normalize,mem", [("fp32", False, False), ("fp32", True, True), ("bf16", False, True),
                                                     ("bf16", True, False)])
@pytest.mark.parametrize("dtype", MP.HALF, ids=HALF_IDS)
def test_eager_half_embed_on_emulation(emu, dtype, precision, normalize, mem):
    MP.test_eager_half_embed_matches_the_fp32_copy(dtype, precision, normalize, mem, ms=64, **SMALL)


@pytest.mark.parametrize("dtype", MP.HALF, ids=HALF_IDS)
def test_half_seg_and_predict_on_emulation(emu, dtype):
    MP.test_half_seg_with_fp32_embed_and_predict_in_place_of_seg(dtype, **SMALL)


def test_fp32_after_half_on_emulation(emu):
    MP.test_fp32_call_after_a_half_call_on_the_same_workspace(**SMALL)


@pytest.mark.parametrize("dtype", MP.HALF, ids=HALF_IDS)
def test_fused_step_on_emulation(emu, dtype):
    MP.test_fused_step_with_full_fill(dtype, False, **SMALL)
    MP.test_fused_step_with_sparse_reset(dtype, False, **SMALL)


@pytest.mark.parametrize("dtype,precision", [(torch.bfloat16, "fp32"), (torch.float16, "bf16")], ids=["bf16-fp32", "fp16-bf16"])
def test_streaming_and_bank_steps_on_emulation(emu, dtype, precision):
    MP.test_streaming_step(dtype, False, precision, **SMALL)
    MP.test_bank_step_with_enqueue_from_half_keys(dtype, False, precision, **SMALL)


@pytest.mark.parametrize("dtype", MP.HALF, ids=HALF_IDS)
def test_dequeue_and_enqueue_on_emulation(emu, dtype):
    MP.test_dequeue_and_enqueue_with_half_keys(dtype, **SMALL)


def test_trainer_hook_under_cpu_autocast_on_emulation(emu, monkeypatch):
    from contrastiveseg_b200 import loss as loss_mod
    monkeypatch.setattr(loss_mod.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)   # fused seg CE on CPU
    MP.test_trainer_hook_with_bank_under_autocast(**SMALL)


def test_refusals_on_emulation(emu):
    MP.test_refusals(**SMALL)


# ------------------------------------------------------------------------------------------------------------------
# the emulator's binary16 conversions (tests/emu/shim/cuda_fp16.h) against torch
# ------------------------------------------------------------------------------------------------------------------
_CONV_SRC = r"""
#include "cuda_fp16.h"
extern "C" void to_half(const float* x, uint16_t* y, int n) { for (int i = 0; i < n; ++i) y[i] = __float2half_rn(x[i]).x; }
extern "C" void from_half(const uint16_t* x, float* y, int n) {
  for (int i = 0; i < n; ++i) { __half h; h.x = x[i]; y[i] = __half2float(h); }
}
"""


def test_fp16_shim_conversions_match_torch(tmp_path):
    src = tmp_path / "conv.cpp"
    src.write_text(_CONV_SRC)
    so = tmp_path / "libconv.so"
    shim = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "shim")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I", shim, str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    f32 = np.float32
    edges = [0.0, -0.0, 1.0, -1.0, 65504.0, 65519.99, 65520.0, -65520.0, 1e6, np.inf, -np.inf,
             2.0 ** -14, 2.0 ** -14 * (1 - 2.0 ** -11), 2.0 ** -24, 2.0 ** -25, 2.0 ** -25 * 1.0000001, 3 * 2.0 ** -26,
             2.0 ** -26, 1e-30, -1e-30, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 1 + 2.0 ** -11 + 2.0 ** -20, 0.1, 1 / 3,
             np.float32(np.finfo(np.float32).tiny), -5.96e-8, 6.1e-5]
    rng = np.random.default_rng(3)
    vals = np.concatenate([np.array(edges, dtype=f32),
                           rng.standard_normal(4000).astype(f32) * np.exp2(rng.integers(-30, 20, 4000)).astype(f32),
                           np.array([np.nan, -np.nan], dtype=f32)])
    n = vals.size
    out = np.zeros(n, dtype=np.uint16)
    lib.to_half(vals.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), n)
    ref = torch.from_numpy(vals).to(torch.float16)
    got = torch.from_numpy(out.view(np.int16)).view(torch.float16)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int16), ref[~nan].view(torch.int16))
    # every binary16 bit pattern back to fp32
    allbits = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    back = np.zeros(65536, dtype=f32)
    lib.from_half(allbits.ctypes.data_as(C.c_void_p), back.ctypes.data_as(C.c_void_p), 65536)
    ref = torch.from_numpy(allbits.view(np.int16)).view(torch.float16).float()
    got = torch.from_numpy(back)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int32), ref[~nan].view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------
# host wiring: half inputs take the fp32 call sequence, with the dtype fields set (and reset by the next fp32 call)
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    HOST_ONLY = {"pcl_version", "pcl_strerror", "pcl_last_cuda_error", "pcl_abi_sizeof", "pcl_select_sizes",
                 "pcl_sweep_sizes", "pcl_tc_sizes", "pcl_topk_scratch_u32", "pcl_seg_ce_scratch_floats",
                 "pcl_bank_packet_floats", "pcl_bank_scratch_floats", "pcl_step_fused_supported", "pcl_launch_count",
                 "pcl_tc_topk_scratch_u32"}

    def __init__(self, real):
        self._real = real
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name in self.HOST_ONLY:
            return fn

        def rec(*args):
            snap = []
            for a in args:
                obj = getattr(a, "_obj", None)               # ctypes.byref(struct): copy the struct at call time
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
    def __init__(self, *a, **k):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


@pytest.fixture
def rec(monkeypatch):
    lib = _Recorder(_abi.load(build_if_missing=True))
    monkeypatch.setattr(Fn._abi, "load", lambda *a, **k: lib)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, name: None)
    monkeypatch.setattr(Fn, "_stream_ptr", lambda device: 0x5EED)
    monkeypatch.setattr(Fn, "_on_device", _NoCtx)
    monkeypatch.setattr(bank_mod, "_is_cuda", lambda t: True)
    Fn.clear_workspaces()
    Fn._BANK_READERS.clear()
    yield lib
    Fn.clear_workspaces()
    Fn._BANK_READERS.clear()


def _inputs(B=2, D=32, h=8, w=8, K=5, s=2):
    g = torch.Generator().manual_seed(0)
    embed = torch.randn(B, D, h, w, generator=g)
    labels = torch.randint(0, K, (B, h * s, w * s), generator=g)
    seg = torch.randn(B, K, h, w, generator=g)
    return embed, labels, seg


def _call(embed, labels, seg, **kw):
    e = embed.detach().clone().requires_grad_(True)
    loss = cs.pixel_contrast_loss(e, labels, seg=seg, options=cs.ContrastOptions(max_samples=64, max_views=4, **kw))
    loss.backward()
    return e


def test_half_inputs_take_the_fp32_call_sequence(rec):
    embed, labels, seg = _inputs()
    for kw in ({}, {"precision": "bf16"}, {"normalize": True}):
        D = 256 if kw.get("precision") == "bf16" else 32
        embed, labels, seg = _inputs(D=D)
        rec.calls.clear()
        _call(embed, labels, seg, **kw)
        ref = [(n, a[0].embed_dtype, a[0].seg_dtype) for n, a in rec.calls]
        assert [r[0] for r in ref] == ["pcl_step_stats", "pcl_step_forward", "pcl_step_backward"]
        assert all(r[1:] == (0, 0) for r in ref)
        for edt, code in ((torch.bfloat16, 1), (torch.float16, 2)):
            for sdt, scode in ((torch.float32, 0), (torch.bfloat16, 1), (torch.float16, 2)):
                rec.calls.clear()
                e = _call(embed.to(edt), labels, seg.to(sdt), **kw)
                assert [(n, a[0].embed_dtype, a[0].seg_dtype) for n, a in rec.calls] == \
                    [(n, code, scode) for n, _, _ in ref]
                d = rec.calls[0][1][0]
                assert d.embed == e.data_ptr() and d.seg != 0
                bw = rec.calls[-1][1][0]
                assert e.grad.dtype == edt and bw.grad_embed == e.grad.data_ptr()
        rec.calls.clear()
        _call(embed, labels, seg, **kw)                          # fp32 again on the same cached workspace
        assert all((a[0].embed_dtype, a[0].seg_dtype) == (0, 0) for _, a in rec.calls)


def test_half_seg_is_not_copied_and_graph_step_and_bank_wiring(rec):
    embed, labels, seg = _inputs(D=256)
    seg_h = seg.to(torch.bfloat16)
    _call(embed, labels, seg_h)
    assert rec.calls[0][1][0].seg == seg_h.data_ptr()           # read in place
    # the fused captured step (eager launch sequence) carries the dtypes into every call
    rec.calls.clear()
    opts = cs.ContrastOptions(max_samples=64, max_views=4, seed=77, precision="bf16")
    e16 = embed.to(torch.float16)
    step = cs.GraphedContrastStep(e16, labels, seg=seg_h, options=opts, capture=False)
    step._fork_zero_fill = lambda: step._side_branch(0)
    step._join_zero_fill = lambda: None
    _, grad = step.replay()
    assert grad.dtype == torch.float16
    assert [c[0] for c in rec.calls] == ["pcl_step_stats", "pcl_step_fused_select", "pcl_step_fused_fill",
                                         "pcl_step_fused_loss", "pcl_step_fused_scatter"]
    assert all((a[0].embed_dtype, a[0].seg_dtype) == (2, 1) for _, a in rec.calls)
    assert rec.calls[-1][1][0].grad_embed == grad.data_ptr()
    # bank: fp32 keys keep pcl_bank_packet, half keys take the typed entry point
    segq, pixq = torch.randn(5, 6, 256), torch.randn(5, 6, 256)
    sp, pp = torch.zeros(5, dtype=torch.long), torch.zeros(5, dtype=torch.long)
    kw = dict(network_stride=2, memory_size=6, pixel_update_freq=3, distributed=False)
    for keys, name, dt in ((embed, "pcl_bank_packet", None), (e16, "pcl_bank_packet_dt", 2),
                           (embed.to(torch.bfloat16), "pcl_bank_packet_dt", 1)):
        rec.calls.clear()
        cs.dequeue_and_enqueue(keys, labels, segq, sp, pixq, pp, **kw)
        assert [c[0] for c in rec.calls] == [name, "pcl_bank_apply"]
        a = rec.calls[0][1]
        assert a[1] == keys.data_ptr()
        if dt is not None:
            assert a[2] == dt and a[3] == labels.data_ptr()
