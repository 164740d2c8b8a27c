"""The dense-gradient writer cases of test_gpu_grad_writers.py on the emulated kernels (tests/emu: the real .cu sources
compiled for host threads), at reduced sizes: both backward entry points on one forward, bit for bit, at every precision,
normalise setting and embed dtype, top-k refused by the prezeroed call, and pcl_scatter_grad against torch."""
import pytest
import torch

import emu_harness
import test_gpu_grad_writers as GW

STEP = dict(B=2, h=12, w=16, ms=80, mv=8, K=5)


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(GW, "DEV", "cpu")
    monkeypatch.setattr(GW, "_stream", lambda: 0)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return lib


@pytest.mark.parametrize("precision,D,normalize,embed_dtype,topk", GW.step_cases())
def test_backward_entry_points_on_emulation(emu, precision, D, normalize, embed_dtype, topk):
    GW.check_backward_entry_points(precision, D, normalize, embed_dtype, topk, **STEP)


@pytest.mark.parametrize("normalize", [0, 1])
def test_scatter_grad_on_emulation(emu, normalize):
    GW.check_scatter_grad(normalize, D=64, h=8, w=12, ms=96, A=90)
