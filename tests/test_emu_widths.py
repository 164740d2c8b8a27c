"""The embedding-width cases of test_gpu_widths.py on the emulated kernels (tests/emu: the real .cu sources compiled for
host threads), at reduced sizes: the exact and top-k sweeps, the eager and the captured step, the bank, the L2-normalise
split, the shared-memory opt-in order and the refusals, at every width the GPU file runs.  tools/emu_mutation_widths.py
checks that these cases catch single-line faults in the width-dependent arithmetic.  186 tests, about one minute with
eight pytest-xdist workers on an 8-core CPU."""
import pytest
import torch

import emu_harness
import test_gpu_widths as W
from contrastiveseg_b200 import graph_step

SWEEP_SIZES = {"explicit": (70, 150, None), "self": (100, None, None), "bank": (70, 13, 9), "bank_m1_0": (70, 20, 0)}
TOPK_SIZES = {"explicit": (70, 150), "self": (80, None), "bank": (60, 8)}
STEP = dict(B=2, h=12, w=16, ms=80, mv=8, K=5, M=12)


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(W, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    # no CUDA graph on a CPU: the captured step runs its launch sequence eagerly, the side branch inline
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_capture", lambda self, warmup: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_fork_zero_fill", lambda self: self._side_branch(0))
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_join_zero_fill", lambda self: None)
    return lib


@pytest.mark.parametrize("mode,D", [pytest.param(m, D, id=f"{m}-{D}-w") for m in SWEEP_SIZES for D in W.WIDTHS])
def test_exact_sweeps_on_emulation(emu, mode, D):
    W.check_sweep(mode, D, *SWEEP_SIZES[mode])


@pytest.mark.parametrize("mode,D,k", [pytest.param(m, D, k, id=f"{m}-{D}-k{k}") for m in TOPK_SIZES
                                      for D in W.TOPK_WIDTHS for k in W.TOPK_KS])
def test_topk_sweeps_on_emulation(emu, mode, D, k):
    W.check_topk(mode, D, k, *TOPK_SIZES[mode])


@pytest.mark.parametrize("D,mem,normalize,dtype", W._step_cases())
def test_eager_step_on_emulation(emu, D, mem, normalize, dtype):
    W.check_eager_step(D, mem, normalize, dtype, **STEP)


@pytest.mark.parametrize("mem,D", [pytest.param(m, D, id=f"{'bank' if m else 'self'}-{D}-fp32") for m in (False, True)
                                   for D in (96, 160)])
def test_captured_step_on_emulation(emu, mem, D):
    W.check_captured_step(D, mem, **STEP)


@pytest.mark.parametrize("D", W.BANK_WIDTHS, ids=[f"D{D}" for D in W.BANK_WIDTHS])
def test_bank_enqueue_on_emulation(emu, D):
    W.check_bank_enqueue(D, h=12, w=12)


@pytest.mark.parametrize("C", W.NORM_CHANNELS)
def test_l2_normalize_on_emulation(emu, C):
    W.check_l2_normalize(C)


def test_smem_opt_in_across_widths_on_emulation(emu):
    W.check_opt_in_order(h=12, w=16, ms=80)


@pytest.mark.parametrize("D", [16, 48, 288])
def test_unsupported_width_is_refused_on_emulation(emu, D):
    W.check_width_refused(D)


def test_tensor_path_and_fused_head_refuse_widths_below_256_on_emulation(emu):
    W.check_bf16_refused_below_256()
