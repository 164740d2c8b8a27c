"""The column-mode checks of test_gpu_graphed_cols.py at small shapes on the emulated kernels (tests/emu: the real .cu
sources compiled for host threads), with the CUDA-graph capture patched out: each step runs its launch sequence with
capture=False semantics."""
import pytest
import torch

import emu_harness
import test_gpu_graphed_cols as GC
import test_gpu_graphed_criterion as T
import test_gpu_projection as P
import test_gpu_projection_bnrelu as PB
import test_gpu_projection_conv1 as PC
import test_gpu_sparse_head as S
from contrastiveseg_b200 import graph_step


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    for m in (GC, T, P, PB, PC, S):
        monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_capture", lambda self, warmup: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_fork_zero_fill", lambda self: self._side_branch(0))
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_join_zero_fill", lambda self: None)
    from contrastiveseg_b200 import loss as loss_mod
    monkeypatch.setattr(loss_mod.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)   # fused seg CE on CPU
    return lib


@pytest.mark.parametrize("mode", list(GC.MODES))
def test_cols_step_matches_the_dense_step_on_emulation(emu, mode):
    GC.check_step(mode, h=8, w=7, ms=48, eager_twin=False)


@pytest.mark.parametrize("mode", ["fused", "simt"])
def test_cols_step_with_a_bf16_embed_on_emulation(emu, mode):
    GC.check_step(mode, torch.bfloat16, h=8, w=7, ms=48, replays=4, eager_twin=False)


def test_fused_cols_past_one_split_on_emulation(emu):
    GC.check_fused_splits(eager_twin=False)


@pytest.mark.parametrize("name", ["ce", "aux_ohem", "mem_rmi"])
def test_cols_criterion_matches_the_dense_criterion_on_emulation(emu, name):
    GC.check_criterion(name, D=32, h=8, w=8)


@pytest.mark.parametrize("conv1", [False, True], ids=["bn_relu", "conv1"])
def test_sparse_head_through_the_cols_step_on_emulation(emu, conv1):
    GC.check_head_apply(conv1, h=8, w=7, replays=3)


def test_sparse_head_through_the_cols_criterion_on_emulation(emu):
    GC.check_head_apply(False, h=8, w=7, replays=2, criterion=True)


def test_retain_grad_falls_back_on_emulation(emu):
    GC.check_retain_grad_falls_back(h=8, w=7)


def test_refusals_and_out_on_emulation(emu):
    GC.check_refusals()
