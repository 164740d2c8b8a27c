"""The tests of test_gpu_graphed_criterion.py on the emulated kernels (tests/emu: the real .cu sources compiled for host
threads), at reduced sizes, with the CUDA-graph capture patched out: the criterion runs its launch sequence eagerly."""
import pytest
import torch

import emu_harness
import test_gpu_graphed_criterion as T
import test_gpu_many_classes as M
from contrastiveseg_b200 import graph_step


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    for m in (T, M):
        monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_capture", lambda self, warmup: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_fork_zero_fill", lambda self: self._side_branch(0))
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_join_zero_fill", lambda self: None)
    return lib


@pytest.mark.parametrize("B,K,h,w,H,W,weighted,ignore_index", [
    (1, 2, 5, 6, 13, 37, False, -1),
    (2, 19, 6, 7, 20, 26, True, 255),
    (1, 25, 6, 7, 20, 26, True, -1),           # two class chunks
    (1, 171, 4, 4, 10, 9, False, 255),
    (1, 19, 11, 35, 11, 35, True, -1),         # identity geometry
])
def test_seg_ce_fwd_bwd_on_emulation(emu, B, K, h, w, H, W, weighted, ignore_index):
    T.check_fwd_bwd(B, K, h, w, H, W, weighted, ignore_index, seed=K)


def test_seg_ce_fwd_bwd_every_pixel_ignored_on_emulation(emu):
    T.check_fwd_bwd(1, 19, 5, 6, 13, 17, True, 255, all_ignored=True)


@pytest.mark.parametrize("H,W", [(5, 11), (9, 6), (4, 5)])
def test_seg_ce_two_call_every_pixel_ignored_below_the_logit_grid_on_emulation(emu, H, W):
    T.check_two_call_every_pixel_ignored(H, W)


def test_seg_ce_fwd_bwd_refuses_down_sampling_on_emulation(emu):
    T.test_seg_ce_fwd_bwd_refuses_down_sampling()


@pytest.fixture
def emu_fused(emu, monkeypatch):
    from contrastiveseg_b200 import loss as loss_mod
    monkeypatch.setattr(loss_mod.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)   # fused seg CE on CPU
    return emu


@pytest.mark.parametrize("name,dtype", [("ce", torch.float32), ("ce_lovasz", torch.bfloat16), ("ce_ohem", torch.float32),
                                        ("aux_ce", torch.bfloat16), ("aux_rmi", torch.float32),
                                        ("aux_ohem", torch.float32), ("mem_rmi", torch.bfloat16)])
def test_graphed_criterion_on_emulation(emu_fused, name, dtype):
    T.check_criterion(name, dtype, D=32, h=8, w=8, replays=2)


def test_graphed_criterion_bank_step_on_emulation(emu_fused):
    T.check_criterion("mem_lovasz", torch.float32, D=32, h=8, w=8, replays=2, enqueue=True)


def test_graphed_criterion_refusals_on_emulation(emu_fused):
    T.check_refusals(D=32, h=8, w=8)
