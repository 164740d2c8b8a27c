"""The many-class cases of test_gpu_many_classes.py on the emulated kernels (tests/emu: the real .cu sources compiled
for host threads; the tensor path on the functional wgmma / TMA model), at reduced sizes: a second class pass of the
seg-CE kernels, the K > 32 argmax loop with ties, the plan past its shared-memory table, the one-kernel InfoNCE of the
captured step with 171 classes and the bank at 256 classes.  tools/emu_mutation_classes.py checks that these cases
catch single-line faults in those paths."""
import pytest
import torch

import emu_harness
import test_gpu_many_classes as M
import test_gpu_parity as G


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    for m in (M, G):
        monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    # the GPU tests rely on `.to(DEV)` producing a NEW tensor (host -> device copy); `.to("cpu")` would alias the source
    orig_to = torch.Tensor.to

    def to(self, *a, **k):
        r = orig_to(self, *a, **k)
        if r is self and len(a) == 1 and not k and isinstance(a[0], str) and a[0] == "cpu":
            return self.clone()
        return r

    monkeypatch.setattr(torch.Tensor, "to", to)
    return lib


@pytest.mark.parametrize("K,weighted", [(25, False), (33, True), (49, False), (171, True)])
def test_seg_ce_class_chunks_on_emulation(emu, K, weighted):
    M.test_seg_ce_class_chunk_boundaries(K, weighted, B=2, h=9, w=11, H=20, W=26)


def test_seg_ce_down_sampling_40_classes_on_emulation(emu):
    """Gather backward; the forward's source patch (200 x 63 cells) leaves room for one class per pass."""
    M.test_seg_ce_other_geometries(1, 40, 200, 200, 24, 24, True)


def test_seg_ce_ignore_255_of_256_classes_on_emulation(emu):
    M.test_seg_ce_dataset_geometries(1, 256, 6, 7, 20, 26, True, 255)


@pytest.mark.parametrize("K", [33, 171])
def test_argmax_ties_on_emulation(emu, K):
    M.test_argmax_ties_take_the_first_maximum(K, torch.bfloat16 if K == 171 else torch.float32, h=32, w=32, ms=1024, mv=3,
                                              D=32)


def test_plan_past_the_shared_table_on_emulation(emu):
    """B = 9, K = 256: the per-(image, key) totals no longer fit the 4096-entry shared table."""
    M.test_plan_counts_past_the_shared_table(9, 256, h=48, w=48, mv=4, D=32)


def test_fused_captured_step_171_classes_on_emulation(emu, monkeypatch):
    from contrastiveseg_b200 import graph_step
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_capture", lambda self, warmup: None)
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_fork_zero_fill", lambda self: self._side_branch(0))
    monkeypatch.setattr(graph_step.GraphedContrastStep, "_join_zero_fill", lambda self: None)
    M.test_fused_captured_step_with_many_anchor_classes(171, 4, 85)


def test_bank_enqueue_256_classes_on_emulation(emu):
    M.test_bank_enqueue_with_many_classes(256, D=32, h=16, w=16)


def test_more_than_256_classes_is_refused_on_emulation(emu):
    M.test_more_than_256_classes_is_refused()
