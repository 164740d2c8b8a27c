"""Bounded differential fuzzing of the real SIMT kernel sources (host-fiber emulation, tests/emu) against the oracle:
random geometries per component, fixed seeds.  `python tools/emu_fuzz.py` runs the same fuzzers for as long as wanted."""
import pytest
import torch

import emu_fuzz
import emu_harness
import test_gpu_parity as G

NGRAPH = 24


@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return emu_harness.use_emulation(monkeypatch)


def test_fuzz_pixel_contrast_loss(emu):
    assert emu_fuzz.fuzz_loss(seed=11, n=40) == []


def test_fuzz_bank_enqueue(emu):
    assert emu_fuzz.fuzz_bank(seed=12, n=25) == []


def test_fuzz_fused_seg_ce(emu):
    assert emu_fuzz.fuzz_segce(seed=13, n=40) == []


def test_fuzz_device_sampling(emu):
    assert emu_fuzz.fuzz_device_sampling(seed=14, n=25, check_sampling=G._check_device_sampling) == []


def test_fuzz_topk(emu):
    assert emu_fuzz.fuzz_topk(seed=15, n=30) == []


def test_fuzz_tensor_path(emu):
    assert emu_fuzz.fuzz_tensor_path(seed=16, n=9) == []


def test_fuzz_graphed_step(emu):
    """The captured step's launch sequence (run eagerly): every path, bank and dtype reached, every replay scored."""
    bad, cov = emu_fuzz.fuzz_graphed_step(seed=17, n=NGRAPH, check_sampling=G._check_device_sampling)
    assert bad == []
    assert all(cov[k] >= 1 for k in emu_fuzz.GRAPH_CATEGORIES), cov


def test_fuzz_trainer_hook(emu):
    assert emu_fuzz.fuzz_trainer_hook(seed=18, n=10) == []


def test_trainer_hook_fuzz_detects_an_early_bank_write(emu, monkeypatch):
    """Negative control: with the bank write applied immediately (before the pending backward, the behaviour of the
    first GPU-verified build) the embedding gradient of the hook flow deviates from the reference by tens of percent."""
    from contrastiveseg_b200 import functional as Fn
    monkeypatch.setattr(Fn, "bank_reader", lambda *a: None)
    bad = emu_fuzz.fuzz_trainer_hook(seed=18, n=8)
    assert len(bad) >= 4 and all("d_embed" in b for b in bad)


def test_fuzz_loss_wrappers(emu):
    assert emu_fuzz.fuzz_wrappers(seed=19, n=30) == []
