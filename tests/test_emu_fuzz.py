"""Bounded differential fuzzing of the real SIMT kernel sources (host-fiber emulation, tests/emu) against the oracle:
random geometries per component, fixed seeds.  `python tools/emu_fuzz.py` runs the same fuzzers for as long as wanted."""
import random

import pytest
import torch

import emu_fuzz
import emu_harness
import test_gpu_parity as G

NGRAPH = 24
NCRIT = 10
NHEAD = 10
HEAD_SEED = 24


@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return emu_harness.use_emulation(monkeypatch)


@pytest.fixture
def emu_fused(emu, monkeypatch):
    """The criterion's launch sequence run eagerly (no CUDA graphs on a CPU, the fill branch inline) and the fused seg
    CE taken for CPU tensors, as in test_emu_graphed_criterion.py."""
    from contrastiveseg_b200 import graph_step, loss as loss_mod
    G_ = graph_step.GraphedContrastStep
    monkeypatch.setattr(G_, "_capture", lambda self, warmup: None)
    monkeypatch.setattr(G_, "_fork_zero_fill", lambda self: self._side_branch(0))
    monkeypatch.setattr(G_, "_join_zero_fill", lambda self: None)
    monkeypatch.setattr(loss_mod.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)
    return emu


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


def test_fuzz_graphed_criterion(emu_fused):
    """The captured criterion's launch sequence (run eagerly) with labels, heads and embed refilled between replays:
    every wrapper x seg term, CE path, dtype, degenerate replay and grad_scale change reached on scored replays."""
    bad, cov = emu_fuzz.fuzz_graphed_criterion(seed=21, n=NCRIT, check_sampling=G._check_device_sampling)
    assert bad == []
    assert all(cov[k] >= 1 for k in emu_fuzz.CRIT_CATEGORIES), cov
    assert cov["scored"] >= 2 * cov["skipped"], cov


def test_criterion_fuzz_detects_a_stale_label_map(emu_fused, monkeypatch):
    """Negative control: seg terms that read a copy of the label map taken when the criterion was built (labels that
    stop changing between replays) fail the fuzzer on a replay after the first, in most cases."""
    from contrastiveseg_b200 import graph_criterion
    init = graph_criterion._Term.__init__

    def stale(self, lib, term, x, target, grad_scale):
        init(self, lib, term, x, target.clone(), grad_scale)
    monkeypatch.setattr(graph_criterion._Term, "__init__", stale)
    bad, _ = emu_fuzz.fuzz_graphed_criterion(seed=21, n=6, check_sampling=G._check_device_sampling)
    assert len(bad) >= 4, bad
    assert not any(b.startswith("replay 0:") or "replay 0: " in b for b in bad), bad


def test_criterion_fuzz_regression_two_call_ce_every_pixel_ignored(emu_fused):
    """The criterion fuzzer's first finding, as a constructed case: case 3 of the fuzzer's draw (ContrastAuxCELoss with
    a label grid smaller than the logits: the two-call seg CE) from a fixed stream, with replay 3 forced to ignore every
    label.  Such a replay gave a NaN gradient in both heads (k_segce_bwd_gather: 0 times grad / 0); it is 0."""
    c, _ = emu_fuzz._draw_criterion_case(random.Random(3), 3, 1, "cpu")
    c.update(all_ignored=True, n_rep=4)
    cov = {k: 0 for k in emu_fuzz.CRIT_CATEGORIES + ("scored", "skipped", "refused")}
    assert c["name"] == "aux_ce" and c["mode"] == "down" and not c["refused"]
    assert emu_fuzz.graphed_criterion_case(c, "cpu", G._check_device_sampling, cov, "regression") == []
    assert cov["CE two-call"] == 1 and cov["all-ignored replay"] == 1, cov


def test_fuzz_projection_head(emu):
    """The fused projection head at every fusion level with the dense, column, loss and fallback backward, inputs and
    weights changed between replays, scored against float64 with a per-element bound: every category reached."""
    bad, cov = emu_fuzz.fuzz_projection_head(seed=HEAD_SEED, n=NHEAD)
    assert bad == []
    assert all(cov[k] >= 1 for k in emu_fuzz.HEAD_CATEGORIES), cov


def test_head_fuzz_detects_a_weight_packed_once(emu, monkeypatch):
    """Negative control: a head that packs the last conv's weight on its first call and reuses that pack (weights that
    stop changing between replays, as a pack captured once would) fails the fuzzer on a replay after the first."""
    from contrastiveseg_b200 import functional as Fn
    orig, packs = Fn._proj_pack, {}

    def packed_once(lib, x, weight, bias, s):
        out = orig(lib, x, weight, bias, s)
        key = (id(weight), weight.data_ptr(), tuple(weight.shape), tuple(x.shape))
        return (packs.setdefault(key, out[0]),) + out[1:]
    monkeypatch.setattr(Fn, "_proj_pack", packed_once)
    bad, _ = emu_fuzz.fuzz_projection_head(seed=HEAD_SEED, n=3)
    assert len(bad) >= 2, bad
    assert not any(b.startswith("replay 0 ") for b in bad), bad


@pytest.mark.parametrize("grad", ["cols", "loss"])
def test_head_fuzz_regression_column_path_at_width_one(emu, grad):
    """The head fuzzer's finding, as a constructed case: a feature map one pixel wide (W = 1).  expand() keeps the
    stride of a size-1 dimension, so the loss's zero placeholder failed _ColumnSink.is_placeholder's stride check and
    the head silently took the dense path.  head_case asserts that the column path ran, on every replay."""
    bad, cov = emu_fuzz.run_head_cases([emu_fuzz.width_one_case(grad)], "cpu")
    assert bad == [] and cov["column hand-off" if grad == "cols" else "contrast loss"] == 1, (bad, cov)


def test_head_fuzz_edge_cases(emu):
    """Constructed head cases: the column path past 256 channels with a clamped anchor just under eps, and bf16
    fallbacks whose deposits add to another gradient term."""
    bad, cov = emu_fuzz.run_head_cases(emu_fuzz.edge_cases(), "cpu", "edge")
    assert bad == [] and cov["clamped pixel"] == 1 and cov["fallback"] == 2, (bad, cov)
