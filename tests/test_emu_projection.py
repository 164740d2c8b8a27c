"""CPU execution of the projection-head GEMMs of csrc/pcl_norm.cu (wgmma / TMA against the functional model of
tests/emu/shim/ptx_sm90.cuh): the tests of test_gpu_projection.py at small shapes with DEV = "cpu" — Cin not a multiple
of 64, several K-blocks, several 256-channel dgrad passes, pixel-tile tails, the bias column of the weight gradient in
its own column tile."""
import pytest
import torch

import emu_harness
import test_gpu_projection as P

SMALL = [(3, 100, 5, 7), (2, 130, 9, 11), (1, 300, 12, 13), (2, 256, 4, 9)]


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(P, "DEV", "cpu")
    return lib


@pytest.mark.parametrize("shape", SMALL)
def test_projection_matches_fp64_on_bf16_operands_on_emulation(emu, shape):
    P.test_matches_fp64_on_bf16_operands(shape)


@pytest.mark.parametrize("shape", SMALL[:2])
def test_projection_matches_fp64_on_fp32_operands_on_emulation(emu, shape):
    P.test_matches_fp64_on_fp32_operands(shape)


def test_projection_clamped_pixel_on_emulation(emu):
    P.test_clamped_pixel_matches_f_normalize()


def test_projection_weight_gradient_is_bit_reproducible_on_emulation(emu):
    P.test_weight_gradient_is_bit_reproducible((3, 100, 5, 7))


@pytest.mark.parametrize("proj", ["convmlp", "linear"])
def test_fused_projection_head_on_emulation(emu, proj):
    P.test_fused_head_matches_the_unfused_head(proj, shape=(2, 40, 6, 7))


def test_fused_projection_head_errors_on_emulation(emu):
    P.test_fused_head_refuses_what_it_does_not_implement()
