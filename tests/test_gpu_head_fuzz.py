"""The fused projection head fuzzed on the device (tests/emu_fuzz.py: fuzz_projection_head): every fusion level, the
dense and the anchor-column backward, the real contrast loss and the fallbacks, with inputs and weights changed in place
between real CUDA-graph replays, each replay scored against float64 with a per-element bound (DESIGN §4).
test_emu_fuzz.py runs the same fuzzer on the emulated kernels."""
import gc

import pytest
import torch

import emu_fuzz

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def test_fuzz_projection_head_on_the_device():
    bad, cov = emu_fuzz.fuzz_projection_head(seed=31, n=36, device=DEV, scale=4)
    print("\nWORST error/bound: " + " ".join(f"{k} {v:.3g}" for k, v in sorted(cov["worst"].items())))
    assert bad == [], bad[:20]
    assert all(cov[k] >= 1 for k in emu_fuzz.HEAD_CATEGORIES), cov


@pytest.mark.parametrize("grad", ["dense", "cols"])
@pytest.mark.parametrize("level", ["bn_relu", "conv1"])
def test_fuzz_projection_head_at_the_s1_shape(level, grad):
    """bench.py's S1 head input (8 x 720 x 128 x 256), bf16, in training, 3 captured replays with inputs and weights
    changed between them; the column case hands over 1024 columns."""
    c = dict(level=level, grad=grad, adv=None, seed=77, act="bf16", train=True, sync=False, momentum=0.1,
             b1=level == "conv1", b2=True, x_grad=True, B=8, Cin=720, H=128, W=256, n_rep=3,
             actions=["both", "both"])
    if grad == "cols":
        c["n_cols"] = 1024
    bad, cov = emu_fuzz.run_head_cases([c], DEV, "S1")
    print(f"\nWORST error/bound S1 {level} {grad}: " +
          " ".join(f"{k} {v:.3g}" for k, v in sorted(cov["worst"].items())))
    assert bad == [], bad


@pytest.mark.parametrize("grad", ["cols", "loss"])
def test_head_fuzz_regression_column_path_at_width_one(grad):
    """The fuzzer's finding on the device: a feature map one pixel wide took the dense path (the zero placeholder's
    size-1 last dimension keeps stride 1 under expand()); the column path must run, captured for the hand-off."""
    bad, cov = emu_fuzz.run_head_cases([emu_fuzz.width_one_case(grad, Cin=257, B=3, H=65)], DEV)
    assert bad == [] and cov["column hand-off" if grad == "cols" else "contrast loss"] == 1, (bad, cov)


def test_head_fuzz_edge_cases():
    """The constructed cases of test_emu_fuzz.py on the device: the column path past 256 channels with a clamped anchor
    just under eps (captured), and bf16 fallbacks whose deposits add to another gradient term."""
    bad, cov = emu_fuzz.run_head_cases(emu_fuzz.edge_cases(), DEV, "edge")
    assert bad == [] and cov["clamped pixel"] == 1 and cov["fallback"] == 2, (bad, cov)
