"""The SM-count-dependent work splits of test_gpu_sm_regimes.py on the CPU emulator built for other SM counts: 132
(H100 SXM), 114 (H100 PCIe) and 7 (odd, small).  The suite's other emulated tests model 6 SMs, where the persistent
grids are short: they never have fewer live pairs than CTAs at a large grid, a POS sweep split over more than 6
slots, or a projection weight gradient split more than 3 ways.  Each shape is derived from the SM count by the
functions of test_gpu_sm_regimes.py, which also check that the plan is the one the case is named after.

At 7 SMs every regime runs (the pairs_3x regime in two modes).  At 114 and 132 SMs a 128 x 256 tile costs the
emulator about 0.1 s, so the large counts run a selection: at 132 SMs two pair counts, the device plan with fewer live
pairs than CTAs, k_tc_pos_t with one unit more than CTAs, the projection weight gradient with more splits than pixel
blocks; the full matrix runs on the H100 (test_gpu_sm_regimes.py).  50 tests in 5.0 minutes on an 8-core CPU."""
import pytest
import torch

import emu_harness
import test_gpu_many_classes as MC
import test_gpu_parity as G
import test_gpu_projection as PP
import test_gpu_projection_bf16 as PF
import test_gpu_projection_bnrelu as PB
import test_gpu_projection_conv1 as PC
import test_gpu_sm_regimes as R

MODES = ("self", "sorted", "unsorted", "bank")
PAIRS = ("pairs_below", "pairs_at", "pairs_above")


def _emulate(monkeypatch, sms):
    lib = emu_harness.use_emulation(monkeypatch, sms=sms)
    for m in (G, MC, PP, PF, PB, PC, R):
        monkeypatch.setattr(m, "DEV", "cpu")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return lib


def _tensor_cases():
    cases = [(7, r, m) for r in PAIRS for m in MODES] + [(7, "pairs_3x", m) for m in ("sorted", "bank")]
    cases += [(7, r, m) for r, m in (("rows_over_sms", "unsorted"), ("bwd_two", "sorted"), ("cols_cap", "unsorted"),
                                     ("cols_cap", "bank"))]
    cases += [(132, "pairs_at", "bank"), (132, "pairs_above", "sorted")]
    cases += [(114, "cols_cap", "bank"), (132, "cols_cap", "unsorted")]
    return [pytest.param(*c, id=f"{c[0]}sm-{c[1]}-{c[2]}") for c in cases]


@pytest.mark.parametrize("sms,regime,mode", _tensor_cases())
def test_tensor_path_work_split_on_emulation(monkeypatch, sms, regime, mode):
    _emulate(monkeypatch, sms)
    R.check_tensor_regime(sms, regime, mode)


@pytest.mark.parametrize("sms", [7, 132])
def test_device_plan_with_fewer_live_pairs_than_ctas_on_emulation(monkeypatch, sms):
    _emulate(monkeypatch, sms)
    R.check_device_plan(sms)


@pytest.mark.parametrize("sms,regime", [(7, r) for r in R.POS_T_REGIMES] + [(132, "above")])
def test_bank_pos_sweep_units_around_the_cta_count_on_emulation(monkeypatch, sms, regime):
    _emulate(monkeypatch, sms)
    R.check_pos_t_units(sms, regime)


@pytest.mark.parametrize("sms,regime", [(7, r) for r in R.SIMT_REGIMES] + [(132, "two")] +
                         [(s, r) for s in (114, 132) for r in ("cols_cap", "sms_cap")])
def test_simt_sweep_work_split_on_emulation(monkeypatch, sms, regime):
    _emulate(monkeypatch, sms)
    R.check_simt_regime(sms, regime)


@pytest.mark.parametrize("sms", [7, 114, 132])
def test_fuzz_pixel_contrast_loss_on_emulation(monkeypatch, sms):
    _emulate(monkeypatch, sms)
    import emu_fuzz
    assert emu_fuzz.fuzz_loss(seed=21, n=8) == []


@pytest.mark.parametrize("sms,Cin", [(7, 255), (7, 256), (7, 257), (132, 255), (132, 256)])
def test_projection_head_bias_tile_on_emulation(monkeypatch, sms, Cin):
    """Two images of 65 pixels: 4 pixel blocks, fewer than the weight gradient's splits at 132 SMs (66 or 33)."""
    _emulate(monkeypatch, sms)
    R.check_projection(2, Cin, 65, dtypes=(torch.float32,))


@pytest.mark.parametrize("C", [256, 257])
@pytest.mark.parametrize("sms", [7, 132])
def test_conv1_one_band_and_a_one_row_band_on_emulation(monkeypatch, sms, C):
    _emulate(monkeypatch, sms)
    for dtype in (torch.float32, R.BF):
        PC.test_conv1_matches_fp64_on_bf16_operands((1, C, 5, 7), dtype)
        PC.test_conv1_sums_match_fp64_sums_of_the_stored_y((1, C, 5, 7), dtype)
