"""The work splits that depend on the SM count, at shapes derived from the device's SM count, against float64.

Several kernels size their grids and partial-sum workspaces from pcl::num_sms():
  tensor-core InfoNCE (make_tc_plan, csrc/pcl_infonce_tc.cu)
    NEG walk     grid = min(pairs, SMs), pairs = row_tiles (128 anchors) x col_tiles (256 columns); partial slots
                 col_tiles / U + 2 (U = pairs / grid) with A known on the host, one per CTA with a device-side plan
    POS sweep    2-D grid of splits = SMs / row_tiles (at least 1, at most col_tiles); in bank mode up to 4096 anchors
                 the transposed sweep k_tc_pos_t instead: one CTA per SM dealt (64-anchor block, 128-column tile) units
    backward     splits_bwd = SMs / row_tiles over 64-column tiles (at least 1, at most their count)
  exact SIMT sweep (csrc/pcl_infonce_simt.cu): splits = 2 SMs / row_tiles (64 anchors), capped by the 64-column tiles
                 and by the SM count
  projection-head weight gradient (layout(), csrc/pcl_norm.cu): splits = SMs / (2 ctiles), ctiles = ceil((Cin + 1) / 256)
                 (the bias is column Cin), capped by the 64-pixel blocks B ceil(HW / 64)

Every shape below is derived from the SM count (here: the device's; tests/test_emu_sm_counts.py runs the same functions on
the CPU emulator built for 7, 114 and 132 SMs), and each tensor-path case first checks with pcl_tc_sizes that the plan
is the one the case is named after.  Regimes and the plans they get on a 132-SM H100 SXM (recompute with pcl_tc_sizes,
pcl_sweep_sizes, pcl_proj_workspace_bytes, or with tc_plan / simt_splits / wgrad_splits below):

  regime             mode        shape at 132 SMs              plan at 132 SMs
  pairs_below        self        A = 2048                      16 x 8 = 128 pairs = grid, slots 8, splits 8
                     explicit    A = 91, N = 33459 (bank 33496)  1 x 131 = 131 pairs = grid, slots 131, splits 131,
                                                               splits_bwd 132
  pairs_at           self        A = 2049                      17 x 9 = 153 pairs, grid 132, slots 9, splits 7
                     explicit    A = 1499, N = 2739 (2776)     12 x 11 = 132 pairs = grid, slots 11, splits 11
  pairs_above        self        A = 2177                      18 x 9 = 162 pairs, grid 132, slots 9, splits 7
                     explicit    A = 859, N = 4787 (4824)      7 x 19 = 133 pairs, grid 132, slots 19, splits 18
  pairs_3x           self        A = 3585                      29 x 15 = 435 pairs, grid 132 (U 3), slots 7, splits 4
                     explicit    A = 1627, N = 7859 (7896)     13 x 31 = 403 pairs, grid 132 (U 3), slots 12, splits 10
  rows_over_sms      unsorted    A = 16901, N = 700            133 x 3 pairs, slots 3, splits 1, splits_bwd 1
                     bank        A = 16901, M = 1691           133 x 53 pairs, splits 1, splits_bwd 1, row-tile POS sweep
  bwd_two            sorted      A = 8411, N = 300             66 x 2 pairs, splits 2, splits_bwd 2
  cols_cap           explicit    A = 100, N = 700 (728)        1 x 3 pairs, splits 3 (column tiles), splits_bwd 11 (12)
  device plan        self        max_samples 2304: 18 x 9 = 162 pairs, grid 132; live A 2040: 16 x 8 = 128 pairs
                                 (one case: the pair-count regimes above run with A known on the host only)
  k_tc_pos_t units   bank        131 / 132 / 133 / 267 (block, tile) units on 132 CTAs: U = 1, 1, 2, 3 units per CTA
                                 (131 / 132 / 67 / 89 CTAs busy), one 128-column tile per class, POS splits >= 10
  POS sweep switch   bank        A = 4095, 4096 (k_tc_pos_t), 4097, 4224 (row-tile POS sweep), 3 classes, M = 704
  SIMT splits        explicit    1 (A = 16897, N = 130), 2 (A = 8448, N = 200), column-tile cap 5 (A = 50, N = 320),
                                 SM cap 132 (A = 50, N = 16896)
  projection wgrad               Cin 8 / 255: ctiles 1, SMs / (2 ctiles) = 66; 256 / 257: ctiles 2, 33; 512: ctiles
                                 3, 22; B = 2 with HW 1..129 has 2..6 pixel blocks, so splits = the pixel blocks
  conv1                          C = 256: one 256-row band of gW1; C = 257: a second band of one row
(explicit: sorted and unsorted contrast sets, and the bank with K = 5, whose column count is given in brackets.)

Bounds: the tensor path uses the bounds of emu_fuzz.fuzz_tensor_path (loss 5e-5 relative, gradient max-abs 6e-3 and
relative Frobenius 5e-3), the SIMT sweep those of test_gpu_parity (loss 2e-6 relative, gradient 1e-5 max-abs), the
projection head those of test_gpu_projection*.py, the device-plan step those of test_gpu_many_classes."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
import emu_fuzz
import test_gpu_many_classes as MC
import test_gpu_parity as G
import test_gpu_projection as PP
import test_gpu_projection_bf16 as PF
import test_gpu_projection_bnrelu as PB
import test_gpu_projection_conv1 as PC
from contrastiveseg_b200 import _abi, functional as Fn
from oracle import ref_port as P

DEV = "cuda:0"
BF = torch.bfloat16
BM, BN, BNB = 128, 256, 64                   # tensor path: anchors per row tile, columns per tile, backward column tile
PT_NB, PT_BM, PT_MAX_ROWS = 64, 128, 4096    # k_tc_pos_t: anchors per block, bank columns per tile, largest anchor set
TM = 64                                      # SIMT sweep tile (rows and columns)


def cdiv(a, b):
    return -(-a // b)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------------
# plan arithmetic (make_tc_plan, simt_make_args, layout()) and the shapes derived from it
# ------------------------------------------------------------------------------------------------------------------
def tc_plan(sms, a_rows, n_cols, device_plan=False):
    rt, ct = cdiv(a_rows, BM), cdiv(max(n_cols, 1), BN)
    splits = min(max(1, sms // rt), ct)
    pairs = rt * ct
    grid = min(pairs, sms)
    slots_neg = grid if device_plan else ct // (pairs // grid) + 2
    slots_neg = max(1, min(slots_neg, grid, ct))
    return dict(row_tiles=rt, col_tiles=ct, pairs=pairs, grid=grid, splits=splits, slots=max(slots_neg, splits),
                splits_bwd=min(max(1, sms // rt), cdiv(max(n_cols, 1), BNB)))


def check_tc_plan(sms, mode, A, n_cols, bank_K=0, bank_R=0):
    """pcl_tc_sizes of the loaded library agrees with tc_plan: the case reaches the plan it is named after."""
    lib = _abi.load()
    d = _abi.TcDesc()
    d.a_rows, d.D, d.mode, d.n_cols = A, 256, {"self": 0, "bank": 1}.get(mode, 2), n_cols
    d.bank_K, d.bank_R, d.temperature, d.base_temperature = bank_K, bank_R, 0.1, 0.07
    ss = _abi.SweepSizes()
    _abi.check(lib.pcl_tc_sizes(C.byref(d), C.byref(ss)), "pcl_tc_sizes")
    p = tc_plan(sms, A, n_cols)
    assert (ss.row_tiles, ss.splits) == (p["row_tiles"], p["slots"]), (ss.row_tiles, ss.splits, p)
    assert ss.dpartial_f32 == p["splits_bwd"] * p["row_tiles"] * BM * 256, p
    return p


def _divisor(P, lo, hi):
    return max([r for r in range(lo, hi + 1) if P % r == 0], default=None)


def pair_shape(sms, regime, bank=False):
    """(row tiles, column tiles) of an explicit contrast set: pairs = SMs - 1, SMs, SMs + 1, or about 3 SMs + 7 with
    several row tiles (CTA ranges cross row tiles).  As many row tiles (up to 16) as divide the pair count; against
    the bank (10 M = 10 (32 c - 5) columns with K = 5) no more anchors than columns."""
    ok = (lambda r, c: 128 * r - 37 <= 10 * (32 * c - 5)) if bank else (lambda r, c: True)     # noqa: E731
    lo = 4 if regime == "pairs_3x" else 1
    P0 = {"pairs_below": sms - 1, "pairs_at": sms, "pairs_above": sms + 1, "pairs_3x": 3 * sms + 7}[regime]
    for P in range(P0, P0 + 1 if lo == 1 else 4 * sms + 8):
        rs = [r for r in range(lo, 17) if P % r == 0 and ok(r, P // r)]
        if rs:
            return max(rs), P // max(rs)
    raise AssertionError(f"no shape for {regime} at {sms} SMs")


def self_anchor_count(sms, regime):
    """Self-contrast: A with pairs (ceil(A / 128) x ceil(A / 256)) just below, at or past, just above SMs, or past 3 SMs."""
    pairs = lambda A: cdiv(A, BM) * cdiv(A, BN)          # noqa: E731
    As = range(1, 128 * 4 * sms)
    if regime == "pairs_below":
        return max(A for A in As if pairs(A) < sms)
    at = min(A for A in As if pairs(A) >= sms)
    if regime == "pairs_at":
        return at
    if regime == "pairs_above":
        return min(A for A in As if pairs(A) > pairs(at))
    return min(A for A in As if pairs(A) >= 3 * sms + 7)


def tensor_shape(sms, regime, mode):
    """(A, N, bank M) of a named regime; N is the column count (bank: (K - 1) 2 M with K = 5)."""
    if regime.startswith("pairs") and mode == "self":
        A = self_anchor_count(sms, regime)
        return A, A, None
    if regime.startswith("pairs"):
        r, c = pair_shape(sms, regime, bank=(mode == "bank"))
        A = 128 * r - 37
    elif regime == "rows_over_sms":                 # row tiles >= SMs: splits = splits_bwd = 1, 3 column tiles
        A, c = 128 * sms + 5, 3
    elif regime == "bwd_two":                       # SMs / row tiles = 2: splits_bwd = 2
        A, c = 128 * (sms // 2) - 37, 2
    else:                                           # cols_cap: one row tile, splits capped by the 3 column tiles
        A, c = 100, 3
    if mode == "bank":          # K = 5: 4 classes of 2 M columns, ceil(8 M / 256) = c tiles (more if A needs the columns)
        M = max(32 * c - 5, cdiv(A, 10))
        return A, 8 * M, M
    return A, {"rows_over_sms": 700, "bwd_two": 300, "cols_cap": 700}.get(regime, 256 * c - 77), None


def simt_splits(sms, A, N):
    return min(max(1, 2 * sms // cdiv(A, TM)), cdiv(N, TM), sms)


def simt_shape(sms, regime):
    """(A, N) of the exact SIMT sweep with splits = 1, 2, capped by the column tiles, capped by the SM count."""
    return {"one": (TM * 2 * sms + 1, 130), "two": (TM * sms, 200), "cols_cap": (50, 320),
            "sms_cap": (50, TM * 2 * sms)}[regime]


def wgrad_splits(sms, B, Cin, HW):
    return max(1, min(sms // (2 * cdiv(Cin + 1, 256)), B * cdiv(HW, 64)))


# ------------------------------------------------------------------------------------------------------------------
# tensor path, explicit calls (A known on the host)
# ------------------------------------------------------------------------------------------------------------------
TC_REGIMES = ([(r, m) for r in ("pairs_below", "pairs_at", "pairs_above", "pairs_3x")
               for m in ("self", "sorted", "unsorted", "bank")] +
              [("rows_over_sms", "unsorted"), ("rows_over_sms", "bank"), ("bwd_two", "sorted"), ("cols_cap", "unsorted"),
               ("cols_cap", "bank")])


def check_tensor_regime(sms, regime, mode, seed=0):
    A, N, M = tensor_shape(sms, regime, mode)
    p = check_tc_plan(sms, mode, A, N, *((5, 2 * M) if mode == "bank" else ()))
    if regime == "pairs_below":
        assert p["pairs"] == p["grid"] < sms
    elif regime in ("pairs_at", "pairs_above", "pairs_3x"):
        assert p["grid"] == sms and p["pairs"] >= sms
    elif regime == "rows_over_sms":
        assert p["splits"] == 1 and p["splits_bwd"] == 1
    elif regime == "bwd_two":
        assert p["splits_bwd"] == 2
    else:
        assert p["splits"] == p["col_tiles"] < sms // p["row_tiles"]
    g = torch.Generator().manual_seed(1000 * seed + sms)
    ref_dev = DEV if DEV != "cpu" and A * N > 2 ** 24 else "cpu"      # large closed forms in float64 on the GPU
    why = emu_fuzz.tensor_case(A, N, 5 if mode == "bank" else 19, 0.1, mode, 0.5, g, M=M, device=DEV, ref_device=ref_dev)
    assert why is None, f"{why}: {regime} {mode} A={A} N={N} M={M} plan={p}"


@pytest.mark.gpu
@pytest.mark.parametrize("regime,mode", TC_REGIMES)
def test_tensor_path_work_split(sms, regime, mode):
    check_tensor_regime(sms, regime, mode)


# ------------------------------------------------------------------------------------------------------------------
# tensor path through the step: device-side plan with fewer live pairs than the grid sized for max_samples
# ------------------------------------------------------------------------------------------------------------------
def device_plan_shape(sms, K=20, second=10):
    """max_samples with a NEG grid of min(pairs, SMs) CTAs, and max_views such that the live anchors (K + second
    (image, class) pairs x V) have fewer pairs than that grid."""
    ms = next(m for m in range(256, 256 * 64, 256) if cdiv(m, BM) * cdiv(m, BN) >= sms)
    grid = min(cdiv(ms, BM) * cdiv(ms, BN), sms)
    TC = K + second
    mv = max(v for v in range(1, ms // TC + 1) if cdiv(TC * v, BM) * cdiv(TC * v, BN) < grid)
    return ms, mv, grid


def check_device_plan(sms, K=20, second=10, h=64, w=64):
    ms, mv, grid = device_plan_shape(sms, K, second)
    embed, lab, seg = MC._two_image_batch(K, second, h, w, 256, seed=sms)
    crit = cs.PixelContrastLoss(G._cfg(0.1, 0.07, ms, mv, K, {"precision": "bf16"}))
    e = embed.to(DEV).requires_grad_(True)
    loss = crit(e, lab.to(DEV), seg=seg.to(DEV))
    ws = Fn.last_workspace(e.device)
    loss.backward()
    A, pix, img, cls, cf = MC._drawn_anchor_oracle(ws, e, ms)
    assert A < ms
    assert cdiv(A, BM) * cdiv(A, BN) < grid, (A, grid)
    MC._check_tensor_or_exact("bf16", loss.item(), e.grad, pix, img, cf)


@pytest.mark.gpu
def test_device_plan_with_fewer_live_pairs_than_ctas(sms):
    check_device_plan(sms)


# ------------------------------------------------------------------------------------------------------------------
# bank mode POS sweeps: k_tc_pos_t's units around the CTA count, and both sides of its 4096-anchor limit
# ------------------------------------------------------------------------------------------------------------------
def bank_case(counts, K, M, seed=0, T=0.1):
    """Bank mode with counts[k] anchors of class rank k (classes 1..K-1, then 0), against the float64 closed form."""
    from contrastiveseg_b200.bank import shadow_rows
    lib = _abi.load()
    g = torch.Generator().manual_seed(seed)
    ya = torch.cat([torch.full((n,), (k + 1) % K, dtype=torch.long) for k, n in enumerate(counts)])
    A = ya.numel()
    centers = F.normalize(torch.randn(K, 256, generator=g), dim=1)
    a = F.normalize(torch.randn(A, 256, generator=g) + 8 * centers[ya], dim=1)
    segq = F.normalize(torch.randn(K, M, 256, generator=g) + 8 * centers[:, None], dim=2)
    pixq = F.normalize(torch.randn(K, M, 256, generator=g) + 8 * centers[:, None], dim=2)
    shadow = torch.empty((shadow_rows(K, M), 256), dtype=BF, device=DEV)
    segq_d, pixq_d = segq.to(DEV), pixq.to(DEV)
    _abi.check(lib.pcl_bank_shadow_rebuild(segq_d.data_ptr(), pixq_d.data_ptr(), K, M, 256, shadow.data_ptr(), None))
    loss, st, state = Fn.infonce_tc_forward(a.to(DEV), ya.to(DEV), bank=(shadow, K, 2 * M),
                                            diag_col=torch.arange(A).to(DEV), temperature=T, base_temperature=0.07)
    dA = Fn.infonce_tc_backward(state, st).double().cpu()
    contrast, yc = P.flatten_queue(torch.cat((emu_fuzz._bf(segq), emu_fuzz._bf(pixq)), 1).double())
    cf = P.infonce_closed_form(emu_fuzz._bf(a).double(), ya, contrast, yc.long(), T, 0.07, self_contrast=False)
    assert torch.equal(st[4].double().cpu(), cf["npos"])
    assert abs(loss.item() - cf["loss"].item()) <= 5e-5 * abs(cf["loss"].item())
    gmax = cf["dA"].abs().max().item()
    assert (dA - cf["dA"]).abs().max().item() <= 6e-3 * gmax
    assert ((dA - cf["dA"]).norm() / cf["dA"].norm()).item() <= 5e-3


POS_T_UNITS = {"below": lambda s: s - 1, "at": lambda s: s, "above": lambda s: s + 1, "twice": lambda s: 2 * s + 3}
POS_T_REGIMES = list(POS_T_UNITS)


def pos_t_layout(sms, regime):
    """Class counts (class ranks 1..K-1, then class 0) whose k_tc_pos_t work list has SMs - 1, SMs, SMs + 1 or 2 SMs + 3
    (block, tile) units, with the CTA count setting the units per CTA.  Each class with columns owns one 128-column
    tile (M = 64, R = 128), so the largest per-block tile count is 1 and the slot floor u_slots is 1 whenever the POS
    sweep has 2 or more splits: U = ceil(units / SMs).  One block per class (1-3 anchors), two for the first classes
    when the units outnumber the 250 classes used; 9 anchors of class 0 (no columns, the analytic zero tail)."""
    units = POS_T_UNITS[regime](sms)
    n_c = min(units, 250)
    base, extra = divmod(units, n_c)
    counts = [PT_NB * (base + (k < extra) - 1) + 1 + k % 3 for k in range(n_c)] + [9]
    return units, counts


def check_pos_t_units(sms, regime):
    units, counts = pos_t_layout(sms, regime)
    K, M, A = len(counts), PT_BM // 2, sum(counts)
    assert A <= PT_MAX_ROWS and K <= 256
    splits = tc_plan(sms, A, (K - 1) * 2 * M)["splits"]
    u_slots = 1 if splits >= 2 else units                # (tmax + splits - 2) / (splits - 1) with tmax = 1
    U = max(cdiv(units, sms), u_slots)
    assert U == cdiv(units, sms), (units, splits, u_slots)     # the CTA count, not the slot floor, sets U
    if regime in ("above", "twice"):
        assert units % sms            # SMs x floor(units / SMs) units would leave some undealt
    bank_case(counts, K, M, seed=sms)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", POS_T_REGIMES)
def test_bank_pos_sweep_units_around_the_cta_count(sms, regime):
    check_pos_t_units(sms, regime)


@pytest.mark.gpu
@pytest.mark.parametrize("A", [4095, 4096, 4097, 4224])
def test_bank_pos_sweep_on_both_sides_of_the_anchor_limit(A):
    """k_tc_pos_t up to 4096 anchors, the row-tile POS sweep from 4097 on: three classes (two with bank columns, each
    11 column tiles of 128 and about 22 blocks of 64 anchors), class 0 included."""
    counts = [A // 2 - 100, A - (A // 2 - 100) - 200, 200]
    bank_case(counts, 3, 704, seed=A)


# ------------------------------------------------------------------------------------------------------------------
# exact SIMT sweep
# ------------------------------------------------------------------------------------------------------------------
SIMT_REGIMES = ["one", "two", "cols_cap", "sms_cap"]


def check_simt_regime(sms, regime, D=64):
    A, N = simt_shape(sms, regime)
    expect = {"one": 1, "two": 2, "cols_cap": cdiv(N, TM), "sms_cap": sms}[regime]
    assert simt_splits(sms, A, N) == expect
    lib = _abi.load()
    d = _abi.SweepDesc()
    d.a_rows, d.D, d.mode, d.n_cols, d.temperature, d.base_temperature = A, D, 2, N, 0.1, 0.07
    ss = _abi.SweepSizes()
    _abi.check(lib.pcl_sweep_sizes(C.byref(d), C.byref(ss)), "pcl_sweep_sizes")
    assert ss.splits == expect, (ss.splits, expect)
    g = torch.Generator().manual_seed(sms + A)
    ya, yc = torch.randint(0, 7, (A,), generator=g), torch.randint(0, 7, (N,), generator=g)
    a = F.normalize(torch.randn(A, D, generator=g), dim=1)
    c = F.normalize(torch.randn(N, D, generator=g), dim=1)
    diag = torch.arange(A) % N
    loss, rs, st = Fn.infonce_forward(a.to(DEV), ya.to(DEV), contrast=c.to(DEV), contrast_cls=yc.to(DEV),
                                      diag_col=diag.to(DEV), temperature=0.1, base_temperature=0.07)
    dA = Fn.infonce_backward(st, rs).double().cpu()
    cf = P.infonce_closed_form(a.double(), ya, c.double(), yc, 0.1, 0.07, self_contrast=False, diag_cols=diag)
    assert emu_fuzz._rel(loss.item(), cf["loss"].item()) < 2e-6, (loss.item(), cf["loss"].item())
    assert (dA - cf["dA"]).abs().max().item() <= 1e-5 * cf["dA"].abs().max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", SIMT_REGIMES)
def test_simt_sweep_work_split(sms, regime):
    check_simt_regime(sms, regime)


# ------------------------------------------------------------------------------------------------------------------
# projection head: the weight gradient's bias tile and its pixel-block splits
# ------------------------------------------------------------------------------------------------------------------
PROJ_CIN = [8, 255, 256, 257, 512]
PROJ_HW = [1, 63, 64, 65, 129]
# The weight and bias gradients on bf16 operands sum B HW products per element: with a few hundred pixels, the rare g_z
# element whose fp32 and float64 values round to neighbouring bf16 values is a visible share of an element.  The worst
# over all 25 (Cin, HW) shapes of PROJ_CIN x PROJ_HW, measured on an H100 80GB HBM3 (132 SMs, 700 W): gw 8.7e-4 and
# gb 4.2e-4, both at (2, 255, 1, 65), above test_gpu_projection's 6e-4 and 4e-4 from images of thousands of pixels;
# the bounds are 3x those.
FEW_PIXELS_BF16 = {"gw": 2.6e-3, "gb": 1.3e-3}


def check_projection(B, Cin, HW, dtypes=(torch.float32, BF)):
    """project_normalize (fp32 and bf16 activations), bn_relu_project_normalize and conv_bn_relu_project_normalize on
    (B, Cin, 1, HW) against the float64 chains of test_gpu_projection*.py.  With one pixel per image and B = 2, training
    BatchNorm sees two values per channel: its output is +-1 whatever y is, the y-gradient is zero up to eps and what
    both sides compute is a rounding residue, so one pixel per image runs BatchNorm in eval mode only."""
    shape = (B, Cin, 1, HW)
    e = PP.measure(shape)["bf16"]
    assert e["zn"][2] <= PP.ZN_ABS_BF16, e
    for k, bound in dict(PP.BF16_REF_MAXABS, **FEW_PIXELS_BF16).items():
        assert e[k][0] <= bound, (k, e)
    PP.test_matches_fp64_on_fp32_operands(shape)
    PF.test_matches_fp64_on_bf16_activations(shape)
    for dtype in dtypes:
        for mode in ("train", "eval") if B * HW > 2 else ("eval",):
            PB.test_matches_fp64(shape, mode, dtype)
            PC.test_head_matches_fp64(shape, mode, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("HW", PROJ_HW)
@pytest.mark.parametrize("Cin", PROJ_CIN)
def test_projection_head_bias_tile_and_pixel_blocks(sms, Cin, HW):
    """Two images: B x ceil(HW / 64) <= 6 pixel blocks, fewer than the weight gradient's splits at every Cin here."""
    assert wgrad_splits(sms, 2, Cin, HW) == min(sms // (2 * cdiv(Cin + 1, 256)), 2 * cdiv(HW, 64))
    check_projection(2, Cin, HW)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("C", [256, 257])
def test_conv1_one_band_and_a_one_row_band(C, dtype):
    shape = (2, C, 5, 13)
    PC.test_conv1_matches_fp64_on_bf16_operands(shape, dtype)
    PC.test_conv1_sums_match_fp64_sums_of_the_stored_y(shape, dtype)


# ------------------------------------------------------------------------------------------------------------------
# the emulator's differential fuzzers on the device.  The tensor path at scale 8 (A <= 3360, N <= 12000: up to about
# 1270 (row tile, column tile) pairs) fills the grid several times over.  The loss and device-sampling fuzzers at
# scale 4 reach 640 and 800 anchors (10 and 13 SIMT row tiles): bounded by their float64 oracle on the host, they
# cover the SIMT splits of 2 SMs / 10 and more; splits of 1 and 2 are the explicit SIMT cases above.
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fuzz_tensor_path_on_the_device():
    assert emu_fuzz.fuzz_tensor_path(seed=16, n=24, device=DEV, scale=8) == []


@pytest.mark.gpu
def test_fuzz_pixel_contrast_loss_on_the_device():
    assert emu_fuzz.fuzz_loss(seed=11, n=30, device=DEV, scale=4) == []


@pytest.mark.gpu
def test_fuzz_topk_on_the_device():
    assert emu_fuzz.fuzz_topk(seed=15, n=30, device=DEV, scale=8) == []


@pytest.mark.gpu
def test_fuzz_device_sampling_on_the_device():
    assert emu_fuzz.fuzz_device_sampling(seed=14, n=25, check_sampling=G._check_device_sampling, device=DEV,
                                         scale=4) == []
