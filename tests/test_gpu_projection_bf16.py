"""bf16 activations through the fused projection head (csrc/pcl_norm.cu k_proj_* <__nv_bfloat16>, pcl_proj_fwd_dt /
pcl_proj_bwd_dt, functional.project_normalize, ProjectionHead(fused=True) under autocast).  Contract: the kernels
take bf16 x as the bf16 GEMM operand it already is, convert zn and gzn on load (exact) and compute in fp32 exactly as
for fp32 activations, so against the fp32 call on the
converted inputs zn and gx are that call's values rounded once to nearest-even, and inv_norm, gW and gb are
bit-identical.  Helpers and bounds come from test_gpu_projection.py; test_emu_projection_bf16.py runs these functions
at small shapes on the emulated kernels (DEV = "cpu")."""
import pytest
import torch

import contrastiveseg_b200 as cs
import test_gpu_projection as P
from contrastiveseg_b200 import _abi, functional as Fn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16

# Against float64 on the bf16 x values with the fp32 weight (the fp32-operand reference of test_gpu_projection.py).
# bf16-path bounds, >= 3x the worst error measured over P.SHAPES on an H100 80GB HBM3 (DESIGN §2), capped by the
# fp32-operand bounds.  Worst measured max-abs / Frobenius: zn 3.66e-3 / 2.35e-3, gx 3.97e-3 / 2.89e-3, gW 1.66e-3 /
# 1.69e-3, gb 1.70e-3 / 1.75e-3.  zn and gx are rounded to bf16 on output (half an ulp, 2^-9 relative, on top of the
# operand rounding), so for them and for gb 3x would exceed the fp32-operand bounds, which stay in force; gW tightens
# (5.5e-3 = 3.3x its worst max-abs, 3.25x its worst Frobenius).
BF16_PATH_MAXABS = {"zn": 8e-3, "gx": 8e-3, "gw": 5.5e-3, "gb": 5e-3}
BF16_PATH_FROB = {"zn": 7.5e-3, "gx": 7.5e-3, "gw": 5.5e-3, "gb": 5.5e-3}


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


def _inputs(shape, seed=0):
    x, w, b, gzn = P._inputs(shape, seed)
    return x.to(BF), w, b, gzn.to(BF)


def _abi_pass(x, w, b, gzn, zn=None, inv=None):
    """pcl_proj_pack + forward + backward through the C ABI.  fp32 x takes pcl_proj_fwd / pcl_proj_bwd, bf16 x the _dt
    entry points.  zn / inv given: the backward runs on them instead of the forward's."""
    lib = _abi.load()
    B, Cin, H, W = x.shape
    HW = H * W
    dev, dt = x.device, Fn.proj_dtype_code(x.dtype)
    wpack = torch.empty(lib.pcl_proj_workspace_bytes(B, Cin, HW, 0), dtype=torch.uint8, device=dev)
    scratch = torch.empty(lib.pcl_proj_workspace_bytes(B, Cin, HW, 1), dtype=torch.uint8, device=dev)
    zf = torch.empty((B, 256, H, W), dtype=x.dtype, device=dev)
    invf = torch.empty(B * HW, dtype=torch.float32, device=dev)
    gx = torch.empty_like(x)
    gw = torch.empty((256, Cin), dtype=torch.float32, device=dev)
    gb = torch.empty(256, dtype=torch.float32, device=dev)
    w2 = w.reshape(256, Cin).contiguous()
    s = Fn._stream_ptr(dev)
    with Fn._on_device(dev):
        _abi.check(lib.pcl_proj_pack(w2.data_ptr(), Cin, wpack.data_ptr(), s))
        if dt == _abi.DT_F32:
            _abi.check(lib.pcl_proj_fwd(x.data_ptr(), wpack.data_ptr(), b.data_ptr(), B, Cin, HW, zf.data_ptr(),
                                        invf.data_ptr(), s))
        else:
            _abi.check(lib.pcl_proj_fwd_dt(x.data_ptr(), dt, wpack.data_ptr(), b.data_ptr(), B, Cin, HW, zf.data_ptr(),
                                           invf.data_ptr(), s))
        zb, ib = (zf, invf) if zn is None else (zn, inv)
        if dt == _abi.DT_F32:
            _abi.check(lib.pcl_proj_bwd(x.data_ptr(), zb.data_ptr(), ib.data_ptr(), gzn.data_ptr(), wpack.data_ptr(), B,
                                        Cin, HW, scratch.data_ptr(), gx.data_ptr(), gw.data_ptr(), gb.data_ptr(), s))
        else:
            _abi.check(lib.pcl_proj_bwd_dt(x.data_ptr(), dt, zb.data_ptr(), ib.data_ptr(), gzn.data_ptr(),
                                           wpack.data_ptr(), B, Cin, HW, scratch.data_ptr(), gx.data_ptr(),
                                           gw.data_ptr(), gb.data_ptr(), s))
    _sync()
    return {"zn": zf, "inv": invf, "gx": gx, "gw": gw, "gb": gb}


def measure(shape):
    """{name: (max-abs / max|ref|, rel Frobenius, max-abs)} of the bf16 path against float64 on the bf16 x values."""
    x, w, b, gzn = _inputs(shape)
    got = P._fused(x, w, b, gzn)
    return P.errors(got, P._reference(x.float(), w, b, gzn.float(), False))


@pytest.mark.parametrize("shape", P.SHAPES)
def test_forward_is_the_fp32_forward_rounded(shape):
    x, w, b, gzn = _inputs(shape)
    h, f = _abi_pass(x, w, b, gzn), _abi_pass(x.float(), w, b, gzn.float())
    assert h["zn"].dtype == BF and torch.equal(h["zn"], f["zn"].to(BF))
    assert torch.equal(h["inv"], f["inv"])
    got = P._fused(x, w, b, gzn)                                    # the public path makes the same calls
    assert got["zn"].dtype == BF and torch.equal(got["zn"], h["zn"])


@pytest.mark.parametrize("shape", P.SHAPES)
def test_backward_is_the_fp32_backward_on_the_converted_inputs(shape):
    x, w, b, gzn = _inputs(shape)
    h = _abi_pass(x, w, b, gzn)
    f = _abi_pass(x.float(), w, b, gzn.float(), zn=h["zn"].float(), inv=h["inv"])
    assert torch.equal(h["gw"], f["gw"]) and torch.equal(h["gb"], f["gb"])
    assert h["gx"].dtype == BF and torch.equal(h["gx"], f["gx"].to(BF))
    got = P._fused(x, w, b, gzn)
    assert got["gx"].dtype == BF and torch.equal(got["gx"], h["gx"])
    assert torch.equal(got["gw"], h["gw"].view_as(w)) and torch.equal(got["gb"], h["gb"])


@pytest.mark.parametrize("shape", P.SHAPES)
def test_matches_fp64_on_bf16_activations(shape):
    e = measure(shape)
    for k in P.FP32_REF_MAXABS:
        assert e[k][0] <= P.FP32_REF_MAXABS[k] and e[k][1] <= P.FP32_REF_FROB[k], (k, e)
        assert e[k][0] <= BF16_PATH_MAXABS[k] and e[k][1] <= BF16_PATH_FROB[k], (k, e)


def test_clamped_pixel_matches_f_normalize():
    """An all-zero pixel column with zero bias: zn exactly 0 there and gz = gzn / eps (F.normalize's clamp); gx there is
    the float64 value to within the final bf16 rounding."""
    x, w, _, gzn = _inputs((2, 100, 5, 7), seed=3)
    x[1, :, 2, 3] = 0.
    b = torch.zeros(256, device=x.device)
    got = P._fused(x, w, b, gzn)
    ref = P._reference(x.float(), w, b, gzn.float(), True)
    assert got["zn"][1, :, 2, 3].abs().max().item() == 0.
    g, r = got["gx"][1, :, 2, 3].double(), ref["gx"][1, :, 2, 3]
    assert r.abs().max().item() > 1e9                                     # the clamped branch: gzn * 1e12
    assert (g - r).abs().max().item() <= 2 ** -8 * r.abs().max().item()
    # the clamped pixel's 1e12-sized gz dominates gb; gW gets nothing from it (x = 0 there)
    assert (got["gb"].double() - ref["gb"]).abs().max().item() <= 1e-5 * ref["gb"].abs().max().item()
    e = P.errors(got, P._reference(x.float(), w, b, gzn.float(), False))
    for k in ("zn", "gw"):
        assert e[k][0] <= BF16_PATH_MAXABS[k] and e[k][1] <= BF16_PATH_FROB[k], (k, e)


@pytest.mark.parametrize("shape", [(2, 2048, 66, 66), (3, 100, 5, 7)])
def test_bit_reproducible(shape):
    x, w, b, gzn = _inputs(shape, seed=5)
    a, c = P._fused(x, w, b, gzn), P._fused(x, w, b, gzn)
    for k in ("zn", "gx", "gw", "gb"):
        assert torch.equal(a[k], c[k]), k


def test_cuda_graph_replay_is_bit_identical_to_eager():
    x, w, b, gzn = _inputs((2, 720, 33, 40), seed=7)
    eager = P._fused(x, w, b, gzn)
    xx, ww, bb = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                             # warm-up outside the capture
        for _ in range(2):
            cs.project_normalize(xx, ww, bb).backward(gzn)
            xx.grad = ww.grad = bb.grad = None
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        zn = cs.project_normalize(xx, ww, bb)
        zn.backward(gzn)
    for _ in range(2):
        xx.grad.zero_(); ww.grad.zero_(); bb.grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
        got = {"zn": zn.detach(), "gx": xx.grad, "gw": ww.grad, "gb": bb.grad}
        for k in ("zn", "gx", "gw", "gb"):
            assert torch.equal(got[k], eager[k]), k


def _autocast():
    return torch.autocast(str(DEV).split(":")[0], dtype=BF)


@pytest.mark.parametrize("proj,xdtype", [("convmlp", torch.float32), ("linear", BF)])
def test_fused_head_under_autocast_matches_the_unfused_head(proj, xdtype, shape=(2, 96, 12, 20)):
    ref, fused = P._heads(proj, shape[1])
    assert list(fused.state_dict().keys()) == list(ref.state_dict().keys())
    x = torch.randn(shape, generator=torch.Generator().manual_seed(12)).to(device=DEV, dtype=xdtype)
    xr, xf = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    with _autocast():
        yr, yf = ref(xr), fused(xf)
    assert yf.dtype == BF                                                 # the last conv's input is bf16 in both cases
    gy = torch.randn(yr.shape, generator=torch.Generator().manual_seed(13)).to(DEV)
    yr.backward(gy.to(yr.dtype))
    yf.backward(gy.to(yf.dtype))
    assert xf.grad.dtype == xdtype and xr.grad.dtype == xdtype
    pairs = [("zn", yf.detach(), yr.detach()), ("gx", xf.grad, xr.grad)]
    pairs += [(n, pf.grad, pr.grad) for (n, pf), (_, pr) in zip(fused.named_parameters(), ref.named_parameters())]
    # both heads round to bf16 at different points (the unfused one rounds the raw projection and the gradient reaching
    # the conv, the fused one zn and gx), each within the FP32_REF bounds of the exact value: their difference is
    # bounded by twice those bounds (the linear head's zn measured at 1.0x the single max-abs bound on an H100)
    for name, a, r in pairs:
        d = a.double() - r.double()
        assert d.abs().max().item() <= 2 * P.FP32_REF_MAXABS["gx"] * r.double().abs().max().item(), name
        assert d.norm().item() <= 2 * P.FP32_REF_FROB["gx"] * r.double().norm().item(), name


def stand_in_pair(B=2, Cin=64, h=16, w=16, K=5):
    """features -> (seg head, convmlp projection head) under autocast -> ContrastCELoss -> backward, with the unfused and
    the fused head on the same weights and the same device-RNG anchors (the seg logits, and so the sampled anchors, are
    identical).  Returns [(embed dtype, contrast term, x.grad)] for the unfused and the fused head.  The seg CE term is
    the same in both runs, so the contrast term (total minus the seg-only loss, over the loss weight) is where the head's
    difference shows."""
    ref, fused = P._heads("convmlp", Cin)
    torch.manual_seed(17)
    cls = torch.nn.Conv2d(Cin, K, 1).to(DEV)
    g = torch.Generator().manual_seed(18)
    feats = torch.randn(B, Cin, h, w, generator=g).to(DEV)
    tgt = torch.randint(0, K, (B, 4 * h, 4 * w), generator=g).to(DEV)
    cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": 4},
                       "loss": {"params": {"ce_ignore_index": -1}},
                       "contrast": {"temperature": 0.1, "base_temperature": 0.07, "max_samples": 128, "max_views": 8,
                                    "loss_weight": 0.1, "use_rmi": False, "use_lovasz": False}})
    out = []
    for head in (ref, fused):
        crit = cs.ContrastCELoss(cfg).to(DEV)
        x = feats.clone().requires_grad_(True)
        with _autocast():
            preds = {"seg": cls(x), "embed": head(x)}
            with torch.no_grad():
                seg_only = crit(preds, tgt, with_embed=False)
            Fn._step_counter[0] = 0                        # the same device-RNG draw for both heads
            loss = crit(preds, tgt, with_embed=True)
        loss.backward()
        _sync()
        contrast = (loss.detach().double() - seg_only.double()) / crit.loss_weight
        out.append((preds["embed"].dtype, contrast, x.grad.double()))
    return out


# relative difference of the contrast term, fused bf16 zn against the unfused head's fp32 zn: >= 3x the worst measured
# (1.65e-5 on an H100 80GB HBM3 at the default shape, 4.2e-5 on the emulated kernels at their small shape)
STAND_IN_CONTRAST_REL = 1.5e-4


def test_autocast_stand_in_iteration_matches_the_unfused_head(B=2, Cin=64, h=16, w=16, K=5):
    (er, cr, gr), (ef, cf, gf) = stand_in_pair(B, Cin, h, w, K)
    assert er == torch.float32 and ef == BF and torch.isfinite(cf) and cr.abs().item() > 0
    assert abs(cf.item() - cr.item()) <= STAND_IN_CONTRAST_REL * abs(cr.item()), (cf.item(), cr.item())
    assert (gf - gr).norm().item() <= P.FP32_REF_FROB["gx"] * gr.norm().item()


def test_refusals():
    head = cs.ProjectionHead(64, 256, "linear", fused=True).to(DEV)
    w, b = head.proj.weight, head.proj.bias
    for dt in (torch.float16, torch.float64):
        x = torch.randn(1, 64, 4, 4, device=DEV, dtype=dt)
        with pytest.raises(_abi.PclError):
            head(x)
        with pytest.raises(_abi.PclError):
            cs.project_normalize(x, w, b)
    mlp = cs.ProjectionHead(64, 256, "convmlp", bn_type="torchbn", fused=True).to(DEV)
    with pytest.raises(_abi.PclError):
        mlp(torch.randn(1, 64, 4, 4, device=DEV, dtype=torch.float16))
    if DEV != "cpu":
        with pytest.raises(_abi.PclError):
            head(torch.randn(1, 64, 4, 4, dtype=BF))
        with pytest.raises(_abi.PclError):
            cs.project_normalize(torch.randn(1, 64, 4, 4, dtype=BF), w, b)
    # the C ABI refuses fp16 and unknown codes
    lib = _abi.load()
    for code in (_abi.DT_F16, 7):
        assert lib.pcl_proj_fwd_dt(1, code, 1, None, 1, 64, 16, 1, 1, None) != 0
        assert lib.pcl_proj_bwd_dt(1, code, 1, 1, 1, 1, 1, 64, 16, 1, 1, 1, None, None) != 0
