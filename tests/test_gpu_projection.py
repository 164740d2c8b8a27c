"""The projection head's last 1x1 conv + L2 normalise as one wgmma GEMM (csrc/pcl_norm.cu, functional.project_normalize,
ProjectionHead(fused=True)) against torch float64 F.conv2d + F.normalize (+ autograd) on the same weights — op for op
lib/models/modules/projection.py:17-24.  tests/test_emu_projection.py runs the same functions at small shapes on the
emulated kernels (DEV = "cpu")."""
import pytest
import torch
import torch.nn.functional as F

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi

DEV = "cuda:0"

# S1 (BASELINE configs[1] head input), DeepLab C4, an odd square image, Cin not a multiple of 64 with a tile tail
SHAPES = [(8, 720, 128, 256), (2, 2048, 66, 66), (1, 720, 97, 97), (3, 100, 5, 7)]

# Bounds relative to max|reference| (max-abs) and to ||reference|| (Frobenius), each >= 3x the worst error measured over
# SHAPES on an H100 80GB HBM3 (DESIGN §2 lists the measured values next to them).
# bf16-rounded x and W, gz rounded to bf16 where the kernel rounds it: what remains is the fp32 accumulation order and the
# rare gz element whose fp32 and fp64 values round to neighbouring bf16 values
ZN_ABS_BF16 = 2e-5
BF16_REF_MAXABS = {"gx": 3e-3, "gw": 6e-4, "gb": 4e-4}
# fp32 operands: dominated by the bf16 rounding of x, W and gz (relative Frobenius ~2.4e-3 on every output, above the
# tensor path's 2e-3 starting bound, so the bounds are set from measurement)
FP32_REF_MAXABS = {"zn": 8e-3, "gx": 8e-3, "gw": 9e-3, "gb": 5e-3}
FP32_REF_FROB = {"zn": 7.5e-3, "gx": 7.5e-3, "gw": 7.5e-3, "gb": 5.5e-3}

def _inputs(shape, seed=0):
    B, Cin, H, W = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    w = torch.randn(256, Cin, 1, 1, generator=g) / Cin ** 0.5
    b = 0.1 * torch.randn(256, generator=g)
    gzn = torch.randn(B, 256, H, W, generator=g)
    return x.to(DEV), w.to(DEV), b.to(DEV), gzn.to(DEV)


def _fused(x, w, b, gzn):
    xx, ww = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    bb = None if b is None else b.clone().requires_grad_(True)
    zn = cs.project_normalize(xx, ww, bb)
    zn.backward(gzn)
    return {"zn": zn.detach(), "gx": xx.grad, "gw": ww.grad, "gb": None if bb is None else bb.grad}


def _reference(x, w, b, gzn, round_bf16):
    """fp64 conv + normalise + autograd; round_bf16: x, W rounded to bf16 and gz rounded to bf16 before the GEMMs."""
    r = (lambda t: t.to(torch.bfloat16).double()) if round_bf16 else (lambda t: t.double())
    x64, w64 = r(x), r(w)
    z = F.conv2d(x64, w64, None if b is None else b.double()).requires_grad_(True)
    zn = F.normalize(z, p=2, dim=1)
    (gz,) = torch.autograd.grad(zn, z, gzn.double())
    if round_bf16:
        gz = gz.float().to(torch.bfloat16).double()
    B, Cin = x.shape[:2]
    gzf, xf, wf = gz.reshape(B, 256, -1), x64.reshape(B, Cin, -1), w64.reshape(256, Cin)
    return {"zn": zn.detach(), "gx": torch.einsum("bnp,nc->bcp", gzf, wf).reshape(x.shape),
            "gw": torch.einsum("bnp,bcp->nc", gzf, xf).reshape(w.shape), "gb": gz.sum((0, 2, 3))}


def errors(got, ref):
    out = {}
    for k, rv in ref.items():
        d = got[k].double() - rv
        out[k] = ((d.abs().max() / rv.abs().max()).item(), (d.norm() / rv.norm()).item(), d.abs().max().item())
    return out


def measure(shape):
    """{"bf16": {name: (max-abs / max|ref|, rel Frobenius, max-abs)}, "fp32": {...}} for one shape."""
    x, w, b, gzn = _inputs(shape)
    got = _fused(x, w, b, gzn)
    res = {"bf16": errors(got, _reference(x, w, b, gzn, True))}
    res["fp32"] = errors(got, _reference(x, w, b, gzn, False))
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_matches_fp64_on_bf16_operands(shape):
    e = measure(shape)["bf16"]
    assert e["zn"][2] <= ZN_ABS_BF16, e
    for k, bound in BF16_REF_MAXABS.items():
        assert e[k][0] <= bound, (k, e)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_matches_fp64_on_fp32_operands(shape):
    e = measure(shape)["fp32"]
    for k in FP32_REF_MAXABS:
        assert e[k][0] <= FP32_REF_MAXABS[k] and e[k][1] <= FP32_REF_FROB[k], (k, e)


@pytest.mark.gpu
def test_clamped_pixel_matches_f_normalize():
    """An all-zero pixel column with zero bias: z = 0 there, zn = 0 and gz = gzn / eps (F.normalize's clamp)."""
    x, w, _, gzn = _inputs((2, 100, 5, 7), seed=3)
    x[1, :, 2, 3] = 0.
    b = torch.zeros(256, device=DEV)
    got = _fused(x, w, b, gzn)
    ref = _reference(x, w, b, gzn, True)
    assert got["zn"][1, :, 2, 3].abs().max().item() == 0.
    assert (got["zn"].double() - ref["zn"]).abs().max().item() <= ZN_ABS_BF16
    g, r = got["gx"][1, :, 2, 3].double(), ref["gx"][1, :, 2, 3]
    assert r.abs().max().item() > 1e9                                     # the clamped branch: gzn * 1e12
    assert (g - r).abs().max().item() <= 1e-5 * r.abs().max().item()
    for k in ("gw", "gb"):
        assert (got[k].double() - ref[k]).abs().max().item() <= 1e-5 * ref[k].abs().max().item(), k


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 2048, 66, 66), (3, 100, 5, 7)])
def test_weight_gradient_is_bit_reproducible(shape):
    x, w, b, gzn = _inputs(shape, seed=5)
    a, c = _fused(x, w, b, gzn), _fused(x, w, b, gzn)
    for k in ("zn", "gx", "gw", "gb"):
        assert torch.equal(a[k], c[k]), k


@pytest.mark.gpu
def test_cuda_graph_replay_is_bit_identical_to_eager():
    x, w, b, gzn = _inputs((2, 720, 33, 40), seed=7)
    eager = _fused(x, w, b, gzn)
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


def _heads(proj, Cin):
    torch.manual_seed(11)
    ref = cs.ProjectionHead(Cin, 256, proj, bn_type="torchbn").to(DEV)
    fused = cs.ProjectionHead(Cin, 256, proj, bn_type="torchbn", fused=True).to(DEV)
    fused.load_state_dict(ref.state_dict())
    # eval: BatchNorm on its running statistics (in training mode the gradient of the bias feeding it is exactly zero,
    # and its two rounding residues cannot be compared relative to their own size)
    return ref.eval(), fused.eval()


@pytest.mark.gpu
@pytest.mark.parametrize("proj", ["convmlp", "linear"])
def test_fused_head_matches_the_unfused_head(proj, shape=(2, 96, 12, 20)):
    ref, fused = _heads(proj, shape[1])
    assert list(fused.state_dict().keys()) == list(ref.state_dict().keys())
    x = torch.randn(shape, generator=torch.Generator().manual_seed(12)).to(DEV)
    xr, xf = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    yr, yf = ref(xr), fused(xf)
    gy = torch.randn(yr.shape, generator=torch.Generator().manual_seed(13)).to(DEV)
    yr.backward(gy)
    yf.backward(gy)
    pairs = [("zn", yf.detach(), yr.detach()), ("gx", xf.grad, xr.grad)]
    pairs += [(n, pf.grad, pr.grad) for (n, pf), (_, pr) in zip(fused.named_parameters(), ref.named_parameters())]
    for name, a, r in pairs:
        d = (a - r).double()
        assert d.abs().max().item() <= FP32_REF_MAXABS["gx"] * r.abs().max().item(), name
        assert d.norm().item() <= FP32_REF_FROB["gx"] * r.double().norm().item(), name


@pytest.mark.gpu
def test_fused_head_refuses_what_it_does_not_implement():
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 128, "linear", fused=True)
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "linear", normalize=False, fused=True)
    head = cs.ProjectionHead(64, 256, "linear", fused=True).to(DEV)
    with pytest.raises(_abi.PclError):
        head(torch.randn(1, 64, 4, 4, device=DEV, dtype=torch.float64))
    with pytest.raises(_abi.PclError):
        head(torch.randn(1, 64, 4, 4, device=DEV, dtype=torch.float16))
    if DEV != "cpu":
        with pytest.raises(_abi.PclError):
            head(torch.randn(1, 64, 4, 4))
