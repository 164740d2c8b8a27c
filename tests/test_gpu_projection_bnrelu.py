"""The projection head's BatchNorm + ReLU fused into the last-conv GEMM (csrc/pcl_norm.cu k_bn_* and the BN
instantiations of k_proj_*, functional.bn_relu_project_normalize, ProjectionHead(fused=True, fuse_bn_relu=True)) against
float64 F.batch_norm + F.relu + F.conv2d + F.normalize (+ autograd), and against the fused=True head whose BN and ReLU
run in torch.  test_emu_projection_bnrelu.py runs these functions at small shapes on the emulated kernels
(DEV = "cpu")."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import contrastiveseg_b200 as cs
import test_gpu_projection as P
from contrastiveseg_b200 import _abi

DEV = "cuda:0"
BF = torch.bfloat16

# a Cin below 128 with a pixel-tile tail, an odd square image, S1 (BASELINE configs[1] head input)
SHAPES = [(2, 96, 12, 20), (1, 720, 97, 97), (8, 720, 128, 256)]
NAMES = ("zn", "gy", "gw", "gb", "ggamma", "gbeta")
# zn, gy (the input gradient, bounded like the plain head's gx), gw and gb: the fp32-operand bounds of the plain fused
# head.  gamma / beta gradients, relative to max|reference| and to ||reference||: 3x the worst measured on an H100 80GB
# HBM3 (700 W) over SHAPES x {train, eval} x {fp32, bf16} (max-abs / Frobenius: ggamma 4.24e-3 / 2.65e-3, gbeta
# 3.14e-3 / 2.68e-3; DESIGN §4).
BN_PARAM_MAXABS = {"ggamma": 1.3e-2, "gbeta": 9.5e-3}
BN_PARAM_FROB = {"ggamma": 8e-3, "gbeta": 8e-3}
# The ReLU mask of an element whose BN output is within rounding of 0 may differ between fp32 and fp64 (a kink, not an
# error): such elements (|BN output| <= KINK * max|BN output| in float64) are left out of gy's max-abs comparison and
# kept in its Frobenius norm.  The fp32 rounding of the BN output is ~1e-7 relative.
KINK = 1e-5
MAXABS = dict(P.FP32_REF_MAXABS, gy=P.FP32_REF_MAXABS["gx"], **BN_PARAM_MAXABS)
FROB = dict(P.FP32_REF_FROB, gy=P.FP32_REF_FROB["gx"], **BN_PARAM_FROB)
STATS_REL = 1e-5


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


def _inputs(shape, mode="train", dtype=torch.float32, seed=0):
    """y with per-channel offsets and scales, a BatchNorm2d with non-trivial affine parameters and running buffers, the
    last conv's weight and bias, and the incoming gradient of zn."""
    B, C, H, W = shape
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(shape, generator=g) * (0.5 + torch.rand(1, C, 1, 1, generator=g)) + \
        0.5 * torch.randn(1, C, 1, 1, generator=g)
    bn = nn.BatchNorm2d(C)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.2 * torch.randn(C, generator=g))
        bn.bias.copy_(0.2 * torch.randn(C, generator=g))
        bn.running_mean.copy_(0.3 * torch.randn(C, generator=g))
        bn.running_var.copy_(0.5 + torch.rand(C, generator=g))
    w = torch.randn(256, C, 1, 1, generator=g) / C ** 0.5
    b = 0.1 * torch.randn(256, generator=g)
    gzn = torch.randn(B, 256, H, W, generator=g)
    bn.train(mode == "train")
    return y.to(device=DEV, dtype=dtype), bn.to(DEV), w.to(DEV), b.to(DEV), gzn.to(device=DEV, dtype=dtype)


def _fused(y, bn, w, b, gzn):
    """One forward + backward of bn_relu_project_normalize; bn's buffers are updated in place (training mode)."""
    yy, ww, bb = y.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    bn.weight.grad = bn.bias.grad = None
    zn = cs.bn_relu_project_normalize(yy, bn, ww, bb)
    zn.backward(gzn)
    _sync()
    return {"zn": zn.detach(), "gy": yy.grad, "gw": ww.grad, "gb": bb.grad, "ggamma": bn.weight.grad.clone(),
            "gbeta": bn.bias.grad.clone()}


def _reference(y, bn, w, b, gzn):
    """float64 BN (+ running-buffer update on copies) + ReLU + conv + normalise and autograd.  Returns the outputs and
    {"mean", "var" (biased), "running_mean", "running_var"} in float64."""
    y64 = y.double().requires_grad_(True)
    g64 = bn.weight.detach().double().requires_grad_(True)
    be64 = bn.bias.detach().double().requires_grad_(True)
    w64, b64 = w.double().requires_grad_(True), b.double().requires_grad_(True)
    rm, rv = bn.running_mean.double().clone(), bn.running_var.double().clone()
    a = F.batch_norm(y64, rm, rv, g64, be64, bn.training, bn.momentum, bn.eps)
    zn = F.normalize(F.conv2d(F.relu(a), w64, b64), p=2, dim=1)
    gy, gg, gbe, gw, gb = torch.autograd.grad(zn, (y64, g64, be64, w64, b64), gzn.double())
    stats = {"mean": y64.detach().mean((0, 2, 3)), "var": y64.detach().var((0, 2, 3), unbiased=False),
             "running_mean": rm, "running_var": rv, "kink": a.detach().abs() <= KINK * a.detach().abs().max()}
    return {"zn": zn.detach(), "gy": gy, "gw": gw, "gb": gb, "ggamma": gg, "gbeta": gbe}, stats


def measure(shape, mode, dtype, seed=0):
    """{name: (max-abs / max|ref|, rel Frobenius, max-abs)}, plus the running buffers' relative errors."""
    y, bn, w, b, gzn = _inputs(shape, mode, dtype, seed)
    ref, st = _reference(y, bn, w, b, gzn)
    got = _fused(y, bn, w, b, gzn)
    e = P.errors(got, ref)
    d = (got["gy"].double() - ref["gy"]).masked_fill(st["kink"], 0.)
    e["gy"] = ((d.abs().max() / ref["gy"].abs().max()).item(),) + e["gy"][1:]
    for k in ("running_mean", "running_var"):
        e[k] = ((getattr(bn, k).double() - st[k]).abs().max() / st[k].abs().max()).item()
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", SHAPES)
def test_matches_fp64(shape, mode, dtype):
    e = measure(shape, mode, dtype)
    print(f"\nMEASURED {shape} {mode} {dtype}: " + " ".join(f"{k} {e[k][0]:.3e}/{e[k][1]:.3e}" for k in NAMES))
    for k in NAMES:
        assert e[k][0] <= MAXABS[k] and e[k][1] <= FROB[k], (k, e)
    for k in ("running_mean", "running_var"):
        assert e[k] <= STATS_REL, (k, e)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 96, 12, 20), (1, 720, 97, 97)])
def test_batch_statistics_and_counter_match_fp64(shape):
    """momentum = 1: the running buffers become the batch mean and the unbiased batch variance."""
    y, bn, w, b, gzn = _inputs(shape, "train", seed=1)
    bn.momentum = 1.0
    _, st = _reference(y, bn, w, b, gzn)
    n = y.numel() // y.shape[1]
    _fused(y, bn, w, b, gzn)
    assert (bn.running_mean.double() - st["mean"]).abs().max() <= STATS_REL * st["mean"].abs().max()
    assert (bn.running_var.double() - st["var"] * n / (n - 1)).abs().max() <= STATS_REL * st["var"].abs().max() * 2
    assert bn.num_batches_tracked.item() == 1


def _heads(Cin, mode, seed=11):
    torch.manual_seed(seed)
    ref = cs.ProjectionHead(Cin, 256, "convmlp", bn_type="torchbn", fused=True).to(DEV)
    new = cs.ProjectionHead(Cin, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True).to(DEV)
    with torch.no_grad():                                  # non-trivial affine parameters and running buffers
        bn = ref.proj[1][0]
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.3, 0.3)
        bn.running_mean.uniform_(-0.2, 0.2)
        bn.running_var.uniform_(0.5, 1.5)
    new.load_state_dict(ref.state_dict())
    return ref.train(mode == "train"), new.train(mode == "train")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_head_matches_the_torch_bn_relu_head(mode, dtype, shape=(2, 96, 12, 20)):
    """The whole head against fused=True alone (torch BN + ReLU, then the fused GEMM) on the same weights: outputs and
    gradients within twice the fp32-operand bounds, running buffers within 1e-5, the same num_batches_tracked.  In
    training mode the gradient of conv1's bias is zero in exact arithmetic; it is bounded against max|gW1|."""
    ref, new = _heads(shape[1], mode)
    assert list(new.state_dict().keys()) == list(ref.state_dict().keys())
    x = torch.randn(shape, generator=torch.Generator().manual_seed(12)).to(DEV)
    xr, xn = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    with torch.autocast(str(DEV).split(":")[0], dtype=BF, enabled=dtype == BF):     # bf16: conv1 hands over bf16 y
        yr, yn = ref(xr), new(xn)
    assert yn.dtype == yr.dtype == dtype
    gzn = torch.randn(yr.shape, generator=torch.Generator().manual_seed(13)).to(device=DEV, dtype=dtype)
    yr.backward(gzn)
    yn.backward(gzn)
    _sync()
    pairs = [("zn", yn.detach(), yr.detach()), ("gx", xn.grad, xr.grad)]
    pairs += [(n, pn.grad, pr.grad) for (n, pn), (_, pr) in zip(new.named_parameters(), ref.named_parameters())]
    gw1 = ref.proj[0].weight.grad.double().abs().max().item()
    for name, a, r in pairs:
        d = (a.double() - r.double())
        if mode == "train" and name == "proj.0.bias":
            assert a.double().abs().max().item() <= 2 * P.FP32_REF_MAXABS["gx"] * gw1, name
            continue
        assert d.abs().max().item() <= 2 * P.FP32_REF_MAXABS["gx"] * r.double().abs().max().item(), name
        assert d.norm().item() <= 2 * P.FP32_REF_FROB["gx"] * r.double().norm().item(), name
    bn_r, bn_n = ref.proj[1][0], new.proj[1][0]
    for k in ("running_mean", "running_var"):
        r = getattr(bn_r, k).double()
        assert (getattr(bn_n, k).double() - r).abs().max().item() <= STATS_REL * r.abs().max().item(), k
    assert bn_n.num_batches_tracked.item() == bn_r.num_batches_tracked.item() == (1 if mode == "train" else 0)


CANCEL_SHAPE = (2, 96, 12, 20)


def _cancellation_inputs():
    """Channel 0 with mean 1000 x its standard deviation (mean 1000, std 1)."""
    y, bn, w, b, gzn = _inputs(CANCEL_SHAPE, "train", seed=4)
    y[:, 0] = 1000. + torch.randn(y[:, 0].shape, generator=torch.Generator().manual_seed(5)).to(y.device)
    bn.momentum = 1.0
    return y, bn, w, b, gzn


@pytest.mark.gpu
def test_large_mean_channel_does_not_cancel():
    y, bn, w, b, gzn = _cancellation_inputs()
    ref, st = _reference(y, bn, w, b, gzn)
    got = _fused(y, bn, w, b, gzn)
    n = y.numel() // y.shape[1]
    var_u = st["var"] * n / (n - 1)
    rel = ((bn.running_var.double() - var_u).abs() / var_u).max().item()
    assert rel <= STATS_REL, rel
    assert ((bn.running_mean.double() - st["mean"]).abs() / st["mean"].abs()).max().item() <= STATS_REL
    e = P.errors(got, ref)
    d = (got["gy"].double() - ref["gy"]).masked_fill(st["kink"], 0.)
    e["gy"] = ((d.abs().max() / ref["gy"].abs().max()).item(),) + e["gy"][1:]
    for k in NAMES:
        assert e[k][0] <= MAXABS[k] and e[k][1] <= FROB[k], (k, e)
    # negative control: the one-pass fp32 formula E[y^2] - E[y]^2 misses the bound on that channel
    y0 = y[:, 0].float()
    one_pass = (y0 * y0).mean() - y0.mean() ** 2
    assert abs(one_pass.double().item() - st["var"][0].item()) / st["var"][0].item() > STATS_REL


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_bit_reproducible(mode, shape=(2, 96, 12, 20)):
    y, bn, w, b, gzn = _inputs(shape, mode, seed=6)
    bn2 = copy.deepcopy(bn)
    a, c = _fused(y, bn, w, b, gzn), _fused(y, bn2, w, b, gzn)
    for k in NAMES:
        assert torch.equal(a[k], c[k]), k
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(bn, k), getattr(bn2, k)), k


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_cuda_graph_replay_is_bit_identical_to_eager(dtype, replays=3):
    """Training mode: every replay equals an eager call, and the running buffers and the counter after warm-up +
    replays equal those after as many eager calls."""
    y, bn, w, b, gzn = _inputs((2, 720, 33, 40), "train", dtype, seed=7)
    bn_g = copy.deepcopy(bn)
    yy, ww, bb = y.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    warm = 2
    with torch.cuda.stream(s):                                             # warm-up outside the capture
        for _ in range(warm):
            cs.bn_relu_project_normalize(yy, bn_g, ww, bb).backward(gzn)
            yy.grad = ww.grad = bb.grad = bn_g.weight.grad = bn_g.bias.grad = None
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        zn = cs.bn_relu_project_normalize(yy, bn_g, ww, bb)
        zn.backward(gzn)
    eager = None
    for _ in range(warm + replays):
        eager = _fused(y, bn, w, b, gzn)
    for _ in range(replays):
        for t in (yy.grad, ww.grad, bb.grad, bn_g.weight.grad, bn_g.bias.grad):
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        got = {"zn": zn.detach(), "gy": yy.grad, "gw": ww.grad, "gb": bb.grad, "ggamma": bn_g.weight.grad,
               "gbeta": bn_g.bias.grad}
        for k in NAMES:
            assert torch.equal(got[k], eager[k]), k
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(bn_g, k), getattr(bn, k)), k
    assert bn_g.num_batches_tracked.item() == warm + replays


@pytest.mark.gpu
def test_refusals():
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "linear", fused=True, fuse_bn_relu=True)
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "convmlp", bn_type="torchbn", fuse_bn_relu=True)
    y, bn, w, b, _ = _inputs((1, 64, 4, 4))
    for kw in ({"momentum": None}, {"affine": False}, {"track_running_stats": False}):
        bad = nn.BatchNorm2d(64, **kw).to(DEV)
        with pytest.raises(_abi.PclError):
            cs.bn_relu_project_normalize(y, bad, w, b)
    with pytest.raises(_abi.PclError):
        cs.bn_relu_project_normalize(y.to(torch.float16), bn, w, b)
    head = cs.ProjectionHead(64, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True).to(DEV)
    head.proj[1][0].momentum = None
    with pytest.raises(_abi.PclError):
        head(torch.randn(1, 64, 4, 4, device=DEV))
    # the C ABI refuses fp16 and unknown codes
    lib = _abi.load()
    for code in (_abi.DT_F16, 7):
        assert lib.pcl_proj_bn_stats_dt(1, code, 1, 64, 16, 1, None) != 0
        assert lib.pcl_proj_bn_fwd_dt(1, code, 1, 1, None, 1, 64, 16, 1, 1, None) != 0
        assert lib.pcl_proj_bn_bwd_dt(1, code, 1, 1, 1, 1, 1, 1, 64, 16, 1, 1, 1, None, 1, None, None, None) != 0
        assert lib.pcl_proj_bn_input_grad_dt(1, code, 1, 1, 1, 64, 16, 1, 1, None) != 0
