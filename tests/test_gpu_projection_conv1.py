"""The projection head's first 1x1 convolution on the engine (csrc/pcl_norm.cu k_conv1_*, the pcl_proj_conv1_* C ABI,
functional.conv_bn_relu_project_normalize, ProjectionHead(fused=True, fuse_bn_relu=True, fuse_conv1=True)): conv1
alone against float64 on its bf16 operands, the BatchNorm sums of its epilogue against float64 sums of the stored y,
the whole head against a float64 conv1 + BN + ReLU + conv2 + normalise (+ autograd), and against the fuse_bn_relu head
whose conv1 is cuDNN's.  test_emu_projection_conv1.py runs these functions at small shapes on the emulated kernels
(DEV = "cpu")."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import contrastiveseg_b200 as cs
import test_gpu_projection as P
import test_gpu_projection_bnrelu as PB
from contrastiveseg_b200 import _abi
from contrastiveseg_b200 import functional as Fn

DEV = "cuda:0"
BF = torch.bfloat16

# a Cin below 128 with a pixel-tile tail, C not a multiple of 8, an odd square image, S1 (BASELINE configs[1] head
# input), DeepLab C4
SHAPES = [(2, 96, 12, 20), (1, 100, 9, 13), (1, 720, 97, 97), (8, 720, 128, 256), (2, 2048, 66, 66)]
DTYPES = [torch.float32, BF]

# conv1 alone, against float64 on the bf16-rounded x, W1 and g_y (max-abs / max|reference|): what remains is the fp32
# accumulation order and, for bf16 y and gx, their rounding to bf16.  3x the worst measured on an H100 80GB HBM3 (700 W)
# over SHAPES x {fp32, bf16} (DESIGN §2).
CONV1_MAXABS = {torch.float32: {"y": 9e-6, "gx": 9e-6, "gw1": 4e-5, "gb1": 1.3e-6},
                BF: {"y": 9.1e-3, "gx": 1e-2, "gw1": 4e-5, "gb1": 1.3e-6}}
SUMS_REL = 1e-12                 # |sum - float64 sum of the stored y| <= SUMS_REL * sum |y| (resp. sum y^2)

# The whole head against the float64 chain on the same inputs, conv1's operands rounded where the GEMMs round them (x, W1
# and g_y to bf16) and y taken as conv1 stored it (checked against the float64 y within CONV1_MAXABS on the way):
# max-abs / max|reference| and relative Frobenius, 3x the worst measured on an H100 80GB HBM3 (700 W) over
# SHAPES x {train, eval} x {fp32, bf16} (DESIGN §2).  Without the stored y, an element whose float64 and fp32 (or bf16)
# values fall on either side of the ReLU's kink takes the other branch, and its gradient reaches every input channel of
# its pixel.  gx is compared with the pixels that hold a ReLU-kink element left out of its max-abs, as gy is in
# test_gpu_projection_bnrelu.py.
NAMES = ("zn", "gx", "gw1", "gb1", "ggamma", "gbeta", "gw2", "gb2")
HEAD_MAXABS = {"zn": 1.3e-2, "gx": 1.8e-2, "gw1": 4e-2, "gb1": 2e-2, "ggamma": 1.1e-2, "gbeta": 1.6e-2, "gw2": 7.5e-3,
               "gb2": 5.8e-3}
HEAD_FROB = {"zn": 9e-3, "gx": 1.3e-2, "gw1": 1.2e-2, "gb1": 1.4e-2, "ggamma": 9.5e-3, "gbeta": 8.5e-3, "gw2": 7.2e-3,
             "gb2": 5.4e-3}
# training gb1 against sum_p |g_y|: the kernel's and the reference's g_y elements round to bf16 values that differ by
# rounding only, so by at most one ulp (<= 2^-7 relative); the fp32 sum adds ~1e-6
GB1_TRAIN_REL = 2. ** -7
KINK = PB.KINK
STATS_REL = PB.STATS_REL


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


def _r(t):
    """t's values as the GEMMs see them: rounded to bf16 (nearest-even), in float64."""
    return t.to(BF).double()


# ------------------------------------------------------------------------------------------------------------------
# conv1 alone through the C ABI
# ------------------------------------------------------------------------------------------------------------------
def conv1_abi(x, w1, b1, gy=None, with_gx=True):
    """pcl_proj_conv1_pack + _fwd_dt (with the sums) and, given gy, _bwd_dt: {"y", "sums"[, "gx", "gw1", "gb1"]}."""
    lib = _abi.load()
    B, C, H, W = x.shape
    HW = H * W
    dt = Fn.proj_dtype_code(x.dtype)
    dev = x.device
    s = Fn._stream_ptr(dev)
    xc = x.contiguous()
    pack = torch.empty(lib.pcl_proj_conv1_workspace_bytes(B, C, HW, 0), dtype=torch.uint8, device=dev)
    scratch = torch.empty(lib.pcl_proj_conv1_workspace_bytes(B, C, HW, 1), dtype=torch.uint8, device=dev)
    y = torch.empty_like(xc)
    sums = torch.empty(2 * C + 1, dtype=torch.float64, device=dev)
    w = w1.reshape(C, C).float().contiguous()
    _abi.check(lib.pcl_proj_conv1_pack(w.data_ptr(), C, pack.data_ptr(), s))
    _abi.check(lib.pcl_proj_conv1_fwd_dt(xc.data_ptr(), dt, pack.data_ptr(), b1.data_ptr(), B, C, HW, y.data_ptr(),
                                         sums.data_ptr(), scratch.data_ptr(), s))
    out = {"y": y, "sums": sums}
    if gy is not None:
        bscr = torch.empty(lib.pcl_proj_conv1_workspace_bytes(B, C, HW, 2), dtype=torch.uint8, device=dev)
        gx = torch.empty_like(xc) if with_gx else None
        gw1 = torch.empty((C, C), dtype=torch.float32, device=dev)
        gb1 = torch.empty(C, dtype=torch.float32, device=dev)
        gyc = gy.contiguous()
        _abi.check(lib.pcl_proj_conv1_bwd_dt(xc.data_ptr(), dt, gyc.data_ptr(), pack.data_ptr(), B, C, HW,
                                             bscr.data_ptr(), _abi.ptr(gx), gw1.data_ptr(), gb1.data_ptr(), s))
        out.update(gx=gx, gw1=gw1, gb1=gb1)
    _sync()
    return out


def _conv1_inputs(shape, dtype, seed=0):
    B, C, H, W = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    w1 = torch.randn(C, C, generator=g) / C ** 0.5
    b1 = 0.1 * torch.randn(C, generator=g)
    gy = torch.randn(shape, generator=g)
    return x.to(device=DEV, dtype=dtype), w1.to(DEV), b1.to(DEV), gy.to(device=DEV, dtype=dtype)


def conv1_reference(x, w1, b1, gy):
    """float64 y, gx, gW1, gb1 on the bf16-rounded x, W1 and gy."""
    B, C = x.shape[:2]
    x64, w64, g64 = _r(x), _r(w1).reshape(C, C), _r(gy)
    y = F.conv2d(x64, w64.reshape(C, C, 1, 1), b1.double())
    gx = F.conv2d(g64, w64.t().reshape(C, C, 1, 1))
    gw = torch.einsum("bnp,bcp->nc", g64.reshape(B, C, -1), x64.reshape(B, C, -1))
    return {"y": y, "gx": gx, "gw1": gw, "gb1": g64.sum((0, 2, 3))}


def measure_conv1(shape, dtype, seed=0):
    x, w1, b1, gy = _conv1_inputs(shape, dtype, seed)
    got = conv1_abi(x, w1, b1, gy)
    ref = conv1_reference(x, w1, b1, gy)
    e = P.errors({k: got[k] for k in ref}, ref)
    # the sums against float64 sums of the stored y
    y = got["y"].double()
    C = shape[1]
    s1, s2 = y.sum((0, 2, 3)), (y * y).sum((0, 2, 3))
    e["sum_y"] = ((got["sums"][:C] - s1).abs() / y.abs().sum((0, 2, 3)).clamp_min(1e-300)).max().item()
    e["sum_y2"] = ((got["sums"][C:2 * C] - s2).abs() / s2.clamp_min(1e-300)).max().item()
    e["count"] = got["sums"][2 * C].item() - y.numel() / C
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES)
def test_conv1_matches_fp64_on_bf16_operands(shape, dtype):
    e = measure_conv1(shape, dtype)
    print(f"\nMEASURED conv1 {shape} {dtype}: " + " ".join(f"{k} {e[k][0]:.3e}" for k in ("y", "gx", "gw1", "gb1")) +
          f" sum_y {e['sum_y']:.3e} sum_y2 {e['sum_y2']:.3e}")
    for k, bound in CONV1_MAXABS[dtype].items():
        assert e[k][0] <= bound, (k, e)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES)
def test_conv1_sums_match_fp64_sums_of_the_stored_y(shape, dtype):
    e = measure_conv1(shape, dtype, seed=1)
    assert e["sum_y"] <= SUMS_REL and e["sum_y2"] <= SUMS_REL, e
    assert e["count"] == 0, e


@pytest.mark.gpu
def test_conv1_without_gx_writes_the_same_weight_gradient(shape=(2, 100, 9, 13)):
    x, w1, b1, gy = _conv1_inputs(shape, torch.float32, seed=2)
    a, c = conv1_abi(x, w1, b1, gy), conv1_abi(x, w1, b1, gy, with_gx=False)
    for k in ("y", "sums", "gw1", "gb1"):
        assert torch.equal(a[k], c[k]), k


# ------------------------------------------------------------------------------------------------------------------
# the whole head
# ------------------------------------------------------------------------------------------------------------------
def _head_inputs(shape, mode="train", dtype=torch.float32, seed=0):
    """x, conv1's weight and bias, a BatchNorm2d with non-trivial affine parameters and running buffers, the last
    conv's weight and bias, and the incoming gradient of zn."""
    B, C, H, W = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    w1 = torch.randn(C, C, 1, 1, generator=g) / C ** 0.5
    b1 = 0.5 * torch.randn(C, generator=g)
    bn = nn.BatchNorm2d(C)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.2 * torch.randn(C, generator=g))
        bn.bias.copy_(0.2 * torch.randn(C, generator=g))
        bn.running_mean.copy_(0.3 * torch.randn(C, generator=g))
        bn.running_var.copy_(0.5 + torch.rand(C, generator=g))
    w2 = torch.randn(256, C, 1, 1, generator=g) / C ** 0.5
    b2 = 0.1 * torch.randn(256, generator=g)
    gzn = torch.randn(B, 256, H, W, generator=g)
    bn.train(mode == "train")
    return (x.to(device=DEV, dtype=dtype), w1.to(DEV), b1.to(DEV), bn.to(DEV), w2.to(DEV), b2.to(DEV),
            gzn.to(device=DEV, dtype=dtype))


def _head(x, w1, b1, bn, w2, b2, gzn):
    """One forward + backward of conv_bn_relu_project_normalize; bn's buffers are updated in place (training mode)."""
    xx = x.clone().requires_grad_(True)
    ps = [t.clone().requires_grad_(True) for t in (w1, b1, w2, b2)]
    bn.weight.grad = bn.bias.grad = None
    zn = cs.conv_bn_relu_project_normalize(xx, ps[0], ps[1], bn, ps[2], ps[3])
    zn.backward(gzn)
    _sync()
    return {"zn": zn.detach(), "gx": xx.grad, "gw1": ps[0].grad, "gb1": ps[1].grad, "ggamma": bn.weight.grad.clone(),
            "gbeta": bn.bias.grad.clone(), "gw2": ps[2].grad, "gb2": ps[3].grad}




def head_reference(x, w1, b1, bn, w2, b2, gzn):
    """float64 conv1 + BN (+ running-buffer update on copies) + ReLU + conv2 + normalise and autograd, with conv1's
    operands as its GEMMs see them: x, W1 and the gradient of y rounded to bf16, and y's value the one conv1 stores
    (after checking it against the float64 y).  Returns the outputs and {"mean", "var" (biased), "running_mean",
    "running_var", "kink"} in float64."""
    x64, w164 = _r(x).requires_grad_(True), _r(w1).requires_grad_(True)
    b164 = b1.double().requires_grad_(True)
    g64 = bn.weight.detach().double().requires_grad_(True)
    be64 = bn.bias.detach().double().requires_grad_(True)
    w264, b264 = w2.double().requires_grad_(True), b2.double().requires_grad_(True)
    y = F.conv2d(x64, w164, b164)
    stored = conv1_abi(x, w1, b1)["y"].double()
    assert (stored - y).abs().max().item() <= CONV1_MAXABS[x.dtype]["y"] * y.abs().max().item()
    y = y + (stored - y).detach()
    gy_abs = []

    def round_grad(g):                                   # g_y as the conv1 GEMMs take it
        gy_abs.append(g.abs().sum((0, 2, 3)))
        return g.to(BF).double()
    y.register_hook(round_grad)
    rm, rv = bn.running_mean.double().clone(), bn.running_var.double().clone()
    a = F.batch_norm(y, rm, rv, g64, be64, bn.training, bn.momentum, bn.eps)
    zn = F.normalize(F.conv2d(F.relu(a), w264, b264), p=2, dim=1)
    grads = torch.autograd.grad(zn, (x64, w164, b164, g64, be64, w264, b264), gzn.double())
    yd, ad = y.detach(), a.detach()
    stats = {"mean": yd.mean((0, 2, 3)), "var": yd.var((0, 2, 3), unbiased=False), "running_mean": rm,
             "running_var": rv, "kink": ad.abs() <= KINK * ad.abs().max(), "gy_abs_sum": gy_abs[0]}
    return dict(zip(NAMES, (zn.detach(),) + grads)), stats


def head_errors(got, ref, st, training):
    """P.errors, gx's max-abs without the kink pixels.  In training gb1 = sum_p g_y is zero in exact arithmetic (the
    batch mean removes b1) and what the GEMM sums is g_y rounded to bf16: its error is taken per channel relative to
    sum_p |g_y| (max over channels, and in norm), and bounded by GB1_TRAIN_REL."""
    e = P.errors(got, ref)
    if training:
        d = got["gb1"].double() - ref["gb1"]
        a = st["gy_abs_sum"]
        e["gb1"] = ((d.abs() / a).max().item(), (d.norm() / a.norm()).item(), d.abs().max().item())
    d = (got["gx"].double() - ref["gx"]).masked_fill(st["kink"].any(1, keepdim=True), 0.)
    e["gx"] = ((d.abs().max() / ref["gx"].abs().max()).item(),) + e["gx"][1:]
    return e


def check_head(e, training):
    for k in NAMES:
        if training and k == "gb1":
            assert e[k][0] <= GB1_TRAIN_REL and e[k][1] <= GB1_TRAIN_REL, (k, e)
        else:
            assert e[k][0] <= HEAD_MAXABS[k] and e[k][1] <= HEAD_FROB[k], (k, e)


def measure_head(shape, mode, dtype, seed=0):
    x, w1, b1, bn, w2, b2, gzn = _head_inputs(shape, mode, dtype, seed)
    ref, st = head_reference(x, w1, b1, bn, w2, b2, gzn)
    got = _head(x, w1, b1, bn, w2, b2, gzn)
    e = head_errors(got, ref, st, bn.training)
    for k in ("running_mean", "running_var"):
        e[k] = ((getattr(bn, k).double() - st[k]).abs().max() / st[k].abs().max()).item()
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", SHAPES)
def test_head_matches_fp64(shape, mode, dtype):
    e = measure_head(shape, mode, dtype)
    print(f"\nMEASURED head {shape} {mode} {dtype}: " + " ".join(f"{k} {e[k][0]:.3e}/{e[k][1]:.3e}" for k in NAMES) +
          f" rm {e['running_mean']:.3e} rv {e['running_var']:.3e}")
    check_head(e, mode == "train")
    for k in ("running_mean", "running_var"):
        assert e[k] <= STATS_REL, (k, e)


def _grid(shape, step, g):
    """Multiples of `step` in [-2 step, 2 step]."""
    return torch.randint(-2, 3, shape, generator=g).float() * step


def _heads(C, mode, seed=11):
    """The fuse_bn_relu head (cuDNN conv1) and the fuse_conv1 head from one state_dict.  conv1's weight and bias are
    multiples of 1/4 in [-1/2, 1/2] and x holds multiples of 1/2 in [-1, 1], so y is a multiple of 1/8 below 32 in
    magnitude (12 standard deviations at C = 96): every product, partial sum, bias add and the bf16 rounding of y are
    exact, and both convolutions form the same y in any order and with any intermediate rounding.  Without that, an
    element the two round to neighbouring values next to the ReLU's kink takes the other branch in one head."""
    torch.manual_seed(seed)
    ref = cs.ProjectionHead(C, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True).to(DEV)
    new = cs.ProjectionHead(C, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                            fuse_conv1=True).to(DEV)
    with torch.no_grad():
        g = torch.Generator().manual_seed(seed)
        ref.proj[0].weight.copy_(_grid(ref.proj[0].weight.shape, 1 / 4, g))
        ref.proj[0].bias.copy_(_grid(ref.proj[0].bias.shape, 1 / 4, g))
        bn = ref.proj[1][0]
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.3, 0.3)
        bn.running_mean.uniform_(-0.2, 0.2)
        bn.running_var.uniform_(0.5, 1.5)
    new.load_state_dict(ref.state_dict())
    return ref.train(mode == "train"), new.train(mode == "train")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "autocast"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_head_matches_the_cudnn_conv1_head(mode, dtype, shape=(2, 96, 12, 20)):
    """fuse_conv1=True against fuse_bn_relu=True alone (cuDNN conv1) on the same weights and x (so the same y), fp32 and
    under autocast(bfloat16): outputs and gradients within twice the whole-head bounds, running buffers within 1e-5,
    the same num_batches_tracked.  In training mode the gradient of conv1's bias is zero in exact arithmetic; it is
    bounded against max|gW1|."""
    ref, new = _heads(shape[1], mode)
    assert list(new.state_dict().keys()) == list(ref.state_dict().keys())
    x = _grid(shape, 1 / 2, torch.Generator().manual_seed(12)).to(DEV)
    xr, xn = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    with torch.autocast(str(DEV).split(":")[0], dtype=BF, enabled=dtype == BF):
        zr, zn = ref(xr), new(xn)
    assert zn.dtype == zr.dtype == dtype
    gzn = torch.randn(zr.shape, generator=torch.Generator().manual_seed(13)).to(device=DEV, dtype=dtype)
    zr.backward(gzn)
    zn.backward(gzn)
    _sync()
    pairs = [("zn", zn.detach(), zr.detach()), ("gx", xn.grad, xr.grad)]
    pairs += [(n, pn.grad, pr.grad) for (n, pn), (_, pr) in zip(new.named_parameters(), ref.named_parameters())]
    gw1 = ref.proj[0].weight.grad.double().abs().max().item()
    for name, a, r in pairs:
        d = a.double() - r.double()
        if mode == "train" and name == "proj.0.bias":
            assert a.double().abs().max().item() <= 2 * HEAD_MAXABS["gb1"] * gw1, name
            continue
        assert d.abs().max().item() <= 2 * HEAD_MAXABS["gx"] * r.double().abs().max().item(), name
        assert d.norm().item() <= 2 * HEAD_FROB["gx"] * r.double().norm().item(), name
    bn_r, bn_n = ref.proj[1][0], new.proj[1][0]
    for k in ("running_mean", "running_var"):
        r = getattr(bn_r, k).double()
        assert (getattr(bn_n, k).double() - r).abs().max().item() <= STATS_REL * r.abs().max().item(), k
    assert bn_n.num_batches_tracked.item() == bn_r.num_batches_tracked.item() == (1 if mode == "train" else 0)


@pytest.mark.gpu
def test_autocast_equals_the_call_on_bf16_x(shape=(2, 96, 12, 20)):
    _, head = _heads(shape[1], "eval")
    x = torch.randn(shape, generator=torch.Generator().manual_seed(14)).to(DEV)
    with torch.autocast(str(DEV).split(":")[0], dtype=BF):
        za = head(x)
    zb = head(x.to(BF))
    assert za.dtype == BF and torch.equal(za, zb)


CANCEL_SHAPE = (2, 96, 12, 20)


@pytest.mark.gpu
def test_large_mean_through_b1_does_not_cancel():
    """Channel 0 of y with mean 1000 x its standard deviation, from b1[0] = 1000."""
    x, w1, b1, bn, w2, b2, gzn = _head_inputs(CANCEL_SHAPE, "train", seed=4)
    b1[0] = 1000.
    bn.momentum = 1.0
    ref, st = head_reference(x, w1, b1, bn, w2, b2, gzn)
    got = _head(x, w1, b1, bn, w2, b2, gzn)
    n = x.numel() // x.shape[1]
    var_u = st["var"] * n / (n - 1)
    assert st["mean"][0].item() > 900 and st["var"][0].item() < 10
    rel = ((bn.running_var.double() - var_u).abs() / var_u).max().item()
    assert rel <= STATS_REL, rel
    assert ((bn.running_mean.double() - st["mean"]).abs() / st["mean"].abs()).max().item() <= STATS_REL
    check_head(head_errors(got, ref, st, True), True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_bit_reproducible(mode, shape=(2, 720, 33, 40)):
    x, w1, b1, bn, w2, b2, gzn = _head_inputs(shape, mode, seed=6)
    bn2 = copy.deepcopy(bn)
    a, c = _head(x, w1, b1, bn, w2, b2, gzn), _head(x, w1, b1, bn2, w2, b2, gzn)
    for k in NAMES:
        assert torch.equal(a[k], c[k]), k
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(bn, k), getattr(bn2, k)), k


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "bf16"])
def test_cuda_graph_replay_is_bit_identical_to_eager(dtype, replays=3):
    """Training mode: every replay of forward + backward equals an eager call, and the running buffers and the counter
    after warm-up + replays equal those after as many eager calls."""
    x, w1, b1, bn, w2, b2, gzn = _head_inputs((2, 720, 33, 40), "train", dtype, seed=7)
    bn_g = copy.deepcopy(bn)
    xx = x.clone().requires_grad_(True)
    ps = [t.clone().requires_grad_(True) for t in (w1, b1, w2, b2)]
    leaves = [xx] + ps + [bn_g.weight, bn_g.bias]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    warm = 2
    with torch.cuda.stream(s):                                             # warm-up outside the capture
        for _ in range(warm):
            cs.conv_bn_relu_project_normalize(xx, ps[0], ps[1], bn_g, ps[2], ps[3]).backward(gzn)
            for t in leaves:
                t.grad = None
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        zn = cs.conv_bn_relu_project_normalize(xx, ps[0], ps[1], bn_g, ps[2], ps[3])
        zn.backward(gzn)
    eager = None
    for _ in range(warm + replays):
        eager = _head(x, w1, b1, bn, w2, b2, gzn)
    for _ in range(replays):
        for t in leaves:
            t.grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
        got = {"zn": zn.detach(), "gx": xx.grad, "gw1": ps[0].grad, "gb1": ps[1].grad, "ggamma": bn_g.weight.grad,
               "gbeta": bn_g.bias.grad, "gw2": ps[2].grad, "gb2": ps[3].grad}
        for k in NAMES:
            assert torch.equal(got[k], eager[k]), k
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(bn_g, k), getattr(bn, k)), k
    assert bn_g.num_batches_tracked.item() == warm + replays


@pytest.mark.gpu
def test_refusals():
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "convmlp", bn_type="torchbn", fused=True, fuse_conv1=True)
    with pytest.raises(_abi.PclError):
        cs.ProjectionHead(64, 256, "linear", fused=True, fuse_bn_relu=True, fuse_conv1=True)
    x, w1, b1, bn, w2, b2, _ = _head_inputs((1, 64, 4, 4))
    for kw in ({"momentum": None}, {"affine": False}, {"track_running_stats": False}):
        bad = nn.BatchNorm2d(64, **kw).to(DEV)
        with pytest.raises(_abi.PclError):
            cs.conv_bn_relu_project_normalize(x, w1, b1, bad, w2, b2)
    bad = nn.BatchNorm2d(64).to(DEV).double()
    with pytest.raises(_abi.PclError):
        cs.conv_bn_relu_project_normalize(x, w1, b1, bad, w2, b2)
    with pytest.raises(_abi.PclError):
        cs.conv_bn_relu_project_normalize(x.to(torch.float16), w1, b1, bn, w2, b2)
    head = cs.ProjectionHead(64, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                             fuse_conv1=True).to(DEV)
    with pytest.raises(_abi.PclError):
        head(x.to(torch.float16))
    with pytest.raises(_abi.PclError):
        with torch.autocast(str(DEV).split(":")[0], dtype=torch.float16):
            head(x)
    head.proj[1][0].momentum = None
    with pytest.raises(_abi.PclError):
        head(x)
    # the C ABI refuses fp16 and unknown codes
    lib = _abi.load()
    for code in (_abi.DT_F16, 7):
        assert lib.pcl_proj_conv1_fwd_dt(1, code, 1, None, 1, 64, 16, 1, None, None, None) != 0
        assert lib.pcl_proj_conv1_bwd_dt(1, code, 1, 1, 1, 64, 16, 1, None, 1, None, None) != 0
