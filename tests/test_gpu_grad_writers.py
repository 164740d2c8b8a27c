"""The dense-gradient writers (csrc/pcl_select.cu, dense_grad) against each other and against torch, bit for bit.

The loss step writes its (B, D, h, w) gradient in one of four ways: zero-fill and scatter in one pass per plane
(k_zero_scatter, from dA or from the sweep's per-split partial rows), a memset and a row scatter (k_scatter, the normalise
projection), or a scatter into a buffer the caller has zeroed (k_scatter_reduce from the partial rows, k_scatter from
dA).  pcl_step_backward and pcl_step_backward_prezeroed take different ones for the same forward, so their gradients
must be the same bits: compared as integers, since torch.equal takes -0 and +0 as equal and a zero-gradient row may hold
-0.  pcl_scatter_grad is checked against a torch index_put of dA (normalise off: bit for bit, -0 and subnormals
included) and against the float64 projection (normalise on: the kernel's warp-sum order is not torch's), with +0 at every
element no anchor owns.  The functions take DEV and their sizes as arguments so that tests/test_emu_grad_writers.py runs
them on the emulated kernels."""
import ctypes as C

import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi, functional as Fn
from contrastiveseg_b200.synth import make_contrast_batch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = "cuda:0"
PCL_ERR_UNSUPPORTED = -3
INT_VIEW = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(INT_VIEW[t.dtype])


def step_cases():
    """(precision, D, normalize, embed dtype, top-k): every combination the step accepts, top-k with fp32 embeds only."""
    cases = [pytest.param(p, D, n, e, 0, id=f"{p}-D{D}-norm{n}-{e}")
             for p, D in (("fp32", 64), ("bf16", 256)) for n in (0, 1) for e in DTYPES]
    cases += [pytest.param(p, D, 0, "fp32", 3, id=f"{p}-D{D}-topk3") for p, D in (("fp32", 64), ("bf16", 256))]
    return cases


def check_backward_entry_points(precision, D, normalize, embed_dtype, topk, B=2, h=24, w=32, ms=200, mv=12, K=6):
    """One forward (stats + forward at a fixed seed), run twice on one workspace: pcl_step_backward into a buffer full of
    garbage, pcl_step_backward_prezeroed into a zeroed one.  The two gradients must be the same bits.  A top-k step is
    refused by the prezeroed call."""
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=4, seed=23)
    dtype = DTYPES[embed_dtype]
    embed, tgt, seg = data["embed"].to(DEV).to(dtype), data["target"].to(DEV), data["seg"].to(DEV)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, seed=5,
                              precision=precision, normalize=bool(normalize), num_classes=K,
                              topk_negatives=topk or None)
    Fn.pixel_contrast_loss(embed, tgt, seg=seg, options=opts)      # binds a workspace and its descriptor
    ws = Fn._LAST_WS[embed.device.index]
    d, lib = ws.desc, _abi.load()
    loss = torch.zeros(1, dtype=torch.float32, device=DEV)
    go = torch.full((1,), -0.75, dtype=torch.float32, device=DEV)      # a negative scale: -0 where a sum is +0
    d.loss, d.seed = loss.data_ptr(), 0x5EED

    def run(backward, grad):
        _abi.check(lib.pcl_step_stats(C.byref(d), _stream()), "pcl_step_stats")
        _abi.check(lib.pcl_step_forward(C.byref(d), _stream()), "pcl_step_forward")
        d.grad_embed, d.embed_dtype = grad.data_ptr(), Fn.DTYPE_CODES[dtype]
        return backward(C.byref(d), go.data_ptr(), _stream())

    g1 = torch.full(embed.shape, -1.5, dtype=dtype, device=DEV)        # every element must be written
    _abi.check(run(lib.pcl_step_backward, g1), "pcl_step_backward")
    torch.cuda.synchronize()
    A = int(ws.plan[2].item())
    assert A > 0
    meta = ws.anchor_meta.view(4, ms)[:, :A].long()
    sampled = torch.zeros(B, h * w, dtype=torch.bool, device=DEV)
    sampled[meta[1], meta[0]] = True
    rows = g1.permute(0, 2, 3, 1).reshape(B, h * w, D)
    assert bool(torch.isfinite(rows[sampled].float()).all())
    assert bool((_bits(rows[~sampled]) == 0).all())                  # +0 wherever no anchor was sampled
    g2 = torch.zeros(embed.shape, dtype=dtype, device=DEV)
    rc = run(lib.pcl_step_backward_prezeroed, g2)
    torch.cuda.synchronize()
    if topk:
        assert rc == PCL_ERR_UNSUPPORTED
        return
    _abi.check(rc, "pcl_step_backward_prezeroed")
    assert int(ws.plan[2].item()) == A
    assert torch.equal(_bits(g1), _bits(g2))


@pytest.mark.parametrize("precision,D,normalize,embed_dtype,topk", step_cases())
def test_backward_entry_points_write_the_same_bits(precision, D, normalize, embed_dtype, topk):
    check_backward_entry_points(precision, D, normalize, embed_dtype, topk)


def check_scatter_grad(normalize, B=2, D=96, h=12, w=20, ms=160, A=150):
    """pcl_scatter_grad on a crafted dA with -0 rows and entries and subnormals, at A distinct sampled pixels."""
    gen = torch.Generator().manual_seed(17)
    HW = h * w
    flat = torch.randperm(B * HW, generator=gen)[:A]
    img, pix = flat // HW, flat % HW
    dA = torch.randn(A, D, generator=gen, dtype=torch.float64).float()
    dA[3] = -0.0                                                       # a zero-gradient row
    dA[7, ::3] = -0.0
    dA[11, 1::4] = torch.tensor(1e-40).float()                        # subnormals
    dA[12, ::5] = -torch.tensor(3e-42).float()
    y = torch.randn(A, D, generator=gen, dtype=torch.float64)
    y = y / y.norm(dim=1, keepdim=True)
    inv = torch.rand(A, generator=gen, dtype=torch.float64) + 0.5
    geom = _abi.Geom(B, D, h, w, h, w, 5, ms, 8, -1)
    plan = torch.zeros(_abi.PLAN_HEADER, dtype=torch.int32)
    plan[2] = A
    meta = torch.full((4, ms), -1, dtype=torch.int32)
    meta[0, :A], meta[1, :A] = pix.int(), img.int()
    pad = lambda t: torch.cat([t, torch.zeros((ms - A,) + t.shape[1:], dtype=t.dtype)])   # noqa: E731
    dev = {k: v.to(DEV).contiguous() for k, v in dict(plan=plan, meta=meta, dA=pad(dA), y=pad(y.float()),
                                                      inv=pad(inv.float())).items()}
    grad = torch.full((B, D, h, w), 7.0, dtype=torch.float32, device=DEV)     # every element must be written
    lib = _abi.load()
    _abi.check(lib.pcl_scatter_grad(C.byref(geom), dev["plan"].data_ptr(), dev["meta"].data_ptr(), dev["dA"].data_ptr(),
                                    dev["y"].data_ptr(), dev["inv"].data_ptr(), normalize, grad.data_ptr(), _stream()),
               "pcl_scatter_grad")
    torch.cuda.synchronize()
    g = grad.cpu().permute(0, 2, 3, 1).reshape(B, HW, D)
    sampled = torch.zeros(B, HW, dtype=torch.bool)
    sampled[img, pix] = True
    assert bool((_bits(g[~sampled]) == 0).all())                      # +0 where no anchor
    if not normalize:
        ref = torch.zeros(B, HW, D, dtype=torch.float32).index_put((img, pix), dA)
        assert torch.equal(_bits(g), _bits(ref))
        return
    yf = y.float().double()                                            # the projection of the fp32 rows the kernel reads
    ref = (dA.double() - yf * (yf * dA.double()).sum(1, keepdim=True)) * inv.float().double()[:, None]
    err = (g[img, pix].double() - ref).abs().max().item()
    assert err <= 1e-5 * ref.abs().max().item()


@pytest.mark.parametrize("normalize", [0, 1])
def test_scatter_grad_against_torch(normalize):
    check_scatter_grad(normalize)
