"""bf16 / fp16 inputs (embed, seg logits, bank keys) taken natively through the loss step.  Contract: the kernels convert on
load and compute in fp32 exactly as for fp32 inputs, so against the SAME engine call on the fp32 copies, with the same
anchors:
  * the loss is bit-identical;
  * the dense gradient has embed's dtype and equals the fp32 gradient rounded to nearest-even, zeros included;
  * the bank (queues, pointers, bf16 shadow) is bit-identical to the enqueue of the fp32 keys.
Eager calls draw their anchors through an injected permutation (the device RNG advances a global counter); graph steps
are built as twins with the same seed.  The functions take DEV and small shapes so that test_emu_mixed_precision.py runs
them on the emulated kernels."""
import pytest
import torch
import torch.nn as nn

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import _abi, bank as bank_mod, functional as Fn
from contrastiveseg_b200.synth import make_contrast_batch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda:0"
HALF = [torch.bfloat16, torch.float16]


def _sync():
    if str(DEV).startswith("cuda"):
        torch.cuda.synchronize()


def _perm(seed):
    """A fresh, seeded permutation source: two calls built with the same seed draw the same anchors."""
    g = torch.Generator().manual_seed(seed)
    return lambda n: torch.randperm(n, generator=g)


def _batch(B=2, D=256, h=32, w=32, K=7, seed=21, raw=False):
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=4, block=16, seed=seed)
    embed = data["embed_raw"] if raw else data["embed"]
    return embed.to(DEV), data["target"].to(DEV), data["seg"].to(DEV)


def _twin_banks(K, M, D, shadow):
    torch.manual_seed(0)
    a = cs.MemoryBank(K, M, D, with_shadow=shadow).to(DEV)
    b = cs.MemoryBank(K, M, D, with_shadow=shadow).to(DEV)
    b.load_state_dict(a.state_dict())
    if shadow:
        a.sync_shadow(); b.sync_shadow()
    return a, b


_BANK_NAMES = ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr")


def _assert_same_bank(a, b, where=""):
    for name in _BANK_NAMES:
        assert torch.equal(getattr(a, name), getattr(b, name)), (where, name)
    if a.shadow is not None or b.shadow is not None:
        assert torch.equal(a.shadow, b.shadow), where


def _assert_rounded(g_half, g32, dtype):
    """The half gradient is the fp32 gradient rounded once (what autograd's cast of an fp32 gradient gives)."""
    assert g_half.dtype == dtype and g32.dtype == torch.float32
    assert torch.equal(g_half, g32.to(dtype))


def _eager(embed, tgt, *, seg=None, predict=None, bank=None, precision="fp32", normalize=False, K=7, ms=128, mv=8):
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, num_classes=K,
                              precision=precision, normalize=normalize, perm_fn=_perm(7))
    kw = {}
    if bank is not None:
        kw = dict(segment_queue=bank.segment_queue, pixel_queue=bank.pixel_queue, bank_shadow=bank.shadow)
    e = embed.detach().clone().requires_grad_(True)
    loss = cs.pixel_contrast_loss(e, tgt, seg=seg, predict=predict, options=opts, **kw)
    ws = Fn.last_workspace(e.device)
    loss.backward()
    _sync()
    return loss.detach(), e.grad, ws.anchor_meta.clone()


# ------------------------------------------------------------------------------------------------------------------
# eager loss
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", [False, True], ids=["self", "bank"])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_eager_half_embed_matches_the_fp32_copy(dtype, precision, normalize, mem, B=2, h=32, w=32, ms=128, mv=8):
    K, D, M = 7, 256, 48
    embed, tgt, seg = _batch(B=B, h=h, w=w, K=K, raw=normalize)
    if normalize:
        embed = embed * 3.0                                      # raw projection: the engine normalises the samples
    e_half = embed.to(dtype)
    bank = None
    if mem:
        bank = cs.MemoryBank(K, M, D, with_shadow=(precision == "bf16")).to(DEV)
        if precision == "bf16":
            bank.sync_shadow()
    kw = dict(bank=bank, precision=precision, normalize=normalize, K=K, ms=ms, mv=mv)
    l_h, g_h, meta_h = _eager(e_half, tgt, seg=seg.to(dtype), **kw)
    l_f, g_f, meta_f = _eager(e_half.float(), tgt, seg=seg.to(dtype).float(), **kw)
    assert torch.equal(meta_h, meta_f)                           # same anchors
    assert torch.equal(l_h, l_f) and torch.isfinite(l_f)
    _assert_rounded(g_h, g_f, dtype)
    assert g_f.abs().sum() > 0


@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_half_seg_with_fp32_embed_and_predict_in_place_of_seg(dtype, B=2, h=32, w=32):
    K = 7
    embed, tgt, seg = _batch(B=B, h=h, w=w, K=K)
    seg_h = seg.to(dtype)
    l_h, g_h, m_h = _eager(embed, tgt, seg=seg_h, K=K)           # half logits: argmax of the converted values
    l_f, g_f, m_f = _eager(embed, tgt, seg=seg_h.float(), K=K)
    assert torch.equal(m_h, m_f) and torch.equal(l_h, l_f) and torch.equal(g_h, g_f)
    pred = seg_h.float().argmax(1)
    e_half = embed.to(dtype)
    l_h, g_h, m_h = _eager(e_half, tgt, predict=pred, K=K)
    l_f, g_f, m_f = _eager(e_half.float(), tgt, predict=pred, K=K)
    assert torch.equal(m_h, m_f) and torch.equal(l_h, l_f)
    _assert_rounded(g_h, g_f, dtype)


def test_fp32_call_after_a_half_call_on_the_same_workspace(B=2, h=32, w=32):
    """The step descriptor is cached per geometry: the dtype fields are set on every call."""
    K = 7
    embed, tgt, seg = _batch(B=B, h=h, w=w, K=K)
    l0, g0, _ = _eager(embed, tgt, seg=seg, K=K)
    _eager(embed.to(torch.bfloat16), tgt, seg=seg.to(torch.float16), K=K)
    assert Fn.last_workspace(embed.device).desc.embed_dtype == _abi.DT_BF16
    l1, g1, _ = _eager(embed, tgt, seg=seg, K=K)
    d = Fn.last_workspace(embed.device).desc
    assert d.embed_dtype == _abi.DT_F32 and d.seg_dtype == _abi.DT_F32
    assert torch.equal(l0, l1) and torch.equal(g0, g1)


# ------------------------------------------------------------------------------------------------------------------
# captured step
# ------------------------------------------------------------------------------------------------------------------
def _twin_steps(dtype, capture, *, fused=None, sparse_reset=False, precision="bf16", B=2, h=32, w=32, ms=128, mv=8,
                seg_dtype=None):
    K = 7
    embed, tgt, seg = _batch(B=B, h=h, w=w, K=K, seed=33)
    e_half = embed.to(dtype)
    s_half = seg.to(seg_dtype or dtype)
    opts = cs.ContrastOptions(temperature=0.1, base_temperature=0.07, max_samples=ms, max_views=mv, seed=5,
                              precision=precision, num_classes=K)
    kw = dict(options=opts, capture=capture, fused=fused, sparse_reset=sparse_reset, grad_scale=0.5)
    st_h = cs.GraphedContrastStep(e_half, tgt, seg=s_half, **kw)
    st_f = cs.GraphedContrastStep(e_half.float(), tgt, seg=s_half.float(), **kw)
    return st_h, st_f


def _replay_twins(st_h, st_f, dtype, replays=3):
    metas = []
    for r in range(replays):
        l_h, g_h = st_h.replay()
        l_f, g_f = st_f.replay()
        _sync()
        assert torch.equal(st_h.ws.anchor_meta, st_f.ws.anchor_meta), r
        metas.append(st_h.ws.anchor_meta.clone())
        assert torch.equal(l_h, l_f), r
        _assert_rounded(g_h, g_f, dtype)
        assert g_f.abs().sum() > 0
    assert not torch.equal(metas[0], metas[1])                  # fresh anchors per replay


@pytest.mark.parametrize("capture", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_fused_step_with_full_fill(dtype, capture, B=2, h=32, w=32):
    st_h, st_f = _twin_steps(dtype, capture, B=B, h=h, w=w)
    assert st_h.fused and st_f.fused and st_h.grad.dtype == dtype
    _replay_twins(st_h, st_f, dtype)


@pytest.mark.parametrize("capture", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_fused_step_with_sparse_reset(dtype, capture, B=2, h=32, w=32):
    """Every replay clears the previous replay's half-precision entries: at least 3 replays."""
    st_h, st_f = _twin_steps(dtype, capture, sparse_reset=True, B=B, h=h, w=w)
    assert st_h.sparse_reset
    _replay_twins(st_h, st_f, dtype, replays=4)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("capture", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_streaming_step(dtype, capture, precision, B=2, h=32, w=32):
    st_h, st_f = _twin_steps(dtype, capture, fused=False, precision=precision, B=B, h=h, w=w,
                             seg_dtype=torch.float16 if dtype == torch.bfloat16 else torch.bfloat16)
    assert not st_h.fused
    _replay_twins(st_h, st_f, dtype)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("capture", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_bank_step_with_enqueue_from_half_keys(dtype, capture, precision, B=2, h=32, w=32):
    K, D, M = 7, 256, 48
    embed, tgt, seg = _batch(B=B, h=h, w=w, K=K)
    e_half = embed.to(dtype)
    shadow = precision == "bf16"
    bank_h, bank_f = _twin_banks(K, M, D, shadow)
    opts = cs.ContrastOptions(temperature=0.07, base_temperature=0.07, max_samples=128, max_views=8, seed=5,
                              precision=precision, num_classes=K)
    steps = []
    for bank, e in ((bank_h, e_half), (bank_f, e_half.float())):
        steps.append(cs.GraphedContrastStep(e, tgt, seg=seg, segment_queue=bank.segment_queue,
                                            pixel_queue=bank.pixel_queue, bank_shadow=bank.shadow, options=opts,
                                            capture=capture,
                                            enqueue=dict(bank=bank, network_stride=4, pixel_update_freq=5, seed=3)))
    assert steps[0].enq["keys"].dtype == dtype
    _assert_same_bank(bank_h, bank_f, "after capture")
    start = bank_h.pixel_queue_ptr.clone()
    for r in range(3):
        l_h, g_h = steps[0].replay()
        l_f, g_f = steps[1].replay()
        _sync()
        assert torch.equal(l_h, l_f), r
        _assert_rounded(g_h, g_f, dtype)
        _assert_same_bank(bank_h, bank_f, r)
    assert not torch.equal(bank_h.pixel_queue_ptr, start)


@pytest.mark.parametrize("dtype", HALF, ids=["bf16", "fp16"])
def test_dequeue_and_enqueue_with_half_keys(dtype, B=2, h=32, w=32):
    K, D, M = 7, 256, 48
    embed, tgt, _ = _batch(B=B, h=h, w=w, K=K)
    keys = (embed * 1.7).to(dtype)                               # not unit rows: the row normalise is exercised
    for shadow in (False, True):
        bank_h, bank_f = _twin_banks(K, M, D, shadow)
        for r in range(2):
            for bank, k in ((bank_h, keys), (bank_f, keys.float())):
                bank_mod._enqueue_counter[0] = 10 + r            # same device-RNG draw for both
                bank.enqueue(k, tgt, network_stride=4, pixel_update_freq=5, seed=3)
            _sync()
            _assert_same_bank(bank_h, bank_f, (shadow, r))
        # the injected-permutation path takes the same entry point
        for bank, k in ((bank_h, keys), (bank_f, keys.float())):
            bank.enqueue(k, tgt, network_stride=4, pixel_update_freq=5, perm_fn=_perm(9))
        _sync()
        _assert_same_bank(bank_h, bank_f, (shadow, "perm"))


# ------------------------------------------------------------------------------------------------------------------
# end to end under autocast
# ------------------------------------------------------------------------------------------------------------------
class _StandIn(nn.Module):
    def __init__(self, K, D):
        super().__init__()
        self.body = nn.Conv2d(3, 32, 3, padding=1)
        self.cls = nn.Conv2d(32, K, 1)
        self.proj = nn.Conv2d(32, D, 1)

    def forward(self, x):
        f = torch.relu(self.body(x))
        return {"seg": self.cls(f), "embed": self.proj(f)}


def _ulp_close(a, b32, dtype):
    """|a - round(b32)| within one unit in the last place of the half dtype."""
    b = b32.to(dtype).float()
    a = a.float()
    eps = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10
    return bool(((a - b).abs() <= b.abs() * eps + 1e-30).all())


def test_trainer_hook_with_bank_under_autocast(B=2, h=32, w=32, dtype=torch.bfloat16):
    K, D, M = 5, 256, 24
    torch.manual_seed(1)
    model = _StandIn(K, D).to(DEV)
    x = torch.randn(B, 3, h, w, device=DEV)
    tgt = _batch(B=B, h=h, w=w, K=K, seed=41)[1]
    cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": 4},
                       "loss": {"loss_type": "mem_contrast_ce_loss", "params": {"ce_ignore_index": -1}},
                       "contrast": {"temperature": 0.1, "base_temperature": 0.07, "max_samples": 128, "max_views": 8,
                                    "loss_weight": 0.1, "use_rmi": False, "use_lovasz": False, "warmup_iters": 0,
                                    "with_memory": True, "memory_size": M, "pixel_update_freq": 5}})
    device_type = str(DEV).split(":")[0]
    with torch.autocast(device_type, dtype=dtype):
        out = model(x)
    assert out["seg"].dtype == dtype and out["embed"].dtype == dtype
    bank_h, bank_f = _twin_banks(K, M, D, False)
    results = []
    for bank, cast in ((bank_h, lambda t: t), (bank_f, lambda t: t.float())):
        seg = cast(out["seg"].detach()).requires_grad_(True)
        embed = cast(out["embed"].detach()).requires_grad_(True)
        hook = cs.ContrastTrainerHook(cfg, bank)
        Fn._step_counter[0] = 0
        bank_mod._enqueue_counter[0] = 0
        with torch.autocast(device_type, dtype=dtype):
            loss = hook.loss_step({"seg": seg, "embed": embed, "key": embed.detach(), "lb_key": tgt}, tgt, iters=1)
        loss.backward()
        _sync()
        results.append((loss.detach(), seg.grad, embed.grad))
    (l_h, gs_h, ge_h), (l_f, gs_f, ge_f) = results
    assert torch.equal(l_h, l_f) and torch.isfinite(l_f)
    _assert_rounded(ge_h, ge_f, dtype)
    assert gs_h.dtype == dtype and _ulp_close(gs_h, gs_f, dtype)    # seg CE: fp32 atomics, 1-2 ulp before rounding
    _assert_same_bank(bank_h, bank_f, "hook")


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def test_refusals(B=2, h=32, w=32):
    K = 7
    embed, tgt, seg = _batch(B=B, h=h, w=w, K=K)
    opts = cs.ContrastOptions(max_samples=128, max_views=8, num_classes=K)
    with pytest.raises(_abi.PclError):
        cs.pixel_contrast_loss(embed.double(), tgt, seg=seg, options=opts)
    topk = cs.ContrastOptions(max_samples=128, max_views=8, num_classes=K, topk_negatives=5)
    for dtype in HALF:
        with pytest.raises(_abi.PclError):
            cs.pixel_contrast_loss(embed.to(dtype), tgt, seg=seg, options=topk)
        with pytest.raises(_abi.PclError):
            cs.GraphedContrastStep(embed.to(dtype), tgt, seg=seg, options=topk, capture=False)
        nc = embed.to(dtype).transpose(2, 3)                     # non-contiguous: a graph cannot read a converted copy
        with pytest.raises(_abi.PclError):
            cs.GraphedContrastStep(nc, tgt, seg=seg.transpose(2, 3).contiguous(), options=opts, capture=False)
        with pytest.raises(_abi.PclError):
            cs.GraphedContrastStep(embed, tgt, seg=seg.to(dtype).transpose(2, 3), options=opts, capture=False)
    with pytest.raises(_abi.PclError):
        cs.GraphedContrastStep(embed.double(), tgt, seg=seg, options=opts, capture=False)
