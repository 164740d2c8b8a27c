"""Full-size parity on the hardware (VERDICT r1 #6 / weak #8): the tensor (bf16 wgmma) and the exact (fp32 SIMT) sweeps
at the contrast-set sizes of BASELINE configs[2] (K=19, M=5000: N = 190 000) and configs[3] (K=171, M=5000: N = 1.71 M,
1.75 GB bank + 0.88 GB shadow) against a column-chunked float64 closed form (tests/helpers.bank_infonce_chunked, plain
torch ops; itself pinned to oracle.ref_port.infonce_closed_form in tests/test_host_logic.py).  What changes at these
sizes and is exercised here: int64 column arithmetic, the analytic zero tail (tail_count = 10 000), the persistent
walk's partial-slot sizing, class-0 anchors, the Q1 diagonal inside the class-1 block.
Also: the bank's checkpoint format round trip (§8f row 3) and BASELINE's memory-bank step through the graphed API.

Tolerances: exact path loss 2e-6 rel / gradient 1e-5 max|g|; tensor path loss 1e-4 rel (north_star bar; operands
rounded to bf16) / gradient 4e-3 max|g|, 2e-3 relative Frobenius (bf16 operands and bf16 gradient tile)."""
import pytest
import torch

import contrastiveseg_b200 as cs
from contrastiveseg_b200 import functional as Fn
from contrastiveseg_b200.synth import make_bank, make_contrast_batch
from helpers import bank_infonce_chunked, rel_err

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda:0"


def _run_module(precision, K, M, B, h, w, stride, block, himg=None, wimg=None, max_views=100, seed=31):
    D = 256
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=stride, block=block, seed=seed, himg=himg,
                               wimg=wimg)
    bank = make_bank(K, M, D, seed + 1)
    segq, pixq = bank["segment_queue"].to(DEV), bank["pixel_queue"].to(DEV)
    cfg = cs.Configer({"data": {"num_classes": K}, "network": {"stride": stride},
                       "loss": {"params": {"ce_ignore_index": -1}},
                       "contrast": {"temperature": 0.07, "base_temperature": 0.07, "max_samples": 1024,
                                    "max_views": max_views, "loss_weight": 0.1, "precision": precision, "seed": 7}})
    crit = cs.PixelContrastLoss(cfg)
    embed = data["embed"].to(DEV).requires_grad_(True)
    loss = crit(embed, data["target"].to(DEV), seg=data["seg"].to(DEV), queue=(segq, pixq))
    ws = Fn.last_workspace(embed.device)
    loss.backward()
    torch.cuda.synchronize()
    A = int(ws.plan[2].item())
    ms = ws.geom.max_samples
    meta = ws.anchor_meta.view(4, ms)[:, :A].long()
    pix, img, cls, diag = meta[0], meta[1], meta[2], meta[3]
    anchors = embed.detach().permute(0, 2, 3, 1).reshape(B, h * w, D)[img, pix]          # rows in the engine's sorted order
    assert torch.equal(anchors, ws.anchors_f32[:A])                                       # the gather is exact
    ref = bank_infonce_chunked(anchors, cls, diag, segq, pixq, 0.07, 0.07, chunk=65536)
    g_rows = embed.grad.permute(0, 2, 3, 1).reshape(B, h * w, D)[img, pix].double()
    # everything outside the sampled pixels is exactly zero
    assert int((embed.grad != 0).sum().item()) <= A * D
    return loss.item(), g_rows, ref, A, cls


def _check(precision, loss, g_rows, ref):
    tol_l, tol_g = (2e-6, 1e-5) if precision == "fp32" else (1e-4, 4e-3)
    assert rel_err(loss, ref["loss"].item()) < tol_l, (loss, ref["loss"].item())
    gmax = ref["dA"].abs().max().item()
    assert (g_rows - ref["dA"]).abs().max().item() <= tol_g * gmax
    if precision == "bf16":
        assert ((g_rows - ref["dA"]).norm() / ref["dA"].norm()).item() < 2e-3


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_configs2_bank_190k_columns_a1024(precision):
    """BASELINE configs[2] heavy variant: one image per rank, K=19, M=5000 (N = 190 000 incl. the 10 000-row zero
    tail), max_views=100 -> A ~ 1000 anchors."""
    loss, g_rows, ref, A, cls = _run_module(precision, K=19, M=5000, B=1, h=128, w=256, stride=4, block=32)
    assert A >= 512 and int((cls == 0).sum()) > 0 and int((cls == 1).sum()) > 0      # class-0 (Q3) and class-1 (Q1) rows
    _check(precision, loss, g_rows, ref)


def test_configs2_reference_config_max_views_1():
    """configs[2] as the reference config has it (max_views=1 -> A = TC <= 19 anchors per rank; HBM-bound bank read)."""
    loss, g_rows, ref, A, cls = _run_module("bf16", K=19, M=5000, B=1, h=128, w=256, stride=4, block=32, max_views=1)
    assert 1 <= A <= 19
    _check("bf16", loss, g_rows, ref)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_configs3_bank_1_71m_columns_k171(precision):
    """BASELINE configs[3]: 171 classes, M=5000 -> N = 1.71 M columns (bank 1.75 GB fp32 + 0.88 GB bf16 shadow),
    520x520 -> 66x66 embedding (non-divisible nearest interpolation), two images per rank."""
    loss, g_rows, ref, A, cls = _run_module(precision, K=171, M=5000, B=2, h=66, w=66, stride=8, block=40, himg=520,
                                            wimg=520, max_views=10)
    assert A >= 256
    _check(precision, loss, g_rows, ref)


def test_bank_checkpoint_round_trip_on_the_gpu():
    """§8f row 3: a reference-shaped state_dict (the four HRNet_W48_MEM buffers, lib/models/nets/hrnet.py:165-171; the
    engine's bf16 shadow is NOT part of it) -> load_state_dict -> sync_shadow -> the tensor-path loss equals the loss on
    the bank the checkpoint came from, bit for bit; enqueue afterwards keeps shadow == bf16(queues)."""
    K, M, D = 7, 64, 256
    data = make_contrast_batch(B=2, D=D, h=32, w=32, num_classes=K, img_stride=4, block=16, seed=3)
    embed, tgt, seg = data["embed"].to(DEV), data["target"].to(DEV), data["seg"].to(DEV)
    src = cs.MemoryBank(K, M, D, with_shadow=True).to(DEV)
    src.enqueue(embed, tgt, network_stride=4, pixel_update_freq=6, seed=1)          # pointers != 0 in the checkpoint
    sd = {k: v.detach().cpu().clone() for k, v in src.state_dict().items()}
    assert sorted(sd) == ["pixel_queue", "pixel_queue_ptr", "segment_queue", "segment_queue_ptr"]
    assert sd["segment_queue"].shape == (K, M, D) and sd["pixel_queue_ptr"].dtype == torch.int64
    dst = cs.MemoryBank(K, M, D, with_shadow=True).to(DEV)
    dst.load_state_dict(sd)
    dst.sync_shadow()
    assert torch.equal(dst.shadow, src.shadow)
    opts = cs.ContrastOptions(temperature=0.07, base_temperature=0.07, max_samples=128, max_views=8, seed=5,
                              precision="bf16", num_classes=K)
    outs = []
    for bank in (src, dst):
        Fn._step_counter[0] = 0
        e = embed.clone().requires_grad_(True)
        l = cs.pixel_contrast_loss(e, tgt, seg=seg, segment_queue=bank.segment_queue, pixel_queue=bank.pixel_queue,
                                   bank_shadow=bank.shadow, options=opts)
        l.backward()
        outs.append((l.detach().clone(), e.grad.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    from contrastiveseg_b200 import bank as bank_mod
    for bank in (src, dst):
        bank_mod._enqueue_counter[0] = 100
        bank.enqueue(embed, tgt, network_stride=4, pixel_update_freq=6, seed=1)
    for name in ("segment_queue", "pixel_queue", "segment_queue_ptr", "pixel_queue_ptr"):
        assert torch.equal(getattr(src, name), getattr(dst, name)), name
    rebuilt = dst.shadow.clone()
    dst.sync_shadow()
    assert torch.equal(rebuilt, dst.shadow)                                            # maintained shadow == rebuild
