"""Generate the Lovasz golden vectors (tests/golden/lovasz_*.npz) by running the UNMODIFIED reference on CPU.

    python tests/golden/make_golden_lovasz.py

FSCELOVASZLoss (lib/loss/loss_helper.py:77-124) at three geometries (identity, integer and non-integer up-sampling),
with ignored pixels and one absent class, and the memory wrapper (lib/loss/loss_contrast_mem.py ContrastCELoss with
contrast.use_lovasz) with a bank and its randperm draws recorded.  The reference sorts without stable=True, so the
inputs of the loss cases are checked to have no exact tie in the errors of a class: their gradients are then
unambiguous.  The wrapper's label map is too large to avoid fp32 ties by chance; its golden pins the loss, which does not
depend on the tie order.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle.ref_loader import DictConfiger, load_reference, patched_randperm  # noqa: E402
from oracle.ref_port import PermRecorder  # noqa: E402
from contrastiveseg_b200.synth import make_bank, make_contrast_batch  # noqa: E402

# name, B, K, h, w, H, W
CASES = [("lovasz_identity", 2, 5, 12, 14, 12, 14),
         ("lovasz_up4", 2, 6, 9, 11, 33, 41),
         ("lovasz_nonint", 1, 7, 7, 9, 26, 31)]


def has_ties(up, target, ignore_index):
    p = torch.softmax(up, 1).permute(0, 2, 3, 1).reshape(-1, up.shape[1])
    t = target.reshape(-1)
    v = t != ignore_index
    return any(torch.unique(e).numel() != e.numel()
               for e in (((t[v] == c).float() - p[v, c]).abs() for c in range(up.shape[1])))


def inputs(B, K, h, w, H, W, seed):
    """Logits and labels (class K-1 absent, 15% ignored) of the first seed from `seed` on without an exact tie."""
    while True:
        g = torch.Generator().manual_seed(seed)
        seg = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * 4
        target = torch.randint(0, K - 1, (B, H, W), generator=g)
        target[torch.rand(B, H, W, generator=g) < 0.15] = -1
        up = F.interpolate(seg, size=(H, W), mode="bilinear", align_corners=True)
        if not has_ties(up, target, -1):
            return seg, target
        seed += 1000


def loss_case(name, B, K, h, w, H, W, seed):
    load_reference()
    import lib.loss.loss_helper as lh
    seg, target = inputs(B, K, h, w, H, W, seed)
    cfg = DictConfiger({"loss": {"params": {"ce_ignore_index": -1, "ce_reduction": "mean"}}})
    x = seg.clone().requires_grad_(True)
    up = F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)
    loss = lh.FSCELOVASZLoss(cfg)(up, target.clone())
    loss.backward()
    ce = F.cross_entropy(up.detach(), target, ignore_index=-1)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), seg=seg.numpy(), target=target.numpy(),
                        loss=np.float32(loss.item()), lovasz=np.float32(loss.item() - ce.item()),
                        grad_seg=x.grad.numpy())
    print(f"{name}: loss={loss.item():.7f}")


def wrapper_case(name, seed):
    ref = load_reference()
    B, D, h, w, K, stride = 2, 32, 16, 20, 5, 4
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=stride, block=8, seed=seed)
    bank = make_bank(K, 10, D, seed)
    d = {"contrast": {"temperature": 0.1, "base_temperature": 0.07, "max_samples": 48, "max_views": 5,
                      "loss_weight": 0.1, "use_rmi": False, "use_lovasz": True, "proj_dim": 256, "stride": 8,
                      "warmup_iters": 0, "with_memory": True, "memory_size": 10, "pixel_update_freq": 3},
         "loss": {"params": {"ce_ignore_index": -1, "ce_reduction": "mean"}},
         "network": {"stride": 8}}
    cfg = DictConfiger(d)
    g = torch.Generator().manual_seed(seed + 2)
    seg0 = data["seg"] + 0.05 * torch.randn(data["seg"].shape, generator=g)     # the synthetic logits are blocky: ties
    seg = seg0.clone().requires_grad_(True)
    embed = data["embed"].clone().requires_grad_(True)
    target = data["target"].clone()
    crit = ref.mem.ContrastCELoss(cfg)
    preds = {"seg": seg, "embed": embed, "segment_queue": bank["segment_queue"], "pixel_queue": bank["pixel_queue"]}
    rec = PermRecorder(torch.Generator().manual_seed(seed + 1))
    with patched_randperm(rec):
        loss = crit(preds, target, with_embed=True)
    loss.backward()
    lens = np.array([len(x) for x in rec.draws], dtype=np.int64)
    flat = np.concatenate([x.numpy() for x in rec.draws]).astype(np.int64) if rec.draws else np.zeros(0, np.int64)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), seg=seg0.numpy(), embed=data["embed"].numpy(),
                        target=data["target"].numpy(), segment_queue=bank["segment_queue"].numpy(),
                        pixel_queue=bank["pixel_queue"].numpy(), perm_flat=flat, perm_lens=lens,
                        loss=np.float32(loss.item()), grad_seg=seg.grad.numpy(), grad_embed=embed.grad.numpy())
    print(f"{name}: loss={loss.item():.7f}")


if __name__ == "__main__":
    for i, c in enumerate(CASES):
        loss_case(*c, seed=60 + i)
    wrapper_case("lovasz_wrapper_mem", seed=71)
