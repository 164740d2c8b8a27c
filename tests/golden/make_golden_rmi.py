"""Generate the RMI golden vectors (tests/golden/rmi_*.npz) by running the UNMODIFIED reference on CPU.

    python tests/golden/make_golden_rmi.py

RMILoss (lib/loss/rmi_loss.py) at a few geometries and parameter sets, and the two contrast wrappers with
contrast.use_rmi (ContrastAuxCELoss -> FSAuxRMILoss, the memory wrapper -> FSRMILoss) with their randperm draws
recorded.  The reference casts its neighbour vectors with .type(torch.cuda.DoubleTensor); on CPU that name is pointed
at torch.DoubleTensor.  Its per-(image, class) float64 0.5 log det is recorded as well (rmi_bc), before the float32 cast.
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
from contrastiveseg_b200.synth import make_contrast_batch  # noqa: E402

torch.cuda.DoubleTensor = torch.DoubleTensor

# name, B, K, h, w, H, W, radius, pool way, stride, lambda_way
CASES = [("rmi_up4_r3_max", 2, 5, 9, 11, 33, 41, 3, 0, 3, 1),
         ("rmi_nonint_r2_avg", 2, 4, 7, 9, 26, 31, 2, 1, 2, 0),
         ("rmi_identity_r1", 1, 3, 12, 14, 12, 14, 1, 0, 1, 1),
         ("rmi_up3_r4_max_s4", 2, 3, 10, 12, 30, 36, 4, 0, 4, 1)]


def rmi_params(K, radius, way, stride, lambda_way):
    return {"use_sigmoid": True, "num_classes": K, "rmi_radius": radius, "rmi_pool_way": way, "rmi_pool_size": stride,
            "rmi_pool_stride": stride, "loss_weight_lambda": 0.5, "loss_weight": 1.0, "lambda_way": lambda_way}


class capture_logdet:
    """Records the float64 output of rmi_loss.log_det_by_cholesky (the reference's rmi_now is 0.5 times it)."""

    def __init__(self, mod):
        self.mod, self.out = mod, []

    def __enter__(self):
        self.orig = self.mod.log_det_by_cholesky

        def spy(m):
            r = self.orig(m)
            self.out.append(r.detach().clone())
            return r
        self.mod.log_det_by_cholesky = spy
        return self

    def __exit__(self, *exc):
        self.mod.log_det_by_cholesky = self.orig
        return False


def inputs(B, K, h, w, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    seg = (torch.rand(B, K, h, w, generator=g) * 2 - 1) * 6
    target = torch.randint(0, K, (B, H, W), generator=g)
    drop = torch.rand(B, H, W, generator=g) < 0.15
    kinds = torch.tensor([-1, 255, K])
    target[drop] = kinds[torch.randint(0, 3, (int(drop.sum()),), generator=g)]
    return seg, target


def loss_case(name, B, K, h, w, H, W, radius, way, stride, lambda_way, seed):
    load_reference()
    import lib.loss.rmi_loss as rmi_mod
    seg, target = inputs(B, K, h, w, H, W, seed)
    cfg = DictConfiger({"loss": {"params": rmi_params(K, radius, way, stride, lambda_way)}})
    x = seg.clone().requires_grad_(True)
    up = F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)
    with capture_logdet(rmi_mod) as cap:
        loss = rmi_mod.RMILoss(cfg)(up, target.clone())
    loss.backward()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), seg=seg.numpy(), target=target.numpy(),
                        loss=np.float32(loss.item()), grad_seg=x.grad.numpy(), rmi_bc=(0.5 * cap.out[0]).numpy(),
                        params=np.array([K, radius, way, stride, 0.5, lambda_way, 1.0]))
    print(f"{name}: loss={loss.item():.7f}")


def wrapper_case(name, mem, seed):
    ref = load_reference()
    B, D, h, w, K, stride = 2, 32, 16, 20, 5, 4
    data = make_contrast_batch(B=B, D=D, h=h, w=w, num_classes=K, img_stride=stride, block=8, seed=seed)
    d = {"contrast": {"temperature": 0.1, "base_temperature": 0.07, "max_samples": 48, "max_views": 5,
                      "loss_weight": 0.1, "use_rmi": True, "use_lovasz": False, "proj_dim": 256, "stride": 8,
                      "warmup_iters": 0},
         "loss": {"params": dict(rmi_params(K, 3, 0, 3, 1), ce_ignore_index=-1, ce_reduction="elementwise_mean")},
         "network": {"stride": 8, "loss_weights": {"seg_loss": 1.0, "aux_loss": 0.4}}}
    if mem:
        d["contrast"].update(with_memory=True, memory_size=10, pixel_update_freq=3)
    cfg = DictConfiger(d)
    g = torch.Generator().manual_seed(seed + 5)
    seg = data["seg"].clone().requires_grad_(True)
    seg_aux = (data["seg"] * 0.5 + torch.randn(data["seg"].shape, generator=g)).requires_grad_(True)
    embed = data["embed"].clone().requires_grad_(True)
    target = data["target"].clone()
    crit = ref.mem.ContrastCELoss(cfg) if mem else ref.nomem.ContrastAuxCELoss(cfg)
    preds = {"seg": seg, "embed": embed}
    if not mem:
        preds["seg_aux"] = seg_aux
    rec = PermRecorder(torch.Generator().manual_seed(seed + 1))
    with patched_randperm(rec):
        loss = crit(preds, target, with_embed=False)     # seg loss + 0 * contrast: the seg composition alone
    loss.backward()
    lens = np.array([len(x) for x in rec.draws], dtype=np.int64)
    flat = np.concatenate([x.numpy() for x in rec.draws]).astype(np.int64) if rec.draws else np.zeros(0, np.int64)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), seg=data["seg"].numpy(), seg_aux=seg_aux.detach().numpy(),
                        embed=data["embed"].numpy(), target=data["target"].numpy(), perm_flat=flat, perm_lens=lens,
                        loss=np.float32(loss.item()), grad_seg=seg.grad.numpy(),
                        grad_seg_aux=(seg_aux.grad.numpy() if not mem else np.zeros(0, np.float32)),
                        params=np.array([K, 3, 0, 3, 0.5, 1, 1.0, 1.0, 0.4, float(mem)]))
    print(f"{name}: loss={loss.item():.7f}")


if __name__ == "__main__":
    for i, c in enumerate(CASES):
        loss_case(*c, seed=40 + i)
    wrapper_case("rmi_wrapper_aux", mem=False, seed=51)
    wrapper_case("rmi_wrapper_mem", mem=True, seed=52)
