"""The CPU port against the unmodified reference on random seeds: the reference's losses, gradients, bank states and
randperm draws are stored under tests/golden/ref_*.npz (tests/golden/make_golden.py random); the inputs are regenerated
from the same seeds by contrastiveseg_b200.synth."""
import pytest
import torch

from oracle import ref_port as P
from contrastiveseg_b200.synth import make_bank, make_contrast_batch
from helpers import load_golden, rel_err, unpack_perms


@pytest.mark.parametrize("seed", [31, 32, 33])
@pytest.mark.parametrize("mem", [False, True])
def test_loss_random_seeds(seed, mem):
    g = load_golden(f"ref_seed{seed}_{'mem' if mem else 'nomem'}")
    K, D = 6, 32
    data = make_contrast_batch(B=3, D=D, h=20, w=24, num_classes=K, img_stride=2, block=6, seed=seed, boost=1.5)
    predict = data["seg"].argmax(1)
    queue = None
    if mem:
        bank = make_bank(K, 15, D, seed)
        queue = torch.cat((bank["segment_queue"], bank["pixel_queue"]), 1)
    replay = P.PermReplay(unpack_perms(g["perm_flat"], g["perm_lens"]))
    e2 = data["embed"].clone().requires_grad_(True)
    l2 = P.pixel_contrast_loss(e2, data["target"], predict, temperature=0.1, base_temperature=0.07, max_samples=50,
                               max_views=7, queue=queue, perm_fn=replay)
    l2.backward()
    assert replay.pos == len(replay.draws)
    assert rel_err(l2.item(), float(g["loss"])) < 2e-6
    assert torch.allclose(e2.grad, torch.from_numpy(g["grad_embed"]), rtol=1e-4, atol=1e-9)


def test_enqueue_random():
    g = load_golden("ref_enqueue_random")
    K, D, M, Fq = 5, 16, 6, 4
    bank = make_bank(K, M, D, 3)
    b = [bank[k].clone() for k in ("segment_queue", "segment_queue_ptr", "pixel_queue", "pixel_queue_ptr")]
    for s in range(5):
        data = make_contrast_batch(B=2, D=D, h=12, w=12, num_classes=K, img_stride=2, block=6, seed=50 + s)
        P.dequeue_and_enqueue(data["embed"], data["target"], *b, network_stride=2, memory_size=M,
                              pixel_update_freq=Fq, perm_fn=P.PermReplay(unpack_perms(g[f"perm_flat{s}"], g[f"perm_lens{s}"])))
        for k, y in zip(("sq", "sp", "pq", "pp"), b):
            assert torch.allclose(torch.from_numpy(g[f"{k}{s + 1}"]).float(), y.float(), atol=1e-6)
