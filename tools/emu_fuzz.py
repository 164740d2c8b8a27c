"""Long-running differential fuzz of the SIMT kernel sources on the CPU emulator (see tests/emu_fuzz.py).

    python tools/emu_fuzz.py [rounds=5] [iterations per fuzzer and round=200] [seed offset=7]
"""
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pytest  # noqa: E402
import torch  # noqa: E402

import emu_fuzz  # noqa: E402
import emu_harness  # noqa: E402
import test_gpu_parity as G  # noqa: E402

if __name__ == "__main__":
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    base = int(sys.argv[3]) if len(sys.argv) > 3 else 7
    mp = pytest.MonkeyPatch()
    mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    emu_harness.use_emulation(mp)

    def criterion(seed, k):
        """fuzz_graphed_criterion with the criterion's launch sequence run eagerly (no CUDA graphs on a CPU) and the
        fused seg CE taken for CPU tensors; the patches are undone afterwards (the other fuzzers run unpatched)."""
        from contrastiveseg_b200 import graph_step, loss as loss_mod
        cp = pytest.MonkeyPatch()
        G_ = graph_step.GraphedContrastStep
        cp.setattr(G_, "_capture", lambda self, warmup: None)
        cp.setattr(G_, "_fork_zero_fill", lambda self: self._side_branch(0))
        cp.setattr(G_, "_join_zero_fill", lambda self: None)
        cp.setattr(loss_mod.ContrastCELoss, "_can_fuse", lambda self, ce, s: self.fused_seg_ce)
        try:
            return emu_fuzz.fuzz_graphed_criterion(seed, k, G._check_device_sampling)[0]
        finally:
            cp.undo()

    total = 0
    for r in range(rounds):
        for name, fn in (("loss", lambda s: emu_fuzz.fuzz_loss(s, n)), ("bank", lambda s: emu_fuzz.fuzz_bank(s, n)),
                         ("segce", lambda s: emu_fuzz.fuzz_segce(s, n)), ("topk", lambda s: emu_fuzz.fuzz_topk(s, n)),
                         ("devrng", lambda s: emu_fuzz.fuzz_device_sampling(s, n, G._check_device_sampling)),
                         ("tensor", lambda s: emu_fuzz.fuzz_tensor_path(s, max(1, n // 5))),
                         ("graph", lambda s: emu_fuzz.fuzz_graphed_step(s, max(1, n // 2),
                                                                        G._check_device_sampling)[0]),
                         ("criterion", lambda s: criterion(s, max(1, n // 4))),
                         ("hook", lambda s: emu_fuzz.fuzz_trainer_hook(s, max(1, n // 2))),
                         ("head", lambda s: emu_fuzz.fuzz_projection_head(s, max(1, n // 10))[0]),
                         ("wrappers", lambda s: emu_fuzz.fuzz_wrappers(s, n))):
            bad = fn(1000 * r + base)
            total += len(bad)
            print(f"round {r} {name}: {len(bad)} failures", flush=True)
            for b in bad[:10]:
                print("   ", b)
    sys.exit(1 if total else 0)
