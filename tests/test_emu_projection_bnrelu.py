"""BatchNorm + ReLU fused into the projection head's last-conv GEMM on CPU: the tests of test_gpu_projection_bnrelu.py
at small shapes on the emulated kernels (DEV = "cpu"), once more under a shuffled thread schedule with poisoned
allocations, and SyncBatchNorm over two gloo ranks against one BatchNorm on the concatenated batch."""
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import emu_harness
import test_gpu_projection as P
import test_gpu_projection_bnrelu as PB

BF = torch.bfloat16
# Cin below 64 with a pixel tail; several K-blocks and dgrad passes; Cin = 256 (the bias column in its own wgrad tile)
SMALL = [(2, 40, 6, 7), (1, 300, 12, 13), (2, 256, 4, 9)]


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    monkeypatch.setattr(P, "DEV", "cpu")
    monkeypatch.setattr(PB, "DEV", "cpu")
    return lib


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", SMALL)
def test_matches_fp64_on_emulation(emu, shape, mode, dtype):
    PB.test_matches_fp64(shape, mode, dtype)


def test_batch_statistics_and_counter_on_emulation(emu):
    PB.test_batch_statistics_and_counter_match_fp64((2, 40, 6, 7))


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_head_matches_the_torch_bn_relu_head_on_emulation(emu, mode, dtype):
    PB.test_head_matches_the_torch_bn_relu_head(mode, dtype, shape=(2, 40, 6, 7))


def test_large_mean_channel_on_emulation(emu, monkeypatch):
    monkeypatch.setattr(PB, "CANCEL_SHAPE", (2, 40, 6, 7))
    PB.test_large_mean_channel_does_not_cancel()


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_bit_reproducible_on_emulation(emu, mode):
    PB.test_bit_reproducible(mode, shape=(2, 40, 6, 7))


def test_refusals_on_emulation(emu):
    PB.test_refusals()


def test_results_do_not_depend_on_the_schedule_or_uninitialised_memory():
    """The emulated cases again with a shuffled thread / block order and every torch.empty buffer poisoned (NaN): a
    missing barrier or a read of memory the kernels never wrote changes the result."""
    env = dict(os.environ, PCL_EMU_SCHED="random:1", PCL_EMU_POISON="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "on_emulation"], env=env, capture_output=True, text=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout


# ------------------------------------------------------------------------------------------------------------------
# SyncBatchNorm over two gloo ranks on the emulated kernels
# ------------------------------------------------------------------------------------------------------------------
SYNC_SHAPES = [(2, 40, 6, 7), (1, 40, 6, 7)]            # rank 0, rank 1: different counts


def _sync_inputs(rank):
    y, bn, w, b, gzn = PB._inputs(SYNC_SHAPES[0], "train", seed=21)       # bn, w, b shared by the ranks
    g = torch.Generator().manual_seed(30 + rank)
    shape = SYNC_SHAPES[rank]
    y = torch.randn(shape, generator=g) * 0.8 + 0.4
    gzn = torch.randn((shape[0], 256) + shape[2:], generator=g)
    return y, bn, w, b, gzn


def _sync_worker(rank, world, port, out_dir):
    import torch.nn as nn
    monkey = pytest.MonkeyPatch()
    emu_harness.use_emulation(monkey)
    monkey.setattr(PB, "DEV", "cpu")
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    y, bn, w, b, gzn = _sync_inputs(rank)
    sbn = nn.SyncBatchNorm(bn.num_features)
    sbn.load_state_dict(bn.state_dict())
    sbn.train()
    got = PB._fused(y, sbn, w, b, gzn)
    got.update({k: getattr(sbn, k).clone() for k in ("running_mean", "running_var", "num_batches_tracked")})
    torch.save(got, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_sync_batchnorm_two_ranks_matches_one_batchnorm_on_the_concatenated_batch(tmp_path, monkeypatch):
    monkeypatch.setattr(PB, "DEV", "cpu")
    port = _free_port()
    mp.spawn(_sync_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r = [torch.load(tmp_path / f"r{k}.pt") for k in range(2)]
    ins = [_sync_inputs(k) for k in range(2)]
    _, bn, w, b, _ = ins[0]
    # float64 reference: one BatchNorm over the concatenated batch
    y64 = torch.cat([i[0] for i in ins]).double().requires_grad_(True)
    gzn = torch.cat([i[4] for i in ins]).double()
    g64 = bn.weight.detach().double().requires_grad_(True)
    be64 = bn.bias.detach().double().requires_grad_(True)
    rm, rv = bn.running_mean.double().clone(), bn.running_var.double().clone()
    a = F.batch_norm(y64, rm, rv, g64, be64, True, bn.momentum, bn.eps)
    zn = F.normalize(F.conv2d(F.relu(a), w.double(), b.double()), p=2, dim=1)
    gy, ga = torch.autograd.grad(zn, (y64, a), gzn)
    xhat = (y64 - y64.mean((0, 2, 3), keepdim=True)) / torch.sqrt(y64.var((0, 2, 3), unbiased=False, keepdim=True)
                                                                   + bn.eps)
    n0 = SYNC_SHAPES[0][0]
    for k, sl in enumerate((slice(0, n0), slice(n0, None))):
        for name in ("running_mean", "running_var", "num_batches_tracked"):
            assert torch.equal(r[k][name], r[0][name]), name                 # identical on both ranks
        for name, ref in (("running_mean", rm), ("running_var", rv)):
            assert (r[k][name].double() - ref).abs().max() <= PB.STATS_REL * ref.abs().max(), name
        assert r[k]["num_batches_tracked"].item() == 1
        local = {"gy": gy[sl], "zn": zn[sl].detach(),
                 "gbeta": ga[sl].sum((0, 2, 3)), "ggamma": (ga[sl] * xhat[sl]).sum((0, 2, 3))}   # rank-local
        e = P.errors({n: r[k][n] for n in local}, local)
        for n in local:
            assert e[n][0] <= PB.MAXABS[n] and e[n][1] <= PB.FROB[n], (k, n, e)


def test_sync_batchnorm_on_one_rank_calls_no_collective(emu, monkeypatch):
    """Without a process group of more than one rank a SyncBatchNorm computes exactly what a BatchNorm2d computes, and
    no collective is called."""
    import torch.nn as nn

    def refuse(*a, **k):
        raise AssertionError("all_reduce called on one rank")
    monkeypatch.setattr(dist, "all_reduce", refuse)
    y, bn, w, b, gzn = PB._inputs((2, 40, 6, 7), "train", seed=22)
    sbn = nn.SyncBatchNorm(bn.num_features)
    sbn.load_state_dict(bn.state_dict())
    sbn.train()
    got_s, got_b = PB._fused(y, sbn, w, b, gzn), PB._fused(y, bn, w, b, gzn)
    for k in PB.NAMES:
        assert torch.equal(got_s[k], got_b[k]), k
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(sbn, k), getattr(bn, k)), k
