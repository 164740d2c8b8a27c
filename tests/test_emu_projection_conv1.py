"""The projection head's first 1x1 convolution on CPU: the tests of test_gpu_projection_conv1.py at small shapes on the
emulated kernels (DEV = "cpu"), once more under a shuffled thread schedule with poisoned allocations, SyncBatchNorm
over two gloo ranks against one BatchNorm on the concatenated batch, and the host wiring of fuse_conv1."""
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
import test_gpu_projection_conv1 as PC
from contrastiveseg_b200 import _abi

BF = torch.bfloat16
# C below 64 with a pixel tail; C not a multiple of 8 over two 256-channel bands, several K-blocks; C = 256 (one full
# band, the weight gradient's bias column in its own tile)
SMALL = [(2, 40, 6, 7), (1, 300, 5, 7), (2, 256, 4, 9)]


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    for m in (P, PB, PC):
        monkeypatch.setattr(m, "DEV", "cpu")
    return lib


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", SMALL)
def test_conv1_matches_fp64_on_emulation(emu, shape, dtype):
    PC.test_conv1_matches_fp64_on_bf16_operands(shape, dtype)
    PC.test_conv1_sums_match_fp64_sums_of_the_stored_y(shape, dtype)


def test_conv1_without_gx_on_emulation(emu):
    PC.test_conv1_without_gx_writes_the_same_weight_gradient((1, 40, 5, 7))


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", SMALL[:2])
def test_head_matches_fp64_on_emulation(emu, shape, mode, dtype):
    PC.test_head_matches_fp64(shape, mode, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "autocast"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_head_matches_the_torch_conv1_head_on_emulation(emu, mode, dtype):
    PC.test_head_matches_the_cudnn_conv1_head(mode, dtype, shape=(2, 40, 6, 7))


def test_autocast_equals_the_call_on_bf16_x_on_emulation(emu):
    PC.test_autocast_equals_the_call_on_bf16_x(shape=(2, 40, 6, 7))


def test_large_mean_through_b1_on_emulation(emu, monkeypatch):
    monkeypatch.setattr(PC, "CANCEL_SHAPE", (2, 40, 6, 7))
    PC.test_large_mean_through_b1_does_not_cancel()


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_bit_reproducible_on_emulation(emu, mode):
    PC.test_bit_reproducible(mode, shape=(2, 40, 6, 7))


def test_refusals_on_emulation(emu):
    PC.test_refusals()


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
# host wiring: which entry points the head calls, with which dtype codes
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if not name.startswith("pcl_proj"):
            return fn

        def rec(*a):
            self.calls.append((name, a))
            return fn(*a)
        return rec


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_head_calls_conv1_entry_points_only_with_fuse_conv1(emu, monkeypatch, dtype):
    rec = _Recorder(emu)
    monkeypatch.setattr(_abi, "load", lambda *a, **k: rec)
    x = torch.randn(2, 40, 6, 7)
    for fuse_conv1 in (False, True):
        rec.calls.clear()
        torch.manual_seed(0)
        head = PC.cs.ProjectionHead(40, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True,
                                    fuse_conv1=fuse_conv1)
        xx = x.clone().requires_grad_(True)
        with torch.autocast("cpu", dtype=BF, enabled=dtype == BF):     # bf16: conv1 hands over (or takes) bf16
            zn = head(xx)
        zn.float().sum().backward()
        names = [c[0] for c in rec.calls]
        conv1 = [c for c in rec.calls if c[0].startswith("pcl_proj_conv1")]
        if not fuse_conv1:
            assert not conv1 and "pcl_proj_bn_stats_dt" in names
            continue
        assert "pcl_proj_bn_stats_dt" not in names                  # the statistics come from conv1's epilogue
        assert [c[0] for c in conv1] == ["pcl_proj_conv1_workspace_bytes", "pcl_proj_conv1_workspace_bytes",
                                         "pcl_proj_conv1_pack", "pcl_proj_conv1_fwd_dt",
                                         "pcl_proj_conv1_workspace_bytes", "pcl_proj_conv1_bwd_dt"]
        code = _abi.DT_F32 if dtype == torch.float32 else _abi.DT_BF16
        for name, a in conv1:
            if name.endswith("_dt"):
                assert a[1] == code, name
        assert names.index("pcl_proj_conv1_fwd_dt") < names.index("pcl_proj_bn_finalize") < \
            names.index("pcl_proj_bn_fwd_dt") < names.index("pcl_proj_bn_bwd_dt") < \
            names.index("pcl_proj_bn_input_grad_dt") < names.index("pcl_proj_conv1_bwd_dt")


def test_x_without_grad_skips_the_data_gradient(emu, monkeypatch):
    rec = _Recorder(emu)
    monkeypatch.setattr(_abi, "load", lambda *a, **k: rec)
    torch.manual_seed(0)
    head = PC.cs.ProjectionHead(40, 256, "convmlp", bn_type="torchbn", fused=True, fuse_bn_relu=True, fuse_conv1=True)
    head(torch.randn(2, 40, 6, 7)).sum().backward()
    (bwd,) = [a for n, a in rec.calls if n == "pcl_proj_conv1_bwd_dt"]
    assert bwd[8] is None                                           # gx
    assert head.proj[0].weight.grad is not None and head.proj[0].bias.grad is not None


# ------------------------------------------------------------------------------------------------------------------
# SyncBatchNorm over two gloo ranks on the emulated kernels
# ------------------------------------------------------------------------------------------------------------------
SYNC_SHAPES = [(2, 40, 6, 7), (1, 40, 6, 7)]            # rank 0, rank 1: different counts


def _sync_inputs(rank):
    x, w1, b1, bn, w2, b2, gzn = PC._head_inputs(SYNC_SHAPES[0], "train", seed=21)    # weights shared by the ranks
    g = torch.Generator().manual_seed(30 + rank)
    shape = SYNC_SHAPES[rank]
    x = torch.randn(shape, generator=g) * 0.8 + 0.4
    gzn = torch.randn((shape[0], 256) + shape[2:], generator=g)
    return x, w1, b1, bn, w2, b2, gzn


def _sync_worker(rank, world, port, out_dir):
    import torch.nn as nn
    monkey = pytest.MonkeyPatch()
    emu_harness.use_emulation(monkey)
    monkey.setattr(PC, "DEV", "cpu")
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    x, w1, b1, bn, w2, b2, gzn = _sync_inputs(rank)
    sbn = nn.SyncBatchNorm(bn.num_features)
    sbn.load_state_dict(bn.state_dict())
    sbn.train()
    got = PC._head(x, w1, b1, sbn, w2, b2, gzn)
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
    monkeypatch.setattr(PC, "DEV", "cpu")
    port = _free_port()
    mp.spawn(_sync_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r = [torch.load(tmp_path / f"r{k}.pt") for k in range(2)]
    ins = [_sync_inputs(k) for k in range(2)]
    _, w1, b1, bn, w2, b2, _ = ins[0]
    # float64 reference: one BatchNorm over the concatenated batch, conv1 on its bf16 operands
    x64 = PC._r(torch.cat([i[0] for i in ins])).requires_grad_(True)
    gzn = torch.cat([i[6] for i in ins]).double()
    g64 = bn.weight.detach().double().requires_grad_(True)
    be64 = bn.bias.detach().double().requires_grad_(True)
    y = F.conv2d(x64, PC._r(w1), b1.double())
    y.register_hook(lambda g: g.to(BF).double())                 # g_y as the conv1 GEMMs take it
    rm, rv = bn.running_mean.double().clone(), bn.running_var.double().clone()
    a = F.batch_norm(y, rm, rv, g64, be64, True, bn.momentum, bn.eps)
    zn = F.normalize(F.conv2d(F.relu(a), w2.double(), b2.double()), p=2, dim=1)
    gx, ga = torch.autograd.grad(zn, (x64, a), gzn)
    yd = y.detach()
    xhat = (yd - yd.mean((0, 2, 3), keepdim=True)) / torch.sqrt(yd.var((0, 2, 3), unbiased=False, keepdim=True) + bn.eps)
    n0 = SYNC_SHAPES[0][0]
    for k, sl in enumerate((slice(0, n0), slice(n0, None))):
        for name in ("running_mean", "running_var", "num_batches_tracked"):
            assert torch.equal(r[k][name], r[0][name]), name                 # identical on both ranks
        for name, ref in (("running_mean", rm), ("running_var", rv)):
            assert (r[k][name].double() - ref).abs().max() <= PC.STATS_REL * ref.abs().max(), name
        assert r[k]["num_batches_tracked"].item() == 1
        local = {"gx": gx[sl], "zn": zn[sl].detach(),
                 "gbeta": ga[sl].sum((0, 2, 3)), "ggamma": (ga[sl] * xhat[sl]).sum((0, 2, 3))}   # rank-local
        e = P.errors({n: r[k][n] for n in local}, local)
        for n in local:
            assert e[n][0] <= PC.HEAD_MAXABS[n] and e[n][1] <= PC.HEAD_FROB[n], (k, n, e)
