"""The anchor-column hand-off of test_gpu_sparse_head.py at small shapes on the emulated kernels (DEV = "cpu"): the
columns against the dense gradient in every step mode, the head's column backward against float64 (train / eval, fp32 /
bf16, Cin 40 / 300 / 720 with pixel tails, with and without the first conv), the contrast wrappers end to end and the
fallbacks against the dense head, once more under a shuffled thread schedule with poisoned allocations, and
SyncBatchNorm over two gloo ranks against one BatchNorm on the concatenated batch."""
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

import emu_harness
import test_emu_projection_bnrelu as EB
import test_gpu_projection as P
import test_gpu_projection_bnrelu as PB
import test_gpu_projection_conv1 as PC
import test_gpu_sparse_head as S

BF = torch.bfloat16
SMALL = [(2, 40, 6, 7), (1, 300, 5, 9), (1, 720, 3, 5)]


@pytest.fixture
def emu(monkeypatch):
    lib = emu_harness.use_emulation(monkeypatch)
    for mod in (P, PB, PC, S):
        monkeypatch.setattr(mod, "DEV", "cpu")
    return lib


@pytest.mark.parametrize("mode", list(S.STEP_MODES))
def test_cols_equal_the_dense_gradient_on_emulation(emu, mode):
    S.check_cols_equal_dense(mode, D=256 if "tensor" in mode else 64, h=8, w=7, ms=48)


@pytest.mark.parametrize("mode", ["simt", "normalize"])
def test_rounded_cols_equal_the_bf16_dense_gradient_on_emulation(emu, mode):
    S.check_cols_equal_dense(mode, BF, D=64, h=8, w=7, ms=48)


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("shape", SMALL)
def test_head_cols_match_fp64_on_emulation(emu, shape, mode, dtype):
    S.check_head_cols(shape, mode, dtype, n=11, dead=3)


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_head_cols_with_conv1_match_fp64_on_emulation(emu, mode, dtype):
    S.check_head_cols_conv1((2, 40, 6, 7), mode, dtype, n=11, dead=3)


def test_head_cols_bit_reproducible_on_emulation(emu):
    S.check_head_cols_bit_reproducible()


@pytest.mark.parametrize("conv1", [False, True], ids=["bn_relu", "conv1"])
@pytest.mark.parametrize("wrapper", S.WRAPPERS)
def test_end_to_end_matches_the_dense_head_on_emulation(emu, wrapper, conv1):
    S.check_end_to_end(wrapper, conv1, Cin=40, h=8, w=7)


def test_trainer_hook_with_enqueue_on_emulation(emu):
    S.check_trainer_hook_with_enqueue(Cin=40, h=8, w=7)


@pytest.mark.parametrize("case", S.FALLBACKS)
def test_fallbacks_give_the_dense_result_on_emulation(emu, case):
    S.check_fallback(case, Cin=40, h=8, w=7)


def test_results_do_not_depend_on_the_schedule_or_uninitialised_memory():
    """The emulated head cases again with a shuffled thread / block order and every torch.empty buffer poisoned."""
    env = dict(os.environ, PCL_EMU_SCHED="random:1", PCL_EMU_POISON="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "head_cols and on_emulation"], env=env, capture_output=True, text=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout


# ------------------------------------------------------------------------------------------------------------------
# SyncBatchNorm over two gloo ranks on the emulated kernels
# ------------------------------------------------------------------------------------------------------------------
def _cols(rank):
    B, C, H, W = EB.SYNC_SHAPES[rank]
    return S._columns(B, H, W, 9, 2, 40 + rank)


def _sync_worker(rank, world, port, out_dir):
    import torch.nn as nn
    monkey = pytest.MonkeyPatch()
    emu_harness.use_emulation(monkey)
    for mod in (PB, S):
        monkey.setattr(mod, "DEV", "cpu")
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    y, bn, w, b, _ = EB._sync_inputs(rank)
    cols, col_pix, _ = _cols(rank)
    sbn = nn.SyncBatchNorm(bn.num_features)
    sbn.load_state_dict(bn.state_dict())
    sbn.train()
    yy = y.clone().requires_grad_(True)
    zn = S.cs.bn_relu_project_normalize(yy, sbn, w, b, sparse_grad=True)
    zn.backward(S._hand_off(zn, cols, col_pix))
    torch.save({"gy": yy.grad, "ggamma": sbn.weight.grad, "gbeta": sbn.bias.grad}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_sync_batchnorm_two_ranks_matches_one_batchnorm_on_the_concatenated_batch(tmp_path, monkeypatch):
    monkeypatch.setattr(PB, "DEV", "cpu")
    monkeypatch.setattr(S, "DEV", "cpu")
    port = EB._free_port()
    mp.spawn(_sync_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r = [torch.load(tmp_path / f"r{k}.pt") for k in range(2)]
    ins = [EB._sync_inputs(k) for k in range(2)]
    _, bn, w, b, _ = ins[0]
    y64 = torch.cat([i[0] for i in ins]).double().requires_grad_(True)
    gzn = torch.cat([_cols(k)[2] for k in range(2)]).double()
    g64 = bn.weight.detach().double()
    be64 = bn.bias.detach().double()
    a = F.batch_norm(y64, bn.running_mean.double().clone(), bn.running_var.double().clone(), g64, be64, True,
                     bn.momentum, bn.eps)
    zn = F.normalize(F.conv2d(F.relu(a), w.double(), b.double()), p=2, dim=1)
    gy, ga = torch.autograd.grad(zn, (y64, a), gzn)
    xhat = (y64 - y64.mean((0, 2, 3), keepdim=True)) / torch.sqrt(y64.var((0, 2, 3), unbiased=False, keepdim=True)
                                                                   + bn.eps)
    n0 = EB.SYNC_SHAPES[0][0]
    for k, sl in enumerate((slice(0, n0), slice(n0, None))):
        local = {"gy": gy[sl], "gbeta": ga[sl].sum((0, 2, 3)), "ggamma": (ga[sl] * xhat[sl]).sum((0, 2, 3))}
        e = P.errors({n: r[k][n] for n in local}, local)
        for n in local:
            assert e[n][0] <= PB.MAXABS[n] and e[n][1] <= PB.FROB[n], (k, n, e)
