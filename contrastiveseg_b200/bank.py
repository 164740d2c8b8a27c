"""Pixel / region memory bank (SURVEY §8 rows a7, a8, e).

* ``MemoryBank``: the four buffers of HRNet_W48_MEM (lib/models/nets/hrnet.py:165-171) with the same names,
  shapes and dtypes (so reference checkpoints load), plus an engine-internal bf16 class-blocked shadow.
* ``dequeue_and_enqueue``: drop-in for Trainer._dequeue_and_enqueue (segmentor/trainer_contrastive.py:102-138):
  mutates the passed buffers in place.  One rank: bit-for-bit the reference's ring-buffer semantics
  (Q2, Q4, Q5, Q6).  Several ranks: every rank builds a fixed-size packet of its new rows, ONE NCCL
  all_gather merges them and every rank applies all packets in rank order, so all banks stay identical
  (replaces the 194.6 MB rank-0 buffer broadcast of DDP, Q9).
  Called between a loss that read the bank and its ``backward()`` (the trainer's order, trainer_contrastive.py:241-255)
  the in-place write is held back until right after that backward: the reference's autograd keeps a copy of the bank
  for its backward, the engine re-reads the bank instead.  Final bank and gradient equal the reference's.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _abi
from . import functional as _fn
from . import rng as _rng


def _is_cuda(t: torch.Tensor) -> bool:
    return t.is_cuda


def shadow_rows(num_classes: int, memory_size: int) -> int:
    rows = max((num_classes - 1) * 2 * memory_size, 1)
    return -(-rows // 256) * 256


class MemoryBank(nn.Module):
    def __init__(self, num_classes: int, memory_size: int, dim: int = 256, with_shadow: bool = False):
        super().__init__()
        self.num_classes, self.memory_size, self.dim = num_classes, memory_size, dim
        self.register_buffer("segment_queue", F.normalize(torch.randn(num_classes, memory_size, dim), p=2, dim=2))
        self.register_buffer("segment_queue_ptr", torch.zeros(num_classes, dtype=torch.long))
        self.register_buffer("pixel_queue", F.normalize(torch.randn(num_classes, memory_size, dim), p=2, dim=2))
        self.register_buffer("pixel_queue_ptr", torch.zeros(num_classes, dtype=torch.long))
        self.with_shadow = with_shadow
        self.shadow = None            # bf16 ((K-1)*2M padded to 256, D), engine-internal (not in state_dict)

    def flush(self) -> None:
        """Apply bank writes still held back for a pending backward (see ``dequeue_and_enqueue``): between ``loss_step``
        and ``backward()`` the buffers hold the bank the loss read, not yet the rows enqueued since."""
        if self.segment_queue.is_cuda:
            _fn._flush_bank(self.segment_queue.device.index, self.segment_queue.data_ptr())

    def state_dict(self, *args, **kwargs):
        self.flush()                  # a checkpoint taken inside that window must contain the enqueued rows
        return super().state_dict(*args, **kwargs)

    def attach(self, outputs: dict) -> dict:
        """What the trainer does before the loss call (trainer_contrastive.py:214-217)."""
        outputs["pixel_queue"] = self.pixel_queue
        outputs["pixel_queue_ptr"] = self.pixel_queue_ptr
        outputs["segment_queue"] = self.segment_queue
        outputs["segment_queue_ptr"] = self.segment_queue_ptr
        if self.with_shadow:
            if self.shadow is None:
                self.sync_shadow()
            outputs["bank_shadow"] = self.shadow          # engine-only: bf16 copy for the wgmma sweep
        return outputs

    def sync_shadow(self) -> torch.Tensor:
        """Rebuild the bf16 shadow from the fp32 queues (after load_state_dict or an external write)."""
        lib = _abi.load()
        dev = self.segment_queue.device
        if not _is_cuda(self.segment_queue):
            raise _abi.PclError("the bank shadow lives on the GPU")
        if self.shadow is None or self.shadow.device != dev:
            self.shadow = torch.empty((shadow_rows(self.num_classes, self.memory_size), self.dim),
                                      dtype=torch.bfloat16, device=dev)
        with torch.cuda.device(dev):
            _abi.check(lib.pcl_bank_shadow_rebuild(self.segment_queue.data_ptr(), self.pixel_queue.data_ptr(),
                                                   self.num_classes, self.memory_size, self.dim,
                                                   self.shadow.data_ptr(),
                                                   torch.cuda.current_stream(dev).cuda_stream),
                       "pcl_bank_shadow_rebuild")
        return self.shadow

    def enqueue(self, keys, labels, *, network_stride: int, pixel_update_freq: int, **kw) -> None:
        if self.with_shadow and self.shadow is None:
            self.sync_shadow()
        dequeue_and_enqueue(keys, labels, self.segment_queue, self.segment_queue_ptr, self.pixel_queue,
                            self.pixel_queue_ptr, network_stride=network_stride, memory_size=self.memory_size,
                            pixel_update_freq=pixel_update_freq, shadow=self.shadow, **kw)


def world_size(group=None) -> int:
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return 1
    return dist.get_world_size(group)


def gather_packets(packet: torch.Tensor, group=None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One all_gather of the fixed-size enqueue packet; returns (world, packet_floats), rank-major.
    ``out``: optional pre-allocated (world, packet_floats) receive buffer (no allocation per step)."""
    import torch.distributed as dist
    world = world_size(group)
    if world == 1:
        return packet.view(1, -1)
    if out is None or out.shape != (world, packet.numel()):
        out = torch.empty((world, packet.numel()), dtype=packet.dtype, device=packet.device)
    if packet.is_cuda:
        dist.all_gather_into_tensor(out, packet.view(-1).contiguous(), group=group)      # NCCL over NVLink
    else:
        dist.all_gather(list(out.unbind(0)), packet.view(-1).contiguous(), group=group)  # gloo (CPU tests)
    return out


_enqueue_counter = [0]

# Per (device, packet geometry, world) scratch / packet / receive buffers, kept across steps: the enqueue allocates
# nothing in steady state (round 1 drew two torch.empty per call).  Re-use is safe in stream order; the one case where a
# buffer may still be needed by a held-back bank write is handled by the caller (fresh buffers for that call).
_ENQ_BUFFERS = {}


def enqueue_buffers(dev: torch.device, n_scratch: int, n_packet: int, world: int, fresh: bool = False):
    key = (dev.index, n_scratch, n_packet, world)
    bufs = None if fresh else _ENQ_BUFFERS.get(key)
    if bufs is None:
        # the packet is zero-filled ONCE: slots of absent (image, class) pairs carry only their count header, the rest of
        # their rows is never written — the all_gather ships the whole packet, so it must not be uninitialised memory
        # (compute-sanitizer initcheck reports it otherwise)
        bufs = (torch.empty(n_scratch, dtype=torch.float32, device=dev),
                torch.zeros(n_packet, dtype=torch.float32, device=dev),
                torch.zeros((world, n_packet), dtype=torch.float32, device=dev) if world > 1 else None)
        if not fresh:
            if len(_ENQ_BUFFERS) >= 8:
                _ENQ_BUFFERS.pop(next(iter(_ENQ_BUFFERS)))
            _ENQ_BUFFERS[key] = bufs
    return bufs


def enqueue_seed(seed: int) -> int:
    """Base of the device-RNG seed of an enqueue; the per-call counter is added to it (host side here, device side in
    a captured step: pcl_bank_packet_dev)."""
    return (int(seed) * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF


def dequeue_and_enqueue(keys: torch.Tensor, labels: torch.Tensor, segment_queue: torch.Tensor,
                        segment_queue_ptr: torch.Tensor, pixel_queue: torch.Tensor, pixel_queue_ptr: torch.Tensor, *,
                        network_stride: int, memory_size: int, pixel_update_freq: int,
                        perm_fn: Optional[Callable[[int], torch.Tensor]] = None, rng: str = "device", seed: int = 304,
                        shadow: Optional[torch.Tensor] = None, group=None, distributed: bool = True,
                        defer_to_backward: bool = True) -> None:
    lib = _abi.load()
    if not _is_cuda(keys):
        raise _abi.PclError("keys must be a CUDA tensor: the engine has no CPU path")
    dev = keys.device
    keys_c = keys.detach()
    if keys_c.dtype not in _fn.DTYPE_CODES:              # bf16 / fp16 keys are read as they are (converted on load)
        keys_c = keys_c.to(torch.float32)
    keys_c = keys_c.contiguous()
    labels_c = labels.to(device=dev, dtype=torch.int64).contiguous()
    B, D, h, w = keys_c.shape
    K, M = segment_queue.shape[0], segment_queue.shape[1]
    if M != memory_size:
        raise _abi.PclError("memory_size differs from the queue shape")
    for t, name in ((segment_queue, "segment_queue"), (pixel_queue, "pixel_queue")):
        if not (_is_cuda(t) and t.dtype == torch.float32 and t.is_contiguous()):
            raise _abi.PclError(f"{name} must be a contiguous fp32 CUDA tensor (updated in place)")
    for t, name in ((segment_queue_ptr, "segment_queue_ptr"), (pixel_queue_ptr, "pixel_queue_ptr")):
        if not (_is_cuda(t) and t.dtype == torch.int64 and t.is_contiguous()):
            raise _abi.PclError(f"{name} must be a contiguous int64 CUDA tensor (updated in place)")
    g = _abi.BankGeom(B, D, h, w, labels_c.shape[1], labels_c.shape[2], K, M, network_stride, pixel_update_freq)
    n_packet = lib.pcl_bank_packet_floats(C.byref(g))
    n_scratch = lib.pcl_bank_scratch_floats(C.byref(g))
    if n_packet < 0:
        _abi.check(int(n_packet), "pcl_bank_packet_floats")
    # a write already held back for a pending backward still reads the cached packet buffers: this (rare) second
    # enqueue inside the same loss -> backward window gets buffers of its own
    reader = _fn.bank_reader(dev.index, segment_queue.data_ptr()) if defer_to_backward else None
    world = world_size(group) if distributed else 1
    scratch, packet, recv = enqueue_buffers(dev, n_scratch, n_packet, world,
                                            fresh=reader is not None and bool(reader.deferred))
    ranks = None
    if perm_fn is not None or rng == "torch_cpu":
        sub = labels_c[:, ::network_stride, ::network_stride].reshape(B, -1)
        valid = (sub > 0) & (sub < K)
        counts = torch.zeros((B, K), dtype=torch.int64, device=dev)
        counts.scatter_add_(1, sub.clamp(0, K - 1), valid.to(torch.int64))
        table = _rng.bank_rank_table(counts.cpu().numpy(), pixel_update_freq, perm_fn or (lambda n: torch.randperm(n)))
        ranks = table.to(dev)
    _enqueue_counter[0] += 1
    s = (enqueue_seed(seed) + _enqueue_counter[0]) & 0xFFFFFFFFFFFFFFFF
    with _fn._on_device(dev):
        if keys_c.dtype == torch.float32:
            _abi.check(lib.pcl_bank_packet(C.byref(g), keys_c.data_ptr(), labels_c.data_ptr(), _abi.ptr(ranks), s,
                                           scratch.data_ptr(), packet.data_ptr(), _fn._stream_ptr(dev)), "pcl_bank_packet")
        else:
            _abi.check(lib.pcl_bank_packet_dt(C.byref(g), keys_c.data_ptr(), _fn.DTYPE_CODES[keys_c.dtype],
                                              labels_c.data_ptr(), _abi.ptr(ranks), s, scratch.data_ptr(), packet.data_ptr(),
                                              _fn._stream_ptr(dev)), "pcl_bank_packet_dt")
        packets = gather_packets(packet, group, out=recv) if distributed else packet.view(1, -1)

    def apply_packets():           # the in-place write (rows, pointers, bf16 shadow): ordered, rank-major
        with _fn._on_device(dev):
            _abi.check(lib.pcl_bank_apply(C.byref(g), packets.data_ptr(), packets.shape[0], segment_queue.data_ptr(),
                                          segment_queue_ptr.data_ptr(), pixel_queue.data_ptr(),
                                          pixel_queue_ptr.data_ptr(), _abi.ptr(shadow), _fn._stream_ptr(dev)),
                       "pcl_bank_apply")

    # A loss that read this bank and has not run its backward yet will re-read the bank in that backward (the reference
    # holds a copy instead, loss_contrast_mem.py:221): hold the write back until right after it.
    if reader is not None:
        reader.deferred.append(apply_packets)
    else:
        apply_packets()
