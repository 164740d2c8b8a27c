"""One pixel-contrast loss step captured in a single CUDA graph (SURVEY §8f row 4).

The eager step costs ~0.14 ms of host time (Python + autograd + 8 kernel launches) against ~0.13-0.16 ms of GPU
time at the Cityscapes shape, so it is host-launch-bound as soon as the host slows down (8 ranks on one box).  The C
ABI neither allocates nor synchronises and all scratch is caller-owned, so the whole sequence

    pcl_step_stats -> pcl_step_forward_ctr -> pcl_step_backward[_prezeroed]

is capturable: a replay is ONE graph launch.  The zero-fill of the dense gradient (the HBM floor of the step) runs as
a parallel branch of the graph from the start of the step (``overlap_zero_fill``), hidden behind the latency-bound
selection and sweep kernels; the backward then scatters only the sampled columns.  Constraints of a captured graph, made explicit here:

* static shapes and static addresses: the tensors given to the constructor are read in place on every replay —
  refill them (``embed.copy_(...)`` or let the producer write into them), do not replace them;
* sampling stays fresh: kernel arguments are frozen in a graph, so the selection kernel draws the anchor ranks from a
  counter in device memory (``pcl_step_forward_ctr``) instead of the by-value seed of the eager path;
* the upstream gradient is a device scalar (``grad_scale``, default 1) folded into the dense gradient by the
  backward kernels, not an autograd input: use it for the loss weight (``contrast.loss_weight``).

The reference RNG stream (``rng='torch_cpu'`` / injected permutations) needs a host round trip and is not capturable.

Memory-bank steps (``enqueue=``): the trainer's order loss -> enqueue -> backward (trainer_contrastive.py:241-255) is part
of the captured sequence: stats -> forward -> enqueue packet | all_gather | backward -> bank write.  One rank: a
single graph.  Several ranks: three graphs and ONE NCCL all_gather of the packet — forward + packet, then the backward
sweep with the all_gather next to it on its own stream, then the bank write (four host calls per step, nothing
allocated, no host synchronisation; ``PCL_GATHER_OVERLAP=0``: two graphs with the all_gather between them); the bank
write comes after the backward sweep that re-reads the bank, so gradient and final bank equal the reference's (same
property as the eager deferred write).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Callable, Optional, Tuple

import torch

from . import _abi
from . import functional as _fn
from .functional import ContrastOptions, ContrastWorkspace


def _canonical(t: Optional[torch.Tensor], dtype: torch.dtype, name: str, device: torch.device) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if t.device != device or t.dtype != dtype or not t.is_contiguous():
        raise _abi.PclError(f"{name} must be a contiguous {dtype} tensor on {device}: a captured graph reads it in "
                            "place on every replay, so no converted copy can be made")
    return t


def _canonical_float(t: Optional[torch.Tensor], name: str, device: torch.device) -> Optional[torch.Tensor]:
    """embed / seg / bank keys: fp32, bf16 or fp16, read in place in their own dtype."""
    if t is None:
        return None
    if t.device != device or t.dtype not in _fn.DTYPE_CODES or not t.is_contiguous():
        raise _abi.PclError(f"{name} must be a contiguous float32, bfloat16 or float16 tensor on {device}: a captured "
                            "graph reads it in place on every replay, so no converted copy can be made")
    return t


class GraphedContrastStep:
    """loss, d loss/d embed of ``pixel_contrast_loss`` for fixed tensors, as one CUDA-graph replay.

    >>> step = GraphedContrastStep(embed, labels, seg=seg, options=opts, grad_scale=loss_weight)
    >>> loss, grad = step.replay()          # 0-dim loss and (B,D,h,w) gradient, both static buffers
    """

    def __init__(self, embed: torch.Tensor, labels: torch.Tensor, *, seg: Optional[torch.Tensor] = None,
                 predict: Optional[torch.Tensor] = None, segment_queue: Optional[torch.Tensor] = None,
                 pixel_queue: Optional[torch.Tensor] = None, bank_shadow: Optional[torch.Tensor] = None,
                 options: Optional[ContrastOptions] = None, grad_scale: float = 1.0, capture: bool = True,
                 warmup: int = 2, overlap_zero_fill: bool = True, enqueue: Optional[dict] = None,
                 fused: Optional[bool] = None, sparse_reset: bool = False,
                 prologue: Optional[Callable[[int], None]] = None, epilogue: Optional[Callable[[int], None]] = None):
        """embed and seg may be fp32, bf16 or fp16 (each independently); ``grad`` has embed's dtype.
        enqueue (bank steps): dict(bank=MemoryBank, keys=(B,D,h,w) fp32/bf16/fp16 [default: embed], labels=(B,Himg,Wimg) int64
        [default: labels], network_stride=int, pixel_update_freq=int, seed=int, group=process group or None).
        prologue / epilogue: work of the caller launched on the step's stream (its handle is the argument) before the
        step's first kernel and after its last, captured into the first and the last graph (GraphedContrastCriterion's
        seg half and total loss)."""
        self.lib = _abi.load()
        self.prologue, self.epilogue = prologue, epilogue
        opts = options or ContrastOptions()
        _fn._require_cuda(embed, "embed")
        device = embed.device
        if opts.rng != "device" or opts.perm_fn is not None:
            raise _abi.PclError("a captured step draws its anchors on the device: rng must be 'device'")
        self.opts = opts
        self.embed = _canonical_float(embed.detach(), "embed", device)
        if self.embed.dtype != torch.float32 and opts.topk_negatives:
            raise _abi.PclError("topk_negatives needs a float32 embed (the top-k sweeps have no half-precision input)")
        self.labels = _canonical(labels, torch.int64, "labels", device)
        self.seg = _canonical_float(None if seg is None else seg.detach(), "seg", device)
        self.predict = _canonical(predict, torch.int64, "predict", device)
        if self.seg is None and self.predict is None:
            raise _abi.PclError("either seg or predict is required")
        self.segq = _canonical(None if segment_queue is None else segment_queue.detach(), torch.float32, "segment_queue", device)
        self.pixq = _canonical(None if pixel_queue is None else pixel_queue.detach(), torch.float32, "pixel_queue", device)
        B, D, h, w = self.embed.shape
        if self.labels.dim() != 3 or self.labels.shape[0] != B:
            raise _abi.PclError("labels must be (B, Himg, Wimg)")
        mode, bank_K, M0, M1 = 0, 0, 0, 0
        if self.segq is not None:
            mode, bank_K, M0 = 1, self.segq.shape[0], self.segq.shape[1]
            M1 = self.pixq.shape[1] if self.pixq is not None else 0
            if self.segq.shape[2] != D:
                raise _abi.PclError("bank feature dim differs from the embedding dim")
        K = opts.num_classes or (self.seg.shape[1] if self.seg is not None else (bank_K if mode == 1 else _abi.MAX_CLASSES))
        if self.seg is not None and (self.seg.shape[1] != K or self.seg.shape[0] != B or tuple(self.seg.shape[2:]) != (h, w)):
            raise _abi.PclError("seg must be (B, K, h, w) at the embedding resolution with K == num_classes")
        geom = _abi.Geom(B, D, h, w, self.labels.shape[1], self.labels.shape[2], K, opts.max_samples, opts.max_views,
                         opts.ignore_label)
        self.ws = ContrastWorkspace(device, geom, mode, bank_K, M0, M1)        # owned by this object, never shared
        self.device = device
        self.loss = torch.zeros((), dtype=torch.float32, device=device)
        self.grad = torch.empty_like(self.embed)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)         # replay index, lives on the device
        self.scale = torch.full((1,), float(grad_scale), dtype=torch.float32, device=device)
        d = self.ws.desc
        d.embed, d.labels = self.embed.data_ptr(), self.labels.data_ptr()
        d.seg, d.predict = _abi.ptr(self.seg), _abi.ptr(self.predict if self.seg is None else None)
        d.embed_dtype = _fn.DTYPE_CODES[self.embed.dtype]
        d.seg_dtype = _fn.DTYPE_CODES[self.seg.dtype] if self.seg is not None else _abi.DT_F32
        d.segment_queue, d.pixel_queue = _abi.ptr(self.segq), _abi.ptr(self.pixq)
        d.temperature, d.base_temperature = opts.temperature, opts.base_temperature
        d.nan_safe, d.normalize = int(opts.nan_safe), int(opts.normalize)
        self.ws.set_topk(int(opts.topk_negatives or 0))
        d.precision = 0
        self.shadow = None
        if opts.precision == "bf16":
            if not self.ws.tc_ok:
                raise _abi.PclError("precision='bf16' (wgmma sweep) needs proj_dim == 256")
            d.precision = 1
            d.contrast_norm_bound = float(opts.contrast_norm_bound)
            if mode == 1:
                if self.pixq is None or M0 != M1:
                    raise _abi.PclError("the tensor sweep reads the bank as (segment_queue, pixel_queue) of equal size")
                if bank_shadow is None:
                    raise _abi.PclError("pass the bank's maintained bf16 shadow (MemoryBank(with_shadow=True).shadow): "
                                        "a captured step cannot rebuild it")
                self.shadow = bank_shadow
                d.shadow_bf16, d.shadow_rows = bank_shadow.data_ptr(), bank_shadow.shape[0]
        elif opts.precision != "fp32":
            raise _abi.PclError(f"unknown precision {opts.precision!r}")
        d.seed = int(opts.seed) & 0xFFFFFFFFFFFFFFFF          # base seed; the per-replay part is the device counter
        d.loss, d.grad_embed = self.loss.data_ptr(), self.grad.data_ptr()
        # Small-anchor shape (no bank, tensor path, D = 256, max_samples <= 1024: BASELINE configs[1]): four launches
        # instead of eleven — scan+plan, selection, ONE kernel for the InfoNCE forward and backward (logits stay in tensor
        # memory), scatter — with the engine's own zero-fill of the dense gradient on a parallel branch.
        ok = bool(self.lib.pcl_step_fused_supported(C.byref(d))) and enqueue is None
        if fused and not ok:
            raise _abi.PclError("fused=True: the step does not qualify (needs no bank, precision='bf16', D=256, "
                                "max_samples<=1024, normalize=False)")
        self.fused = ok if fused is None else bool(fused)
        # sparse_reset (fused steps): ``grad`` persists between replays, zero-filled once here; every replay clears exactly
        # the A*D entries the previous one scattered instead of re-filling B*D*h*w zeros (268 MB at the Cityscapes shape).
        # Contract: nobody else writes ``grad`` (call ``reset_grad()`` if that happened).
        self.sparse_reset = bool(sparse_reset) and self.fused
        self.prev_rows = None
        if self.sparse_reset:
            self.prev_rows = torch.zeros(1 + 2 * opts.max_samples, dtype=torch.int32, device=device)
            self.grad.zero_()
        self.graph = None
        self.graph_b = None
        self.graph_c = None                    # split steps: the bank write as a graph of its own (see replay)
        self._gather_stream = None
        self.replays = 0
        self.enq = None
        if enqueue is not None:
            self._init_enqueue(enqueue)
        # The zero-fill of the dense gradient (B*D*h*w*4 bytes, the HBM floor of the step) does not depend on anything
        # the step computes: run it on a second stream from the start of the step, behind the latency-bound selection
        # and sweep kernels, and let the backward scatter only the sampled columns (pcl_step_backward_prezeroed).  Not for
        # top-k steps: their backward writes the dense gradient itself (zero-fill + scatter).
        self.overlap_zero_fill = bool(overlap_zero_fill) and not opts.topk_negatives
        self.side = None
        if capture:
            self._capture(max(1, int(warmup)))

    def _init_enqueue(self, e: dict) -> None:
        from . import bank as _bank
        bank = e["bank"]
        if self.segq is None or bank.segment_queue.data_ptr() != self.segq.data_ptr():
            raise _abi.PclError("enqueue=: the step must read the bank it writes (pass bank.segment_queue / pixel_queue)")
        dev = self.device
        keys = _canonical_float(e.get("keys", self.embed).detach(), "keys", dev)
        labels = _canonical(e.get("labels", self.labels), torch.int64, "lb_key", dev)
        B, D, h, w = keys.shape
        g = _abi.BankGeom(B, D, h, w, labels.shape[1], labels.shape[2], bank.num_classes, bank.memory_size,
                          int(e["network_stride"]), int(e["pixel_update_freq"]))
        n_packet = self.lib.pcl_bank_packet_floats(C.byref(g))
        n_scratch = self.lib.pcl_bank_scratch_floats(C.byref(g))
        if n_packet < 0:
            _abi.check(int(n_packet), "pcl_bank_packet_floats")
        group = e.get("group")
        world = _bank.world_size(group)
        # buffers owned by this object (a captured graph holds their addresses)
        scratch, packet, recv = _bank.enqueue_buffers(dev, int(n_scratch), int(n_packet), world, fresh=True)
        if bank.with_shadow and bank.shadow is None:
            bank.sync_shadow()
        # the enqueue has its own device counter: its packet is built on a parallel branch of the graph (it depends on the
        # inputs only), so it must not read the step counter the forward branch advances; replay r uses offset r + 1 like
        # the eager enqueue (bank._enqueue_counter pre-increments)
        self.enq_counter = torch.zeros(1, dtype=torch.int64, device=dev)
        self.enq = dict(bank=bank, keys=keys, labels=labels, g=g, scratch=scratch, packet=packet, recv=recv, world=world,
                        group=group, seed=(_bank.enqueue_seed(int(e.get("seed", 304))) + 1) & 0xFFFFFFFFFFFFFFFF)

    def _enqueue_packet(self, stream: int) -> None:
        q = self.enq
        keys = q["keys"]
        if keys.dtype != torch.float32:        # bf16 / fp16 keys: converted on load, same packet as from fp32 keys
            _abi.check(self.lib.pcl_bank_packet_dev_dt(C.byref(q["g"]), keys.data_ptr(), _fn.DTYPE_CODES[keys.dtype],
                                                       q["labels"].data_ptr(), q["seed"], self.enq_counter.data_ptr(),
                                                       q["scratch"].data_ptr(), q["packet"].data_ptr(), stream),
                       "pcl_bank_packet_dev_dt")
            return
        _abi.check(self.lib.pcl_bank_packet_dev(C.byref(q["g"]), keys.data_ptr(), q["labels"].data_ptr(), q["seed"],
                                                self.enq_counter.data_ptr(), q["scratch"].data_ptr(), q["packet"].data_ptr(),
                                                stream), "pcl_bank_packet_dev")

    def _gather(self) -> torch.Tensor:
        q = self.enq
        if q["world"] == 1:
            return q["packet"].view(1, -1)
        from . import bank as _bank
        return _bank.gather_packets(q["packet"], q["group"], out=q["recv"])        # NCCL over NVLink (gloo in CPU tests)

    def _enqueue_apply(self, stream: int) -> None:
        q = self.enq
        b = q["bank"]
        pk = q["recv"] if q["world"] > 1 else q["packet"]
        _abi.check(self.lib.pcl_bank_apply_ctr(C.byref(q["g"]), pk.data_ptr(), q["world"], b.segment_queue.data_ptr(),
                                               b.segment_queue_ptr.data_ptr(), b.pixel_queue.data_ptr(),
                                               b.pixel_queue_ptr.data_ptr(), _abi.ptr(b.shadow),
                                               self.enq_counter.data_ptr(), stream), "pcl_bank_apply_ctr")

    # fork / join of the overlapped zero-fill (torch streams + events; inside a capture these become graph edges)
    def _fork_zero_fill(self) -> None:
        main = torch.cuda.current_stream(self.device)
        if self.side is None:
            self.side = torch.cuda.Stream(self.device)
        self.side.wait_stream(main)                  # the previous consumer of `grad` is ordered before the fill
        with torch.cuda.stream(self.side):
            self._side_branch(self.side.cuda_stream)

    def _side_branch(self, stream: int) -> None:
        """Work that depends on the step's inputs only: zero-fill of the dense gradient, enqueue packet."""
        if self.fused:           # the engine's own fill kernel (small CTAs that share the SMs with the loss kernels)
            _abi.check(self.lib.pcl_step_fused_fill(C.byref(self.ws.desc), stream), "pcl_step_fused_fill")
        elif self.overlap_zero_fill:
            self.grad.zero_()
        if self.enq is not None:
            # the enqueue packet (label counts, segment sums over the keys, pixel rows: ~70 us at the Cityscapes shape)
            # runs on this branch, next to the forward sweeps
            self._enqueue_packet(stream)

    def _join_zero_fill(self) -> None:
        torch.cuda.current_stream(self.device).wait_stream(self.side)

    # the launch sequence (also usable eagerly: capture=False)
    def _enqueue_a(self, stream: int) -> None:
        """First half: (zero-fill branch ||) stats -> forward -> this rank's enqueue packet."""
        lib, d = self.lib, self.ws.desc
        if self.prologue is not None:
            self.prologue(stream)
        if self.fused:
            _abi.check(lib.pcl_step_stats(C.byref(d), stream), "pcl_step_stats")
            _abi.check(lib.pcl_step_fused_select(C.byref(d), self.counter.data_ptr(), _abi.ptr(self.prev_rows), stream),
                       "pcl_step_fused_select")
            # full-fill mode: the fill forks AFTER scan and selection — next to it their DRAM reads slow down (measured
            # in-graph on H100: scan 24 -> 91 us, selection 15 -> 22 us; step 0.164 -> 0.179 ms), only the L2-resident
            # InfoNCE kernel hides behind it
            if not self.sparse_reset:
                self._fork_zero_fill()
            _abi.check(lib.pcl_step_fused_loss(C.byref(d), stream), "pcl_step_fused_loss")
            if not self.sparse_reset:
                self._join_zero_fill()
            return
        side = self.overlap_zero_fill or self.enq is not None
        if side:
            self._fork_zero_fill()
        _abi.check(lib.pcl_step_stats(C.byref(d), stream), "pcl_step_stats")
        # the selection kernel draws the anchors from the device counter itself (no separate rank-draw launch)
        _abi.check(lib.pcl_step_forward_ctr(C.byref(d), self.counter.data_ptr(), stream), "pcl_step_forward_ctr")
        if side:
            self._join_zero_fill()

    def _enqueue_b(self, stream: int) -> None:
        """Second half: backward -> dense gradient -> (after the sweep that re-reads the bank) the bank write."""
        lib, d = self.lib, self.ws.desc
        if self.fused:
            _abi.check(lib.pcl_step_fused_scatter(C.byref(d), self.scale.data_ptr(), self.counter.data_ptr(),
                                                  _abi.ptr(self.prev_rows), stream), "pcl_step_fused_scatter")
            return
        if self.overlap_zero_fill:
            _abi.check(lib.pcl_step_backward_prezeroed(C.byref(d), self.scale.data_ptr(), stream),
                       "pcl_step_backward_prezeroed")
        else:
            _abi.check(lib.pcl_step_backward(C.byref(d), self.scale.data_ptr(), stream), "pcl_step_backward")
        if self.enq is not None and not self._apply_separately:
            self._enqueue_apply(stream)

    @property
    def split(self) -> bool:
        """Two graphs with the all_gather between them (bank step on several ranks)."""
        return self.enq is not None and self.enq["world"] > 1

    @property
    def _apply_separately(self) -> bool:
        """Split steps launch the bank write on its own (third graph) so that the all_gather can run under the backward
        sweep; PCL_GATHER_OVERLAP=0 restores the two-graph sequence with the all_gather between them."""
        return self.split and os.environ.get("PCL_GATHER_OVERLAP", "1") != "0"

    def _enqueue(self, stream: int) -> None:
        self._enqueue_a(stream)
        if self.split:
            self._gather()
        self._enqueue_b(stream)
        if self._apply_separately:
            self._enqueue_apply(stream)
        if self.epilogue is not None:
            self.epilogue(stream)

    def _capture(self, warmup: int) -> None:
        dev = self.device
        cap = torch.cuda.Stream(dev)           # capture stream (graphs cannot be captured on the default stream)
        cap.wait_stream(torch.cuda.current_stream(dev))
        if self.enq is not None:               # the warm-up runs write the bank: put it back afterwards
            b = self.enq["bank"]
            self._bank_snapshot = [t.clone() for t in (b.segment_queue, b.segment_queue_ptr, b.pixel_queue,
                                                       b.pixel_queue_ptr)] + ([b.shadow.clone()] if b.shadow is not None else [])
        with torch.cuda.device(dev), torch.cuda.stream(cap):
            for _ in range(warmup):            # eager runs first: kernels get loaded, function attributes set, TMA
                self._enqueue(cap.cuda_stream)  # descriptors encoded — none of that may happen under capture
        torch.cuda.current_stream(dev).wait_stream(cap)
        self.counter.zero_()
        if self.enq is not None:
            torch.cuda.synchronize(dev)
            self.enq_counter.zero_()
            self._restore_bank()
        # thread_local: only this thread's CUDA calls are policed during the capture (the NCCL watchdog of a DDP job polls
        # events from another thread)
        graph = torch.cuda.CUDAGraph()
        if not self.split:
            with torch.cuda.device(dev), torch.cuda.graph(graph, stream=cap, capture_error_mode="thread_local"):
                s = torch.cuda.current_stream(dev).cuda_stream
                self._enqueue_a(s)
                self._enqueue_b(s)
                if self.epilogue is not None:
                    self.epilogue(s)
            self.graph = graph
        else:
            graph_b = torch.cuda.CUDAGraph()
            with torch.cuda.device(dev), torch.cuda.graph(graph, stream=cap, capture_error_mode="thread_local"):
                self._enqueue_a(torch.cuda.current_stream(dev).cuda_stream)
            with torch.cuda.device(dev), torch.cuda.graph(graph_b, stream=cap, capture_error_mode="thread_local"):
                self._enqueue_b(torch.cuda.current_stream(dev).cuda_stream)
                if self.epilogue is not None and not self._apply_separately:
                    self.epilogue(torch.cuda.current_stream(dev).cuda_stream)
            if self._apply_separately:         # third graph: the bank write, after the all_gather that ran under graph_b
                graph_c = torch.cuda.CUDAGraph()
                with torch.cuda.device(dev), torch.cuda.graph(graph_c, stream=cap, capture_error_mode="thread_local"):
                    self._enqueue_apply(torch.cuda.current_stream(dev).cuda_stream)
                    if self.epilogue is not None:
                        self.epilogue(torch.cuda.current_stream(dev).cuda_stream)
                self.graph_c = graph_c
                self._gather_stream = torch.cuda.Stream(dev)
            self.graph, self.graph_b = graph, graph_b

    def _restore_bank(self) -> None:
        b = self.enq["bank"]
        snap, self._bank_snapshot = self._bank_snapshot, None
        for t, v in zip((b.segment_queue, b.segment_queue_ptr, b.pixel_queue, b.pixel_queue_ptr), snap):
            t.copy_(v)
        if b.shadow is not None:
            b.shadow.copy_(snap[4])

    def reset_grad(self) -> None:
        """sparse_reset steps: re-establish the all-zero state of ``grad`` after somebody else wrote into it."""
        if self.sparse_reset:
            self.grad.zero_()
            self.prev_rows.zero_()

    def set_grad_scale(self, value: float) -> None:
        self.scale.fill_(float(value))

    def replay(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """Run one step on the current stream.  Returns (loss, grad_embed): static buffers, overwritten by the next
        replay; grad_embed = grad_scale * d loss / d embed."""
        if self.graph is not None:
            self.graph.replay()
            if self.graph_c is not None:
                # Only the bank WRITE needs the other ranks' packets: the all_gather runs on its own stream UNDER the
                # backward sweep (graph_b), the write (graph_c) waits for both.
                cur = torch.cuda.current_stream(self.device)
                self._gather_stream.wait_stream(cur)
                with torch.cuda.stream(self._gather_stream):
                    self._gather()
                self.graph_b.replay()
                cur.wait_stream(self._gather_stream)
                self.graph_c.replay()
            elif self.graph_b is not None:
                self._gather()
                self.graph_b.replay()
        else:
            with _fn._on_device(self.device):
                self._enqueue(_fn._stream_ptr(self.device))
        self.replays += 1
        return self.loss, self.grad

    def apply(self, embed: torch.Tensor) -> torch.Tensor:
        """Autograd hand-off: replays the graph and returns the loss connected to ``embed`` (which must be the tensor
        the graph was captured on); its backward returns the pre-computed static gradient.  Valid when the returned
        loss enters the total loss with coefficient 1 and ``backward`` starts from gradient 1 (fold weights into
        ``grad_scale``): the upstream gradient is NOT multiplied in (that would cost another pass over the dense
        gradient)."""
        if embed.data_ptr() != self.embed.data_ptr():
            raise _abi.PclError("apply() must receive the tensor the step was captured on")
        return _GraphedFn.apply(embed, self)


class _GraphedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, embed, step: GraphedContrastStep):
        loss, _ = step.replay()
        ctx.step = step
        return loss.view(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        # the static gradient already contains grad_scale; an upstream factor other than 1 (loss weight applied outside,
        # AMP loss scaling) would be silently dropped -> asynchronous device-side assertion (no host sync, one tiny kernel)
        torch._assert_async((grad_out == 1).all(),
                            "GraphedContrastStep.apply(): upstream gradient != 1; fold the factor into grad_scale")
        return ctx.step.grad, None
