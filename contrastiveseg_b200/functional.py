"""Autograd entry points of the engine: thin Python over the C ABI (include/pcl.h).

PyTorch is plumbing here (device memory, streams, autograd hand-off); all arithmetic of the path runs in
the CUDA kernels of libpcl_b200.so.  No fallback: tensors must be CUDA tensors and the library must load.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import weakref
from typing import Callable, Optional, Tuple

import torch

from . import _abi
from . import rng as _rng


@dataclasses.dataclass
class ContrastOptions:
    temperature: float = 0.1
    base_temperature: float = 0.07
    max_samples: int = 1024
    max_views: int = 100
    ignore_label: int = -1
    num_classes: Optional[int] = None      # class ids tracked; default: seg planes / bank classes / 256
    normalize: bool = False                # True: `embed` is the raw projection, the engine normalises the sampled columns
    nan_safe: bool = False                 # False reproduces the reference's NaN for rows without positives (Q8)
    rng: str = "device"                    # "device" (no host sync) | "torch_cpu" (reference RNG stream)
    perm_fn: Optional[Callable[[int], torch.Tensor]] = None   # injected permutations (parity tests)
    seed: int = 304
    precision: str = "fp32"                # "fp32" exact SIMT sweep | "bf16" wgmma sweep (bank / large problems)
    contrast_norm_bound: float = 1.0       # bound of the contrast rows' L2 norm (tensor path stabiliser; 1 = normalised)
    topk_negatives: Optional[int] = None   # a10 extension: keep only the k hardest negatives per anchor (None = reference)


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class _on_device:
    """torch.cuda.device(...) only when the tensor's device is not already current (saves ~10 us per call)."""

    __slots__ = ("ctx",)

    def __init__(self, device: torch.device):
        self.ctx = None if torch.cuda.current_device() == device.index else torch.cuda.device(device)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)
        return False


# Element types the engine reads natively (embed, seg, bank keys): converted to fp32 on load inside the kernels, the
# dense gradient written in embed's dtype (the fp32 gradient rounded once to nearest-even).
DTYPE_CODES = {torch.float32: _abi.DT_F32, torch.bfloat16: _abi.DT_BF16, torch.float16: _abi.DT_F16}


def dtype_code(t: torch.Tensor, name: str) -> int:
    code = DTYPE_CODES.get(t.dtype)
    if code is None:
        raise _abi.PclError(f"{name} must be float32, bfloat16 or float16, got {t.dtype}")
    return code


def _require_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise _abi.PclError(f"{name} must be a CUDA tensor: the engine has no CPU path")


class ContrastWorkspace:
    """Caller-owned scratch for one geometry (torch allocator owns the memory; the C side keeps no state)."""

    def __init__(self, device: torch.device, geom: _abi.Geom, mode: int, bank_K: int, bank_M0: int, bank_M1: int):
        lib = _abi.load()
        self.device = device
        self.geom = geom
        sizes = _abi.SelectSizes()
        _abi.check(lib.pcl_select_sizes(C.byref(geom), C.byref(sizes)), "pcl_select_sizes")
        self.sizes = sizes
        ms, D = geom.max_samples, geom.D
        sw = _abi.SweepDesc()
        sw.a_rows, sw.D, sw.mode = ms, D, mode
        sw.bank_K, sw.bank_M0, sw.bank_M1 = bank_K, bank_M0, bank_M1
        sw.temperature, sw.base_temperature = 1.0, 1.0
        ss = _abi.SweepSizes()
        _abi.check(lib.pcl_sweep_sizes(C.byref(sw), C.byref(ss)), "pcl_sweep_sizes")
        self.sweep_sizes = ss
        n_partial, n_dpartial = ss.partial_f32, ss.dpartial_f32
        n_topk = lib.pcl_topk_scratch_u32(C.byref(sw))              # a10 selection scratch (negative: pcl_status)
        if n_topk < 0:
            _abi.check(int(n_topk), "pcl_topk_scratch_u32")
        self.tc_ok = D == 256
        if self.tc_ok:                       # the tensor sweep uses its own split count: size for the larger of the two
            td = _abi.TcDesc()
            td.a_rows, td.D, td.mode = ms, D, mode
            # the step passes the device-side plan (live anchor count unknown on the host): the partial-slot count
            # depends on that, so size with a non-null plan exactly like the runtime descriptor
            self.plan = torch.zeros(sizes.plan_i32, dtype=torch.int32, device=device)
            td.plan = self.plan.data_ptr()
            td.bank_K, td.bank_R = bank_K, bank_M0 + bank_M1
            td.temperature, td.base_temperature = 1.0, 1.0
            ts = _abi.SweepSizes()
            _abi.check(lib.pcl_tc_sizes(C.byref(td), C.byref(ts)), "pcl_tc_sizes")
            n_partial, n_dpartial = max(n_partial, ts.partial_f32), max(n_dpartial, ts.dpartial_f32)
            n_tc_topk = lib.pcl_tc_topk_scratch_u32(C.byref(td))
            if n_tc_topk < 0:
                _abi.check(int(n_tc_topk), "pcl_tc_topk_scratch_u32")
            n_topk = max(n_topk, n_tc_topk)
            if mode == 0 and ms <= 1024:     # the fused self-contrast kernel: one slot per 256-column tile
                a_pad = -(-ms // 128) * 128
                s_max = -(-a_pad // 256)
                n_partial, n_dpartial = max(n_partial, s_max * a_pad), max(n_dpartial, s_max * a_pad * 256)
        i32 = dict(dtype=torch.int32, device=device)
        f32 = dict(dtype=torch.float32, device=device)
        self.keys = torch.empty(sizes.keys_u16, dtype=torch.int16, device=device)
        self.chunk_pref = torch.empty(sizes.chunk_pref_i32, **i32)
        self.counts = torch.empty(sizes.counts_i32, **i32)
        if not hasattr(self, "plan"):
            self.plan = torch.zeros(sizes.plan_i32, **i32)
        self.anchor_meta = torch.empty(sizes.anchor_meta_i32, **i32)
        self.anchors_f32 = torch.empty((ms, D), **f32)
        self.anchors_bf16 = torch.empty((-(-ms // 128) * 128, D), dtype=torch.bfloat16, device=device)
        self.inv_norm = torch.empty(ms, **f32)
        self.partials = torch.empty(5 * n_partial, **f32)
        self.rowstats = torch.empty(6 * ss.rowstat_f32, **f32)
        self.dpartials = torch.empty(n_dpartial, **f32)
        self.row_m2 = torch.empty(-(-ms // 256) * 256 + 512, **f32)
        self.dA = torch.empty((ms, D), **f32)
        self.loss = torch.zeros(1, **f32)
        self.ranks = torch.zeros(ms, **i32)
        self.ranks_host = torch.zeros(ms, dtype=torch.int32).pin_memory() if torch.cuda.is_available() else None
        self.sync = torch.zeros(1024, **i32)      # inter-CTA counters of the fused kernels (re-armed by the kernels themselves)
        self.topk_scratch_u32 = int(n_topk)
        self.topk_scratch = None     # a10 selection state (radix bins + per-row result), allocated by the first top-k step
        self.busy = False
        self.token = 0               # generation counter: a stale autograd node must not release a re-used workspace
        self.bank_key = None         # (device index, segment_queue address) while a backward that re-reads that bank is pending
        self.deferred = []           # bank writes held back until that backward has run (see bank.dequeue_and_enqueue)
        d = _abi.StepDesc()
        d.g = geom
        d.mode, d.bank_K, d.bank_M0, d.bank_M1 = mode, bank_K, bank_M0, bank_M1
        for name in ("keys", "chunk_pref", "counts", "plan", "anchor_meta", "anchors_f32", "anchors_bf16", "inv_norm",
                     "partials", "rowstats", "dpartials", "dA", "loss", "row_m2", "sync"):   # norm_max: optional, unused
            setattr(d, name, getattr(self, name).data_ptr())
        self.desc = d

    def set_topk(self, k: int) -> None:
        """a10 fields of the step descriptor: keep the k hardest negatives of every anchor (0 = all, the reference)."""
        if k < 0:
            raise _abi.PclError("topk_negatives must be >= 1 (None disables the selection)")
        if k and self.topk_scratch is None:
            self.topk_scratch = torch.empty(self.topk_scratch_u32, dtype=torch.int32, device=self.device)
        self.desc.topk_negatives = k
        self.desc.topk_scratch = _abi.ptr(self.topk_scratch)

    # views used by tests / diagnostics
    def plan_header(self):
        return self.plan[:_abi.PLAN_HEADER].tolist()


_WS_CACHE = {}                   # (device index, geometry key) -> [workspaces]; insertion order = age of the geometry
_WS_CACHE_MAX = int(os.environ.get("PCL_WS_CACHE_MAX", "8"))    # geometries kept (multi-scale / random-crop training)


_LAST_WS = {}


def _get_workspace(device, key, geom, mode, bank_K, bank_M0, bank_M1) -> ContrastWorkspace:
    ck = (device.index, key)
    lst = _WS_CACHE.get(ck)
    if lst is None:
        # a new geometry: forget the oldest idle ones first (their scratch goes back to the torch allocator; a
        # workspace still referenced by a pending autograd graph stays alive through that graph)
        if len(_WS_CACHE) >= _WS_CACHE_MAX:
            for old in list(_WS_CACHE):
                if len(_WS_CACHE) < _WS_CACHE_MAX:
                    break
                if not any(w.busy for w in _WS_CACHE[old]):
                    del _WS_CACHE[old]
        lst = _WS_CACHE[ck] = []
    for ws in lst:
        if not ws.busy:
            _LAST_WS[device.index] = ws
            return ws
    try:
        ws = ContrastWorkspace(device, geom, mode, bank_K, bank_M0, bank_M1)
    except _abi.PclError:
        if not lst:                      # a refused geometry leaves no cache entry behind
            del _WS_CACHE[ck]
        raise
    lst.append(ws)
    _LAST_WS[device.index] = ws
    return ws


def clear_workspaces() -> None:
    for key in list(_BANK_READERS):          # bank writes still held back go in before the bookkeeping is dropped
        _flush_bank(*key)
    _WS_CACHE.clear()
    _LAST_WS.clear()


_step_counter = [0]


# ---- banks with a pending reader -------------------------------------------------------------------------------
# The reference's autograd keeps its own copy of the bank for the backward (torch.cat in loss_contrast_mem.py:221), so
# the trainer may overwrite bank rows between the loss and loss.backward() (trainer_contrastive.py:241-255).  The engine
# keeps no copy: its backward sweep re-reads the bank.  A bank write that arrives while such a backward is pending is
# therefore held back and applied right after it (same final bank, same gradient as the reference).
_BANK_READERS = {}               # (device index, segment_queue address) -> [workspaces with a pending backward]


def bank_reader(device_index, segq_ptr):
    """The most recent loss whose pending backward will re-read the bank at this address, or None."""
    lst = _BANK_READERS.get((device_index, segq_ptr))
    return lst[-1] if lst else None


def _run_deferred(ws) -> None:
    calls, ws.deferred = ws.deferred, []
    for fn in calls:
        fn()


def _drop_bank_reader(ws) -> None:
    key, ws.bank_key = ws.bank_key, None
    if key is not None:
        lst = _BANK_READERS.get(key)
        if lst is not None:
            if ws in lst:
                lst.remove(ws)
            if not lst:
                del _BANK_READERS[key]
    _run_deferred(ws)


def _flush_bank(device_index, segq_ptr) -> None:
    """A new forward is about to read this bank: writes still held back for older pending losses go in first."""
    lst = _BANK_READERS.pop((device_index, segq_ptr), None)
    if lst:
        for ws in lst:
            ws.bank_key = None
            _run_deferred(ws)


def _release_workspace(ws, token) -> None:
    if ws.token == token:
        if ws.bank_key is not None or ws.deferred:
            _drop_bank_reader(ws)
        ws.busy = False


# ---- anchor-column hand-off (ProjectionHead(..., sparse_grad=True)) ----------------------------------------------
# The contrast loss reads zn at no more than max_samples pixels, so d loss / d zn is zero elsewhere.  A fused BN head
# built with sparse_grad=True registers its output zn here; an engine loss whose embed IS that zn (same tensor, same
# version) deposits its anchor columns in the sink and hands autograd a zero placeholder that costs no memory.  The
# head's backward takes the column path only when its incoming gradient is exactly that placeholder; anything else
# (other consumers of zn, two losses) is the dense path on the gradient autograd summed, plus every deposit.
class _ColumnSink:
    __slots__ = ("ref", "version", "deposits", "zeros")

    def __init__(self, zn: torch.Tensor):
        self.ref = weakref.ref(zn)
        self.version = zn._version
        self.deposits = []                   # [(cols (max_samples, D) fp32, col_pix (max_samples,) int32)]
        self.zeros = []                      # the placeholders' one-element storages

    def accepts(self) -> bool:
        """At the loss's backward: zn is alive and nobody reads its own gradient (retain_grad, tensor hooks)."""
        zn = self.ref()
        return zn is not None and not zn.retains_grad and not zn._backward_hooks

    def deposit(self, cols, col_pix, shape):
        zero = torch.zeros(1, dtype=self.ref().dtype, device=cols.device)
        self.deposits.append((cols, col_pix))
        self.zeros.append(zero)
        return zero.expand(shape)

    def is_placeholder(self, g: torch.Tensor) -> bool:
        # expand() keeps the stride of a dimension of size 1 (W = 1, or HW = 1): only the others must be 0
        return (len(self.deposits) == 1 and len(self.zeros) == 1
                and all(st == 0 or n == 1 for st, n in zip(g.stride(), g.shape))
                and g.data_ptr() == self.zeros[0].data_ptr())

    def take(self):
        deps, self.deposits, self.zeros = self.deposits, [], []
        return deps


_SINKS = {}                                  # id(zn) -> _ColumnSink (dropped with zn)


def _register_sink(zn: torch.Tensor) -> _ColumnSink:
    sink = _ColumnSink(zn)
    key = id(zn)
    _SINKS[key] = sink
    weakref.finalize(zn, _SINKS.pop, key, None).atexit = False
    return sink


def _sink_of(embed: torch.Tensor) -> Optional[_ColumnSink]:
    sink = _SINKS.get(id(embed))
    if sink is None or sink.ref() is not embed or sink.version != embed._version:
        return None
    return sink


def _with_deposits(gzn: torch.Tensor, deposits, dtype) -> torch.Tensor:
    """gzn (as autograd summed it) plus every deposited column, each rounded to zn's dtype as the loss's dense gradient
    would have been: the gradient the dense path would have received."""
    g = gzn.to(dtype=dtype).contiguous().clone()
    B, D = g.shape[0], g.shape[1]
    gv = g.view(B, D, -1)
    HW = gv.shape[2]
    for cols, col_pix in deposits:
        live = col_pix >= 0
        q = col_pix[live].long()
        b, p = q // HW, q % HW
        gv[b, :, p] += cols[live].to(dtype)
    return g


def cols_to_dense(cols: torch.Tensor, col_pix: torch.Tensor, shape, dtype: torch.dtype) -> torch.Tensor:
    """The dense (B, D, h, w) gradient of ``dtype`` that holds the anchor columns (cols (n, D) fp32, col_pix[s] =
    b*h*w + pix or < 0 for an unused row) and +0 elsewhere: each column rounded once to ``dtype`` and stored, not
    added, so the result equals the loss step's dense gradient to the bit (a -0 entry included).  No host
    synchronisation: every row is stored, an unused row into D scratch elements past the end of the tensor (its values
    are zero, so the rows that share them store the same bits)."""
    B, D = shape[0], shape[1]
    n = 1
    for e in shape:
        n *= e
    HW = n // (B * D)
    flat = torch.zeros(n + D, dtype=dtype, device=cols.device)
    q = col_pix.long()
    live = q >= 0
    q = q.clamp(min=0)
    base = torch.where(live, (q // HW) * (D * HW) + q % HW, torch.full_like(q, n))        # (rows,)
    step = torch.where(live, torch.full_like(q, HW), torch.ones_like(q))                  # channel stride
    idx = base[:, None] + step[:, None] * torch.arange(D, device=cols.device)[None, :]    # (rows, D)
    flat.index_put_((idx.reshape(-1),), cols.to(dtype).reshape(-1))
    return flat[:n].view(shape)


class _PixelContrastFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, embed, labels, seg, predict, segq, pixq, shadow, opts: ContrastOptions):
        lib = _abi.load()
        _require_cuda(embed, "embed")
        device = embed.device
        embed_dt = dtype_code(embed, "embed")
        if embed_dt != _abi.DT_F32 and opts.topk_negatives:
            raise _abi.PclError("topk_negatives needs a float32 embed (the top-k sweeps have no half-precision input)")
        embed_c = embed if embed.is_contiguous() else embed.contiguous()
        labels_c = labels
        if labels.device != device or labels.dtype != torch.int64 or not labels.is_contiguous():
            labels_c = labels.to(device=device, dtype=torch.int64).contiguous()
        B, D, h, w = embed_c.shape
        if labels_c.dim() != 3 or labels_c.shape[0] != B:
            raise _abi.PclError("labels must be (B, Himg, Wimg)")
        seg_c = pred_c = None
        if seg is not None:
            seg_c = seg.detach()
            if seg_c.dtype not in DTYPE_CODES:          # bf16 / fp16 logits are read as they are (autocast)
                seg_c = seg_c.to(torch.float32)
            if not seg_c.is_contiguous():
                seg_c = seg_c.contiguous()
            if seg_c.shape[0] != B or tuple(seg_c.shape[2:]) != (h, w):
                raise _abi.PclError("seg must be (B, K, h, w) at the embedding resolution")
        elif predict is not None:
            pred_c = predict.to(device=device, dtype=torch.int64).contiguous()
        else:
            raise _abi.PclError("either seg or predict is required")
        mode, bank_K, M0, M1 = 0, 0, 0, 0
        segq_c = pixq_c = None
        if segq is not None:
            mode = 1
            segq_c = segq.detach()
            if segq_c.dtype != torch.float32 or not segq_c.is_contiguous():
                segq_c = segq_c.to(torch.float32).contiguous()
            bank_K, M0 = segq_c.shape[0], segq_c.shape[1]
            if pixq is not None:
                pixq_c = pixq.detach()
                if pixq_c.dtype != torch.float32 or not pixq_c.is_contiguous():
                    pixq_c = pixq_c.to(torch.float32).contiguous()
                M1 = pixq_c.shape[1]
            if segq_c.shape[2] != D:
                raise _abi.PclError("bank feature dim differs from the embedding dim")
            if _BANK_READERS:
                _flush_bank(device.index, segq_c.data_ptr())
        K = opts.num_classes or (seg_c.shape[1] if seg_c is not None else (bank_K if mode == 1 else _abi.MAX_CLASSES))
        if seg_c is not None and seg_c.shape[1] != K:
            raise _abi.PclError("num_classes differs from the number of seg planes")
        key = (B, D, h, w, labels_c.shape[1], labels_c.shape[2], K, opts.max_samples, opts.max_views,
               opts.ignore_label, mode, bank_K, M0, M1)
        lst = _WS_CACHE.get((device.index, key))
        ws = None
        if lst:
            for cand in lst:
                if not cand.busy:
                    ws = cand
                    _LAST_WS[device.index] = ws
                    break
        if ws is None:
            geom = _abi.Geom(B, D, h, w, labels_c.shape[1], labels_c.shape[2], K, opts.max_samples, opts.max_views,
                             opts.ignore_label)
            ws = _get_workspace(device, key, geom, mode, bank_K, M0, M1)
        d = ws.desc
        d.embed, d.labels = embed_c.data_ptr(), labels_c.data_ptr()
        d.seg = _abi.ptr(seg_c)
        # every call: the descriptor is cached with the workspace, an fp32 call after a half one must not inherit its types
        d.embed_dtype = embed_dt
        d.seg_dtype = DTYPE_CODES[seg_c.dtype] if seg_c is not None else _abi.DT_F32
        d.predict = _abi.ptr(pred_c)
        d.segment_queue, d.pixel_queue = _abi.ptr(segq_c), _abi.ptr(pixq_c)
        d.temperature, d.base_temperature = opts.temperature, opts.base_temperature
        d.nan_safe = int(opts.nan_safe)
        d.normalize = int(opts.normalize)
        ws.set_topk(int(opts.topk_negatives or 0))
        d.precision = 0
        shadow_c = None
        if opts.precision == "bf16":
            if not ws.tc_ok:
                raise _abi.PclError("precision='bf16' (wgmma sweep) needs proj_dim == 256")
            d.precision = 1
            d.contrast_norm_bound = float(opts.contrast_norm_bound)
            if mode == 1:
                if pixq_c is None or M0 != M1:
                    raise _abi.PclError("the tensor sweep reads the bank as (segment_queue, pixel_queue) of equal size")
                if shadow is None:           # no maintained shadow: rebuild it from the fp32 queues (one extra pass)
                    from .bank import shadow_rows
                    shadow = torch.empty((shadow_rows(bank_K, M0), D), dtype=torch.bfloat16, device=device)
                    with torch.cuda.device(device):
                        _abi.check(lib.pcl_bank_shadow_rebuild(segq_c.data_ptr(), pixq_c.data_ptr(), bank_K, M0, D,
                                                               shadow.data_ptr(), _stream_ptr(device)),
                                   "pcl_bank_shadow_rebuild")
                shadow_c = shadow
                d.shadow_bf16, d.shadow_rows = shadow_c.data_ptr(), shadow_c.shape[0]
        elif opts.precision != "fp32":
            raise _abi.PclError(f"unknown precision {opts.precision!r}")
        _step_counter[0] += 1
        d.seed = (int(opts.seed) * 0x9E3779B97F4A7C15 + _step_counter[0]) & 0xFFFFFFFFFFFFFFFF
        out = torch.empty((), dtype=torch.float32, device=device)     # the loss is written here directly
        d.loss = out.data_ptr()
        with _on_device(device):
            stream = _stream_ptr(device)
            _abi.check(lib.pcl_step_stats(C.byref(d), stream), "pcl_step_stats")
            if opts.perm_fn is not None or opts.rng == "torch_cpu":
                # reference RNG stream: one small D2H copy (B*2K int32), then randperm in the reference's order
                counts = ws.counts.view(B, 2 * K).cpu().numpy()
                pairs, TC, V = _rng.host_plan(counts, opts.max_samples, opts.max_views)
                table = _rng.anchor_rank_table(pairs, V, opts.perm_fn or (lambda n: torch.randperm(n)))
                flat = table[:max(TC, 1), :max(V, 1)].reshape(-1)
                n = min(flat.numel(), ws.ranks.numel())
                ws.ranks_host[:n].copy_(flat[:n])
                ws.ranks[:n].copy_(ws.ranks_host[:n], non_blocking=True)
                d.ranks = ws.ranks.data_ptr()
            elif opts.rng == "device":
                d.ranks = None
            else:
                raise _abi.PclError(f"unknown rng mode {opts.rng!r}")
            _abi.check(lib.pcl_step_forward(C.byref(d), stream), "pcl_step_forward")
        ctx.ws = ws
        ctx.sink = _sink_of(embed)               # embed IS the zn of a sparse_grad head: hand it the anchor columns
        ctx.embed_shape, ctx.embed_dtype = tuple(embed_c.shape), embed_c.dtype
        ctx.keep = (embed_c, labels_c, seg_c, pred_c, segq_c, pixq_c, shadow_c)   # keep inputs alive until kernels ran
        if ctx.needs_input_grad[0]:          # (grad mode is always off inside forward: ask the ctx, not torch)
            ws.busy = True
            ws.token += 1
            ctx.token = ws.token
            if mode == 1:
                ws.bank_key = (device.index, segq_c.data_ptr())
                _BANK_READERS.setdefault(ws.bank_key, []).append(ws)
            # if the graph is dropped without a backward (e.g. a loss that is only logged) give the workspace back
            weakref.finalize(ctx, _release_workspace, ws, ws.token).atexit = False
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        lib = _abi.load()
        ws = ctx.ws
        device = ws.device
        # The backward sweep re-reads the workspace scratch and the input tensors of THIS forward.  Both are handed back
        # after the first backward (another forward may have overwritten them since), so a second backward through the
        # same node (retain_graph=True) cannot be served: fail loudly instead of returning a gradient of something else.
        if ctx.keep is None or ws.token != getattr(ctx, "token", None):
            raise _abi.PclError("pixel_contrast_loss: backward ran twice on the same graph (retain_graph=True is not "
                                "supported: the engine keeps no copy of the forward's scratch); call the loss again")
        go = grad_out
        if go.device != device or go.dtype != torch.float32 or not go.is_contiguous():
            go = go.detach().to(device=device, dtype=torch.float32).contiguous()
        d = ws.desc
        d.embed_dtype = DTYPE_CODES[ctx.embed_dtype]
        sink = ctx.sink if ctx.sink is not None and ctx.sink.accepts() else None
        if sink is not None:                 # the anchor columns go to the head's backward, zn gets a zero placeholder
            ms = ws.geom.max_samples
            cols = torch.empty((ms, ws.geom.D), dtype=torch.float32, device=device)
            col_pix = torch.empty(ms, dtype=torch.int32, device=device)
            with _on_device(device):
                _abi.check(lib.pcl_step_backward_cols(C.byref(d), go.data_ptr(), cols.data_ptr(), col_pix.data_ptr(),
                                                      _stream_ptr(device)), "pcl_step_backward_cols")
            grad = sink.deposit(cols, col_pix, ctx.embed_shape)
        else:
            grad = torch.empty(ctx.embed_shape, dtype=ctx.embed_dtype, device=device)     # written in embed's dtype
            d.grad_embed = grad.data_ptr()
            with _on_device(device):
                _abi.check(lib.pcl_step_backward(C.byref(d), go.data_ptr(), _stream_ptr(device)), "pcl_step_backward")
        _release_workspace(ws, getattr(ctx, "token", ws.token))     # also applies bank writes held back for this backward
        ctx.keep = None
        return grad, None, None, None, None, None, None, None


def pixel_contrast_loss(embed: torch.Tensor, labels: torch.Tensor, *, seg: Optional[torch.Tensor] = None,
                        predict: Optional[torch.Tensor] = None, segment_queue: Optional[torch.Tensor] = None,
                        pixel_queue: Optional[torch.Tensor] = None, bank_shadow: Optional[torch.Tensor] = None,
                        options: Optional[ContrastOptions] = None):
    """Pixel-contrast loss (lib/loss/loss_contrast.py:130-147 / loss_contrast_mem.py:154-171) on the GPU engine.

    embed (B,D,h,w) fp32, bf16 or fp16 CUDA; labels (B,Himg,Wimg) int64; either seg (B,K,h,w) logits (fp32, bf16 or
    fp16; argmax fused) or predict (B,h,w) int64; optional bank queues (K,M,D) fp32.  Returns a 0-dim fp32 tensor with
    autograd to embed; the gradient has embed's dtype.  Half inputs are read in place and converted on load, so loss
    and gradient equal those of the fp32 copies (the gradient rounded once)."""
    return _PixelContrastFn.apply(embed, labels, seg, predict, segment_queue, pixel_queue, bank_shadow,
                                  options or ContrastOptions())


def last_workspace(embed_device: torch.device):
    """Workspace used by the most recent loss call on a device (diagnostics / tests)."""
    return _LAST_WS.get(embed_device.index)


# ------------------------------------------------------------------------------------------------
# direct InfoNCE on explicit anchors / contrast rows (S4 sweeps, kernel tests)
# ------------------------------------------------------------------------------------------------
def infonce_forward(anchors: torch.Tensor, anchor_cls: torch.Tensor, *, contrast: Optional[torch.Tensor] = None,
                    contrast_cls: Optional[torch.Tensor] = None, queues: Optional[Tuple[torch.Tensor, ...]] = None,
                    diag_col: Optional[torch.Tensor] = None, temperature: float = 0.1, base_temperature: float = 0.07,
                    nan_safe: bool = False, topk: Optional[int] = None):
    """Returns (loss (1,), rowstats (6, A), desc-state) for the exact fp32 sweep.
    Modes: self-contrast (contrast None, queues None), explicit matrix (contrast given), bank (queues given).
    Bank mode expects the anchors grouped by class in the engine's row order (class rank 1, 2, ..., K-1, 0 — what the
    selection kernel produces): the positive sweep only visits the column range of a row tile's classes.
    topk=k keeps only the k hardest negatives of every anchor (a10 extension; None = all, the reference)."""
    lib = _abi.load()
    _require_cuda(anchors, "anchors")
    dev = anchors.device
    a = anchors.detach().to(torch.float32).contiguous()
    A, D = a.shape
    cls = anchor_cls.to(device=dev, dtype=torch.int32).contiguous()
    sw = _abi.SweepDesc()
    sw.anchors, sw.anchor_cls = a.data_ptr(), cls.data_ptr()
    dg = None
    if diag_col is not None:
        dg = diag_col.to(device=dev, dtype=torch.int32).contiguous()
        sw.diag_col = dg.data_ptr()
    sw.a_rows, sw.D = A, D
    keep = [a, cls, dg]
    if queues is not None:
        sw.mode = 1
        sq = queues[0].detach().to(torch.float32).contiguous()
        pq = queues[1].detach().to(torch.float32).contiguous() if len(queues) > 1 and queues[1] is not None else None
        sw.segment_queue, sw.pixel_queue = sq.data_ptr(), _abi.ptr(pq)
        sw.bank_K, sw.bank_M0, sw.bank_M1 = sq.shape[0], sq.shape[1], (pq.shape[1] if pq is not None else 0)
        keep += [sq, pq]
    elif contrast is not None:
        sw.mode = 2
        c = contrast.detach().to(torch.float32).contiguous()
        cc = contrast_cls.to(device=dev, dtype=torch.int32).contiguous()
        sw.contrast, sw.contrast_cls, sw.n_cols = c.data_ptr(), cc.data_ptr(), c.shape[0]
        keep += [c, cc]
    else:
        sw.mode = 0
    sw.temperature, sw.base_temperature, sw.nan_safe = temperature, base_temperature, int(nan_safe)
    ss = _abi.SweepSizes()
    _abi.check(lib.pcl_sweep_sizes(C.byref(sw), C.byref(ss)), "pcl_sweep_sizes")
    partials = torch.empty(5 * ss.partial_f32, dtype=torch.float32, device=dev)
    rowstats = torch.empty(6 * ss.rowstat_f32, dtype=torch.float32, device=dev)
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    if topk is not None:
        n = lib.pcl_topk_scratch_u32(C.byref(sw))
        if n < 0:
            _abi.check(int(n), "pcl_topk_scratch_u32")
        scratch = torch.empty(n, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _abi.check(lib.pcl_infonce_topk_fwd(C.byref(sw), int(topk), scratch.data_ptr(), partials.data_ptr(),
                                                rowstats.data_ptr(), loss.data_ptr(), _stream_ptr(dev)),
                       "pcl_infonce_topk_fwd")
        return loss, rowstats.view(6, A), (sw, ss, keep, int(topk), scratch)
    with torch.cuda.device(dev):
        _abi.check(lib.pcl_infonce_fwd(C.byref(sw), partials.data_ptr(), rowstats.data_ptr(), loss.data_ptr(),
                                       _stream_ptr(dev)), "pcl_infonce_fwd")
    return loss, rowstats.view(6, A), (sw, ss, keep)


def topk_selection(state, a_rows: int):
    """Selection result of a topk forward (diagnostics/tests): (tau_key uint32 as int64, tie_weight f32, n_above, n_ties)."""
    scratch = state[-1]                      # (exact sweep: 5-tuple, tensor sweep: 6-tuple; the scratch comes last)
    sel = scratch[scratch.numel() - 4 * a_rows:].view(4, a_rows)
    key = sel[0].to(torch.int64) & 0xFFFFFFFF
    return key, sel[1].view(torch.float32), sel[2].to(torch.int64) & 0xFFFFFFFF, sel[3].to(torch.int64) & 0xFFFFFFFF


def infonce_backward(state, rowstats: torch.Tensor, grad_loss: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _abi.load()
    sw, ss, keep = state[:3]
    dev = keep[0].device
    dpart = torch.empty(ss.dpartial_f32, dtype=torch.float32, device=dev)
    dA = torch.empty((sw.a_rows, sw.D), dtype=torch.float32, device=dev)
    if len(state) == 5:                          # forward ran with topk: same scratch (selection result) in the backward
        k, scratch = state[3], state[4]
        with torch.cuda.device(dev):
            _abi.check(lib.pcl_infonce_topk_bwd(C.byref(sw), k, scratch.data_ptr(), rowstats.contiguous().data_ptr(),
                                                _abi.ptr(grad_loss), dpart.data_ptr(), dA.data_ptr(), _stream_ptr(dev)),
                       "pcl_infonce_topk_bwd")
        return dA
    with torch.cuda.device(dev):
        _abi.check(lib.pcl_infonce_bwd(C.byref(sw), rowstats.contiguous().data_ptr(), _abi.ptr(grad_loss),
                                       dpart.data_ptr(), dA.data_ptr(), _stream_ptr(dev)), "pcl_infonce_bwd")
    return dA


# ------------------------------------------------------------------------------------------------
# a1: projection-head normalise (lib/models/modules/projection.py:24)
# ------------------------------------------------------------------------------------------------
class _L2NormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        lib = _abi.load()
        _require_cuda(x, "x")
        xc = x.to(torch.float32).contiguous()
        B, D = xc.shape[0], xc.shape[1]
        HW = xc.numel() // (B * D)
        y = torch.empty_like(xc)
        with torch.cuda.device(xc.device):
            _abi.check(lib.pcl_l2norm_fwd(xc.data_ptr(), y.data_ptr(), B, D, HW, _stream_ptr(xc.device)), "pcl_l2norm_fwd")
        ctx.save_for_backward(xc)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy):
        lib = _abi.load()
        (xc,) = ctx.saved_tensors
        B, D = xc.shape[0], xc.shape[1]
        HW = xc.numel() // (B * D)
        g = gy.to(torch.float32).contiguous()
        gx = torch.empty_like(xc)
        with torch.cuda.device(xc.device):
            _abi.check(lib.pcl_l2norm_bwd(xc.data_ptr(), g.data_ptr(), gx.data_ptr(), B, D, HW, _stream_ptr(xc.device)),
                       "pcl_l2norm_bwd")
        return gx


def l2_normalize(x: torch.Tensor) -> torch.Tensor:
    """F.normalize(x, p=2, dim=1) for (B, D, ...) CUDA tensors on the engine kernel."""
    return _L2NormFn.apply(x)


# ------------------------------------------------------------------------------------------------
# §8f row 2: projection head's last 1x1 conv + L2 normalise as one wgmma GEMM (lib/models/modules/projection.py:17-24)
# ------------------------------------------------------------------------------------------------
PROJ_DIM = 256


def _proj_dims(x: torch.Tensor, weight: torch.Tensor):
    if x.dim() != 4:
        raise _abi.PclError(f"project_normalize: x must be (B, Cin, H, W), got {tuple(x.shape)}")
    B, Cin, H, W = x.shape
    if weight.shape[0] != PROJ_DIM or weight.numel() != PROJ_DIM * Cin:
        raise _abi.PclError(f"project_normalize: weight must be ({PROJ_DIM}, {Cin}, 1, 1), got {tuple(weight.shape)}")
    return B, Cin, H * W


# activation dtypes of the fused head -> PCL_DT_* code (fp16 is refused: its values would be rounded to the bf16 operands)
_PROJ_DTYPES = {torch.float32: _abi.DT_F32, torch.bfloat16: _abi.DT_BF16}


def proj_dtype_code(dtype: torch.dtype, what: str = "project_normalize") -> int:
    """PCL_DT_* code of a fused-head activation dtype; PclError for anything but float32 / bfloat16."""
    code = _PROJ_DTYPES.get(dtype)
    if code is None:
        raise _abi.PclError(f"{what}: x must be float32 or bfloat16, got {dtype}")
    return code


def _conv1x1_f32(weight, bias, rows, cols, dev):
    """A 1x1 conv's weight as a contiguous fp32 (rows, cols) matrix on dev, its bias as contiguous fp32 (or None)."""
    w = weight.detach().to(device=dev, dtype=torch.float32).reshape(rows, cols).contiguous()
    return w, None if bias is None else bias.detach().to(device=dev, dtype=torch.float32).contiguous()


def _proj_pack(lib, x, weight, bias, s):
    """For the fused last conv on x (B, Cin, H, W): wpack (pcl_proj_pack), the fp32 (256, Cin) weight, the fp32 bias or
    None and inv_norm."""
    B, Cin, HW, dev = x.shape[0], x.shape[1], x[0, 0].numel(), x.device
    w, bc = _conv1x1_f32(weight, bias, PROJ_DIM, Cin, dev)
    wpack = torch.empty(lib.pcl_proj_workspace_bytes(B, Cin, HW, 0), dtype=torch.uint8, device=dev)
    inv = torch.empty(B * HW, dtype=torch.float32, device=dev)
    _abi.check(lib.pcl_proj_pack(w.data_ptr(), Cin, wpack.data_ptr(), s), "pcl_proj_pack")
    return wpack, w, bc, inv


def _zn_buffer(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """zn (B, 256, H, W) of x's dtype for the fused last conv on x: ``out`` when given (checked by _check_zn_out)."""
    if out is not None:
        return out
    return torch.empty((x.shape[0], PROJ_DIM) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device)


def _check_zn_out(name: str, x: torch.Tensor, out: Optional[torch.Tensor]) -> None:
    """out= of the fused BN heads: a contiguous (B, 256, H, W) tensor of zn's dtype (x's) on x's device that nobody
    differentiates through, e.g. the static embed of a captured contrast step (zn written in place, no copy)."""
    if out is None:
        return
    shape = (x.shape[0], PROJ_DIM) + tuple(x.shape[2:])
    if (tuple(out.shape) != shape or out.dtype != x.dtype or out.device != x.device or not out.is_contiguous()
            or out.requires_grad):
        raise _abi.PclError(f"{name}: out must be a contiguous {x.dtype} tensor of shape {shape} on {x.device} that "
                            f"does not require grad, got {out.dtype} {tuple(out.shape)} on {out.device}")


def _proj_grad_buffers(x, zn, gzn, scratch_bytes, has_bias):
    """The fused last conv's backward buffers: gzn in zn's dtype, scratch, x's gradient, gw (256, Cin), gb or None."""
    dev = x.device
    g = gzn.to(device=dev, dtype=zn.dtype).contiguous()
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    gw = torch.empty((PROJ_DIM, x.shape[1]), dtype=torch.float32, device=dev)
    gb = torch.empty(PROJ_DIM, dtype=torch.float32, device=dev) if has_bias else None
    return g, scratch, torch.empty_like(x), gw, gb


class _ProjNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        lib = _abi.load()
        _require_cuda(x, "x")
        dt = proj_dtype_code(x.dtype)
        B, Cin, HW = _proj_dims(x, weight)
        dev = x.device
        xc = x.contiguous()
        with _on_device(dev):
            s = _stream_ptr(dev)
            wpack, _, bc, inv = _proj_pack(lib, xc, weight, bias, s)
            zn = _zn_buffer(xc)
            _abi.check(lib.pcl_proj_fwd_dt(xc.data_ptr(), dt, wpack.data_ptr(), _abi.ptr(bc), B, Cin, HW, zn.data_ptr(),
                                           inv.data_ptr(), s), "pcl_proj_fwd_dt")
        ctx.save_for_backward(xc, zn, inv, wpack)
        ctx.dims = (B, Cin, HW, tuple(weight.shape), bias is not None, dt)
        return zn

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gzn):
        lib = _abi.load()
        xc, zn, inv, wpack = ctx.saved_tensors
        B, Cin, HW, wshape, has_bias, dt = ctx.dims
        g, scratch, gx, gw, gb = _proj_grad_buffers(xc, zn, gzn, lib.pcl_proj_workspace_bytes(B, Cin, HW, 1), has_bias)
        with _on_device(xc.device):
            _abi.check(lib.pcl_proj_bwd_dt(xc.data_ptr(), dt, zn.data_ptr(), inv.data_ptr(), g.data_ptr(),
                                           wpack.data_ptr(), B, Cin, HW, scratch.data_ptr(), gx.data_ptr(),
                                           gw.data_ptr(), _abi.ptr(gb), _stream_ptr(xc.device)), "pcl_proj_bwd_dt")
        return gx, gw.view(wshape), gb


def project_normalize(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.normalize(F.conv2d(x, weight, bias), p=2, dim=1) for a 1x1 convolution to 256 channels, as one bf16 wgmma GEMM
    with the normalise in its epilogue (fp32 accumulate; backward: gz in bf16, split-K weight gradient reduced in a
    fixed order).  x (B, Cin, H, W) fp32 or bf16 CUDA, weight (256, Cin, 1, 1), bias (256) or None.  zn and x's
    gradient have x's dtype; a bf16 x computes exactly what x.float() computes, with zn and the gradient rounded once to
    bf16.  The autocast state is not consulted: the dtype of x decides."""
    return _ProjNormFn.apply(x, weight, bias)


def _bn_sync_group(bn):
    """The process group a SyncBatchNorm in training mode reduces over (as torch's SyncBatchNorm.forward decides), or
    None: BatchNorm2d, eval mode, no initialised process group, or a group of one rank."""
    if not isinstance(bn, torch.nn.SyncBatchNorm) or not bn.training:
        return None
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group or dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


def _check_bn(bn) -> None:
    if not isinstance(bn, (torch.nn.BatchNorm2d, torch.nn.SyncBatchNorm)):
        raise _abi.PclError(f"bn_relu_project_normalize: bn must be BatchNorm2d or SyncBatchNorm, got {type(bn).__name__}")
    if not bn.affine or not bn.track_running_stats:
        raise _abi.PclError("bn_relu_project_normalize: bn needs affine=True and track_running_stats=True")
    if bn.momentum is None:
        raise _abi.PclError("bn_relu_project_normalize: momentum=None (cumulative moving average) is not supported")
    for name in ("weight", "bias", "running_mean", "running_var"):
        if getattr(bn, name).dtype != torch.float32:
            raise _abi.PclError(f"bn_relu_project_normalize: bn.{name} must be float32")


def _check_bn_input(what, name, x, gamma, training) -> None:
    """bn against its input x (B, C, H, W): C channels, and in training more than one value per channel (as torch)."""
    if gamma.numel() != x.shape[1]:
        raise _abi.PclError(f"{what}: bn has {gamma.numel()} channels, {name} has {x.shape[1]}")
    if training and x.shape[0] * x[0, 0].numel() == 1:
        raise ValueError(f"Expected more than 1 value per channel when training, got input size {tuple(x.shape)}")


def _bn_head_forward(lib, yc, dt, bn, gamma, beta, weight, bias, sums, group, s, out=None):
    """From conv1's output y on: (training) the all-reduce of the statistics ``sums`` for a multi-rank SyncBatchNorm and
    the counter, the BN state (batch or running statistics, running buffers updated), the last conv's packed weight
    and the fused GEMM.  Returns zn (``out`` when given), inv_norm, wpack, the fp32 weight, bn_state."""
    B, Cin, HW = yc.shape[0], yc.shape[1], yc[0, 0].numel()
    g32, b32 = gamma.detach().contiguous(), beta.detach().contiguous()
    state = torch.empty(lib.pcl_proj_bn_workspace_bytes(B, Cin, HW, 0), dtype=torch.uint8, device=yc.device)
    training = sums is not None
    if training:
        if group is not None:                            # fp64 sums and counts add up over the ranks
            torch.distributed.all_reduce(sums, group=group)
        bn.num_batches_tracked.add_(1)
    _abi.check(lib.pcl_proj_bn_finalize(_abi.ptr(sums), g32.data_ptr(), b32.data_ptr(), bn.running_mean.data_ptr(),
                                        bn.running_var.data_ptr(), Cin, bn.eps, bn.momentum, int(training),
                                        state.data_ptr(), s), "pcl_proj_bn_finalize")
    wpack, w, bc, inv = _proj_pack(lib, yc, weight, bias, s)
    zn = _zn_buffer(yc, out)
    _abi.check(lib.pcl_proj_bn_fwd_dt(yc.data_ptr(), dt, state.data_ptr(), wpack.data_ptr(), _abi.ptr(bc), B, Cin, HW,
                                      zn.data_ptr(), inv.data_ptr(), s), "pcl_proj_bn_fwd_dt")
    return zn, inv, wpack, w, state


def _bn_head_backward(lib, yc, dt, zn, inv, wpack, w2, state, gzn, has_bias, training, group, sink, s):
    """The backward of _bn_head_forward: returns the gradients of y, gamma, beta (rank-local), weight (256, Cin) and
    bias (or None).  sink (sparse_grad): the column path when gzn is its placeholder, else the dense path on gzn plus
    the sink's deposits."""
    if sink is not None:
        if sink.is_placeholder(gzn):
            ((cols, col_pix),) = sink.take()
            return _bn_head_backward_cols(lib, yc, dt, zn, inv, w2, state, cols, col_pix, has_bias, training, group, s)
        deposits = sink.take()
        if deposits:
            gzn = _with_deposits(gzn, deposits, zn.dtype)
    B, Cin, HW = yc.shape[0], yc.shape[1], yc[0, 0].numel()
    dev = yc.device
    g, scratch, gy, gw, gb = _proj_grad_buffers(yc, zn, gzn, lib.pcl_proj_bn_workspace_bytes(B, Cin, HW, 1), has_bias)
    gsum = torch.empty(2 * Cin, dtype=torch.float32, device=dev)
    ggamma = torch.empty(Cin, dtype=torch.float32, device=dev)
    gbeta = torch.empty(Cin, dtype=torch.float32, device=dev)
    _abi.check(lib.pcl_proj_bn_bwd_dt(yc.data_ptr(), dt, state.data_ptr(), zn.data_ptr(), inv.data_ptr(), g.data_ptr(),
                                      wpack.data_ptr(), B, Cin, HW, scratch.data_ptr(), gy.data_ptr(), gw.data_ptr(),
                                      _abi.ptr(gb), gsum.data_ptr(), ggamma.data_ptr(), gbeta.data_ptr(), s),
               "pcl_proj_bn_bwd_dt")
    if training and group is not None:                   # gamma / beta gradients stay rank-local, as in torch
        torch.distributed.all_reduce(gsum, group=group)
    _abi.check(lib.pcl_proj_bn_input_grad_dt(yc.data_ptr(), dt, state.data_ptr(), gsum.data_ptr(), B, Cin, HW,
                                             int(training), gy.data_ptr(), s), "pcl_proj_bn_input_grad_dt")
    return gy, ggamma, gbeta, gw, gb


def _bn_head_backward_cols(lib, yc, dt, zn, inv, w2, state, cols, col_pix, has_bias, training, group, s):
    """_bn_head_backward from the anchor columns of gzn alone (zero elsewhere): the last conv's gradients and the BN
    backward's sums over the columns, then the dense gradient of y from y and those sums."""
    B, Cin, HW = yc.shape[0], yc.shape[1], yc[0, 0].numel()
    dev = yc.device
    n = col_pix.numel()
    scratch = _byte_scratch(lib.pcl_proj_bn_cols_workspace_bytes(n, Cin), "pcl_proj_bn_cols_workspace_bytes", dev)
    gw = torch.empty((PROJ_DIM, Cin), dtype=torch.float32, device=dev)
    gb = torch.empty(PROJ_DIM, dtype=torch.float32, device=dev) if has_bias else None
    gsum = torch.empty(2 * Cin, dtype=torch.float32, device=dev)
    ggamma = torch.empty(Cin, dtype=torch.float32, device=dev)
    gbeta = torch.empty(Cin, dtype=torch.float32, device=dev)
    _abi.check(lib.pcl_proj_bn_bwd_cols_dt(yc.data_ptr(), dt, state.data_ptr(), zn.data_ptr(), inv.data_ptr(),
                                           cols.data_ptr(), col_pix.data_ptr(), n, w2.data_ptr(), B, Cin, HW,
                                           scratch.data_ptr(), gw.data_ptr(), _abi.ptr(gb), gsum.data_ptr(),
                                           ggamma.data_ptr(), gbeta.data_ptr(), s), "pcl_proj_bn_bwd_cols_dt")
    if training and group is not None:                   # gamma / beta gradients stay rank-local, as in torch
        torch.distributed.all_reduce(gsum, group=group)
    gy = torch.empty_like(yc)
    _abi.check(lib.pcl_proj_bn_input_grad_cols_dt(yc.data_ptr(), dt, state.data_ptr(), gsum.data_ptr(),
                                                  scratch.data_ptr(), col_pix.data_ptr(), n, B, Cin, HW, int(training),
                                                  gy.data_ptr(), s), "pcl_proj_bn_input_grad_cols_dt")
    return gy, ggamma, gbeta, gw, gb


def _sparse_output(zn: torch.Tensor, sparse_grad: bool) -> torch.Tensor:
    """A sparse_grad head's zn registered as the sink of the engine loss that reads it (when autograd records zn)."""
    if sparse_grad and zn.grad_fn is not None:
        zn.grad_fn.sink = _register_sink(zn)
    return zn


class _BnProjNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, gamma, beta, weight, bias, bn, sparse_grad, out):
        lib = _abi.load()
        _require_cuda(y, "y")
        dt = proj_dtype_code(y.dtype, "bn_relu_project_normalize")
        B, Cin, HW = _proj_dims(y, weight)
        _check_zn_out("bn_relu_project_normalize", y, out)
        training = bn.training
        _check_bn_input("bn_relu_project_normalize", "y", y, gamma, training)
        group = _bn_sync_group(bn)
        dev = y.device
        yc = y.contiguous()
        with _on_device(dev):
            s = _stream_ptr(dev)
            sums = None
            if training:
                sums = torch.empty(2 * Cin + 1, dtype=torch.float64, device=dev)
                _abi.check(lib.pcl_proj_bn_stats_dt(yc.data_ptr(), dt, B, Cin, HW, sums.data_ptr(), s),
                           "pcl_proj_bn_stats_dt")
            zn, inv, wpack, w2, state = _bn_head_forward(lib, yc, dt, bn, gamma, beta, weight, bias, sums, group, s,
                                                         out)
        if out is not None:                  # a fresh alias: autograd's history goes on it, not on the caller's buffer
            zn = out.view_as(out)
        ctx.save_for_backward(yc, zn, inv, wpack, w2 if sparse_grad else None, state)
        ctx.meta = (tuple(weight.shape), bias is not None, dt, training, group, gamma.dtype)
        ctx.sink = None
        return zn

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gzn):
        lib = _abi.load()
        yc, zn, inv, wpack, w2, state = ctx.saved_tensors
        wshape, has_bias, dt, training, group, gdtype = ctx.meta
        dev = yc.device
        with _on_device(dev):
            gy, ggamma, gbeta, gw, gb = _bn_head_backward(lib, yc, dt, zn, inv, wpack, w2, state, gzn, has_bias,
                                                          training, group, ctx.sink, _stream_ptr(dev))
        return gy, ggamma.to(gdtype), gbeta.to(gdtype), gw.view(wshape), gb, None, None, None


def bn_relu_project_normalize(y: torch.Tensor, bn: torch.nn.Module, weight: torch.Tensor,
                              bias: Optional[torch.Tensor] = None, *, sparse_grad: bool = False,
                              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.normalize(F.conv2d(relu(bn(y)), weight, bias), p=2, dim=1): the projection head from the output y of its
    first conv to zn, with bn a BatchNorm2d or SyncBatchNorm (affine, tracking running stats, numeric momentum).  In
    training mode the batch statistics (fp64 sums; over all ranks of a SyncBatchNorm's process group, one all_reduce
    each way) normalise y, and running_mean / running_var / num_batches_tracked are updated as nn.BatchNorm2d does; in
    eval mode the running statistics are used.  The BN output and the ReLU output are never written: the GEMMs apply
    max(0, y scale + shift) where they convert their activation tile.  y (B, Cin, H, W) fp32 or bf16 CUDA, as for
    project_normalize; autograd reaches y, bn.weight, bn.bias, weight and bias (bn's gradients rank-local).
    sparse_grad=True: an engine contrast loss whose embed is the returned zn hands this node its anchor columns instead
    of a dense gradient, and zn itself receives a zero placeholder (INTEGRATION §1); the backward then runs over those
    columns only.
    out: zn is written into this (B, 256, H, W) tensor of y's dtype (contiguous, not requiring grad) and the result
    shares its storage, e.g. the static embed of a GraphedContrastStep, whose apply() and column hand-off accept it."""
    _check_bn(bn)
    return _sparse_output(_BnProjNormFn.apply(y, bn.weight, bn.bias, weight, bias, bn, bool(sparse_grad), out),
                          sparse_grad)


class _ConvBnProjNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, b1, gamma, beta, w2, b2, bn, sparse_grad, out):
        lib = _abi.load()
        _require_cuda(x, "x")
        dt = proj_dtype_code(x.dtype, "conv_bn_relu_project_normalize")
        B, C, HW = _proj_dims(x, w2)
        _check_zn_out("conv_bn_relu_project_normalize", x, out)
        if w1.shape[0] != C or w1.numel() != C * C:
            raise _abi.PclError(f"conv_bn_relu_project_normalize: w1 must be ({C}, {C}, 1, 1), got {tuple(w1.shape)}")
        if b1 is not None and b1.numel() != C:
            raise _abi.PclError(f"conv_bn_relu_project_normalize: b1 must have {C} elements, got {b1.numel()}")
        training = bn.training
        _check_bn_input("conv_bn_relu_project_normalize", "x", x, gamma, training)
        group = _bn_sync_group(bn)
        dev = x.device
        xc = x.contiguous()
        w, bc = _conv1x1_f32(w1, b1, C, C, dev)
        pack = torch.empty(lib.pcl_proj_conv1_workspace_bytes(B, C, HW, 0), dtype=torch.uint8, device=dev)
        y = torch.empty_like(xc)
        with _on_device(dev):
            s = _stream_ptr(dev)
            sums = scratch = None
            if training:                                 # the statistics of y come out of conv1's epilogue
                sums = torch.empty(2 * C + 1, dtype=torch.float64, device=dev)
                scratch = torch.empty(lib.pcl_proj_conv1_workspace_bytes(B, C, HW, 1), dtype=torch.uint8, device=dev)
            _abi.check(lib.pcl_proj_conv1_pack(w.data_ptr(), C, pack.data_ptr(), s), "pcl_proj_conv1_pack")
            _abi.check(lib.pcl_proj_conv1_fwd_dt(xc.data_ptr(), dt, pack.data_ptr(), _abi.ptr(bc), B, C, HW,
                                                 y.data_ptr(), _abi.ptr(sums), _abi.ptr(scratch), s),
                       "pcl_proj_conv1_fwd_dt")
            zn, inv, wpack, w2f, state = _bn_head_forward(lib, y, dt, bn, gamma, beta, w2, b2, sums, group, s, out)
        if out is not None:                  # a fresh alias: autograd's history goes on it, not on the caller's buffer
            zn = out.view_as(out)
        ctx.save_for_backward(xc, y, zn, inv, pack, wpack, w2f if sparse_grad else None, state)
        ctx.sink = None
        ctx.meta = (tuple(w1.shape), b1 is not None, tuple(w2.shape), b2 is not None, dt, training, group, gamma.dtype)
        return zn

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gzn):
        lib = _abi.load()
        xc, y, zn, inv, pack, wpack, w2f, state = ctx.saved_tensors
        w1shape, has_b1, w2shape, has_b2, dt, training, group, gdtype = ctx.meta
        B, C, HW = xc.shape[0], xc.shape[1], xc[0, 0].numel()
        dev = xc.device
        gx = torch.empty_like(xc) if ctx.needs_input_grad[0] else None
        gw1 = torch.empty((C, C), dtype=torch.float32, device=dev)
        gb1 = torch.empty(C, dtype=torch.float32, device=dev) if has_b1 else None
        with _on_device(dev):
            s = _stream_ptr(dev)
            gy, ggamma, gbeta, gw2, gb2 = _bn_head_backward(lib, y, dt, zn, inv, wpack, w2f, state, gzn, has_b2,
                                                            training, group, ctx.sink, s)
            scratch = torch.empty(lib.pcl_proj_conv1_workspace_bytes(B, C, HW, 2), dtype=torch.uint8, device=dev)
            _abi.check(lib.pcl_proj_conv1_bwd_dt(xc.data_ptr(), dt, gy.data_ptr(), pack.data_ptr(), B, C, HW,
                                                 scratch.data_ptr(), _abi.ptr(gx), gw1.data_ptr(), _abi.ptr(gb1), s),
                       "pcl_proj_conv1_bwd_dt")
        return (gx, gw1.view(w1shape), gb1, ggamma.to(gdtype), gbeta.to(gdtype), gw2.view(w2shape), gb2, None, None,
                None)


def conv_bn_relu_project_normalize(x: torch.Tensor, w1: torch.Tensor, b1: Optional[torch.Tensor], bn: torch.nn.Module,
                                   w2: torch.Tensor, b2: Optional[torch.Tensor] = None, *,
                                   sparse_grad: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.normalize(F.conv2d(relu(bn(F.conv2d(x, w1, b1))), w2, b2), p=2, dim=1): the whole ``convmlp`` projection head
    on the engine.  The first 1x1 convolution (w1 (C, C, 1, 1), b1 (C) or None) is a bf16 wgmma GEMM whose epilogue
    also sums the BatchNorm statistics of its output y; y then goes through bn_relu_project_normalize's kernels (same
    rules for bn: batch statistics in training with the running buffers and num_batches_tracked updated, SyncBatchNorm
    reduced over its process group, running statistics in eval).  x (B, C, H, W) fp32 or bf16 CUDA decides y's and
    zn's dtype (fp32 x is rounded to the bf16 GEMM operand).  autograd reaches x, w1, b1, bn.weight, bn.bias, w2 and b2
    (bn's gradients rank-local); x's gradient is skipped when x needs none.  No cuDNN call: forward and backward are
    capturable and bit-reproducible run to run.  sparse_grad and out as for bn_relu_project_normalize (out has x's
    dtype)."""
    _check_bn(bn)
    return _sparse_output(_ConvBnProjNormFn.apply(x, w1, b1, bn.weight, bn.bias, w2, b2, bn, bool(sparse_grad), out),
                          sparse_grad)


# ------------------------------------------------------------------------------------------------
# tensor-core (wgmma) InfoNCE on explicit operands — D must be 256
# ------------------------------------------------------------------------------------------------
def to_bf16_rows(x: torch.Tensor, rows_alloc: int) -> torch.Tensor:
    """fp32 (n, 256) -> bf16 (rows_alloc, 256) zero-padded copy on the engine's conversion kernel."""
    lib = _abi.load()
    xc = x.detach().to(torch.float32).contiguous()
    out = torch.empty((rows_alloc, xc.shape[1]), dtype=torch.bfloat16, device=xc.device)
    with torch.cuda.device(xc.device):
        _abi.check(lib.pcl_to_bf16(xc.data_ptr(), out.data_ptr(), xc.numel(), out.numel(), _stream_ptr(xc.device)),
                   "pcl_to_bf16")
    return out


def _tc_desc(anchors, anchor_cls, contrast_bf16, contrast_cls, n_cols, bank, diag_col, temperature, base_temperature,
             nan_safe, sorted_cols, norm_bound):
    dev = anchors.device
    a = anchors.detach().to(torch.float32).contiguous()
    A, D = a.shape
    a_pad = -(-A // 256) * 256                      # row tiles of the forward sweep
    a16 = torch.empty((-(-A // 128) * 128, D), dtype=torch.bfloat16, device=dev)
    cls = anchor_cls.to(device=dev, dtype=torch.int32).contiguous()
    d = _abi.TcDesc()
    d.anchors_f32, d.anchors_bf16, d.anchor_cls = a.data_ptr(), a16.data_ptr(), cls.data_ptr()
    keep = [a, a16, cls]
    if diag_col is not None:
        dg = diag_col.to(device=dev, dtype=torch.int32).contiguous()
        d.diag_col = dg.data_ptr()
        keep.append(dg)
    d.a_rows, d.D = A, D
    if bank is not None:                       # (shadow bf16, K, R)
        shadow, K, R = bank
        d.mode, d.contrast_bf16, d.bank_K, d.bank_R = 1, shadow.data_ptr(), K, R
        d.contrast_rows_alloc = shadow.shape[0]
        keep.append(shadow)
    elif contrast_bf16 is not None:
        cc = contrast_cls.to(device=dev, dtype=torch.int32).contiguous()
        d.mode, d.contrast_bf16, d.contrast_cls = 2, contrast_bf16.data_ptr(), cc.data_ptr()
        d.n_cols, d.contrast_rows_alloc, d.sorted = n_cols, contrast_bf16.shape[0], int(sorted_cols)
        keep += [contrast_bf16, cc]
    else:
        d.mode = 0
    d.contrast_norm_bound = norm_bound
    d.temperature, d.base_temperature, d.nan_safe = temperature, base_temperature, int(nan_safe)
    return d, keep, a_pad


def infonce_tc_forward(anchors: torch.Tensor, anchor_cls: torch.Tensor, *, contrast_bf16: Optional[torch.Tensor] = None,
                       contrast_cls: Optional[torch.Tensor] = None, n_cols: int = 0, bank=None,
                       diag_col: Optional[torch.Tensor] = None, temperature: float = 0.1, base_temperature: float = 0.07,
                       nan_safe: bool = False, sorted_cols: bool = True, norm_bound: float = 1.0, neg_only: bool = False,
                       topk: Optional[int] = None):
    """bf16 wgmma sweep.  Returns (loss (1,), rowstats (6, A), state).  neg_only=True runs just the similarity +
    negative-sum sweep (roofline measurement of the dense contraction).  topk=k: a10, the k hardest negatives per anchor
    (radix select in the sweep's epilogue)."""
    lib = _abi.load()
    _require_cuda(anchors, "anchors")
    dev = anchors.device
    d, keep, a_pad = _tc_desc(anchors, anchor_cls, contrast_bf16, contrast_cls, n_cols, bank, diag_col, temperature,
                              base_temperature, nan_safe, sorted_cols, norm_bound)
    d.neg_only = int(neg_only)
    ss = _abi.SweepSizes()
    _abi.check(lib.pcl_tc_sizes(C.byref(d), C.byref(ss)), "pcl_tc_sizes")
    row_m2 = torch.empty(a_pad + 512, dtype=torch.float32, device=dev)
    partials = torch.empty(5 * ss.partial_f32, dtype=torch.float32, device=dev)
    rowstats = torch.empty(6 * ss.rowstat_f32, dtype=torch.float32, device=dev)
    loss = torch.zeros(1, dtype=torch.float32, device=dev)
    if topk is not None:
        n = lib.pcl_tc_topk_scratch_u32(C.byref(d))
        if n < 0:
            _abi.check(int(n), "pcl_tc_topk_scratch_u32")
        scratch = torch.empty(n, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _abi.check(lib.pcl_infonce_tc_topk_fwd(C.byref(d), int(topk), scratch.data_ptr(), row_m2.data_ptr(),
                                                   partials.data_ptr(), rowstats.data_ptr(), loss.data_ptr(),
                                                   _stream_ptr(dev)), "pcl_infonce_tc_topk_fwd")
        return loss, rowstats.view(6, d.a_rows), (d, ss, keep, row_m2, int(topk), scratch)
    with torch.cuda.device(dev):
        _abi.check(lib.pcl_infonce_tc_fwd(C.byref(d), row_m2.data_ptr(), partials.data_ptr(), rowstats.data_ptr(),
                                          loss.data_ptr(), _stream_ptr(dev)), "pcl_infonce_tc_fwd")
    return loss, rowstats.view(6, d.a_rows), (d, ss, keep, row_m2)


def tc_dump_logits(anchors: torch.Tensor, contrast_bf16: Optional[torch.Tensor], n_cols: int) -> torch.Tensor:
    """Raw S = A.C^T from the TMA/wgmma pipeline (self-test of descriptors and barriers)."""
    lib = _abi.load()
    dev = anchors.device
    A = anchors.shape[0]
    cls = torch.zeros(A, dtype=torch.int32, device=dev)
    ccls = torch.zeros(max(n_cols, 1), dtype=torch.int32, device=dev)
    d, keep, a_pad = _tc_desc(anchors, cls, contrast_bf16, ccls if contrast_bf16 is not None else None, n_cols, None,
                              None, 1.0, 1.0, False, False, 1.0)
    ncols = n_cols if contrast_bf16 is not None else A
    ld = -(-ncols // 256) * 256
    dump = torch.zeros((a_pad, ld), dtype=torch.float32, device=dev)
    row_m2 = torch.empty(a_pad + 512, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _abi.check(lib.pcl_tc_dump_logits(C.byref(d), row_m2.data_ptr(), dump.data_ptr(), _stream_ptr(dev)),
                   "pcl_tc_dump_logits")
    return dump[:A, :ncols]


def infonce_tc_backward(state, rowstats: torch.Tensor, grad_loss: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dA (A, 256) fp32 from the wgmma backward sweep (recompute S, G tile in shared memory, dA += G.C)."""
    lib = _abi.load()
    d, ss, keep, row_m2 = state[:4]
    dev = row_m2.device
    dpart = torch.empty(ss.dpartial_f32, dtype=torch.float32, device=dev)
    dA = torch.empty((d.a_rows, d.D), dtype=torch.float32, device=dev)
    if len(state) == 6:                          # forward ran with topk: same selection state in the backward
        with torch.cuda.device(dev):
            _abi.check(lib.pcl_infonce_tc_topk_bwd(C.byref(d), state[4], state[5].data_ptr(), row_m2.data_ptr(),
                                                   rowstats.contiguous().data_ptr(), _abi.ptr(grad_loss), dpart.data_ptr(),
                                                   dA.data_ptr(), _stream_ptr(dev)), "pcl_infonce_tc_topk_bwd")
        return dA
    with torch.cuda.device(dev):
        _abi.check(lib.pcl_infonce_tc_bwd(C.byref(d), row_m2.data_ptr(), rowstats.contiguous().data_ptr(),
                                          _abi.ptr(grad_loss), dpart.data_ptr(), dA.data_ptr(), _stream_ptr(dev)),
                   "pcl_infonce_tc_bwd")
    return dA


# ------------------------------------------------------------------------------------------------
# Operands of the fused up-sampling segmentation losses below (seg CE, RMI, Lovasz, OHEM CE)
# ------------------------------------------------------------------------------------------------
def _seg_operands(seg, target, weight=None):
    """(seg as contiguous fp32, target as contiguous int64 on seg's device, class weights as contiguous fp32 there or
    None, (B, K, h, w, H, W))."""
    _require_cuda(seg, "seg")
    dev = seg.device
    seg_c = seg if (seg.dtype == torch.float32 and seg.is_contiguous()) else seg.to(torch.float32).contiguous()
    tgt = target
    if tgt.device != dev or tgt.dtype != torch.int64 or not tgt.is_contiguous():
        tgt = tgt.to(device=dev, dtype=torch.int64).contiguous()
    wt = None if weight is None else weight.to(device=dev, dtype=torch.float32).contiguous()
    B, K, h, w = seg_c.shape
    return seg_c, tgt, wt, (B, K, h, w, tgt.shape[1], tgt.shape[2])


def _byte_scratch(n: int, name: str, dev) -> torch.Tensor:
    """The uint8 scratch of a *_scratch_bytes query; a negative n is the query's error code."""
    if n < 0:
        _abi.check(n, name)
    return torch.empty(n, dtype=torch.uint8, device=dev)


def _grad_scalar(grad_out: torch.Tensor, dev) -> torch.Tensor:
    """The incoming loss gradient as a contiguous fp32 scalar on dev."""
    if grad_out.device != dev or grad_out.dtype != torch.float32 or not grad_out.is_contiguous():
        grad_out = grad_out.detach().to(device=dev, dtype=torch.float32).contiguous()
    return grad_out


# ------------------------------------------------------------------------------------------------
# §8f row 1: fused bilinear up-sampling (align_corners=True) + weighted cross-entropy with ignore_index
# (lib/loss/loss_contrast.py:180-181 + lib/loss/loss_helper.py:169-212)
# ------------------------------------------------------------------------------------------------
class _SegCeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seg, target, weight, ignore_index):
        lib = _abi.load()
        seg_c, tgt, wt, (B, K, h, w, H, W) = _seg_operands(seg, target, weight)
        dev = seg_c.device
        scratch = torch.empty(lib.pcl_seg_ce_scratch_floats(B, H, W), dtype=torch.float32, device=dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with _on_device(dev):
            _abi.check(lib.pcl_seg_ce_fwd(seg_c.data_ptr(), tgt.data_ptr(), _abi.ptr(wt), B, K, h, w, H, W, int(ignore_index),
                                          scratch.data_ptr(), out.data_ptr(), _stream_ptr(dev)), "pcl_seg_ce_fwd")
        ctx.keep = (seg_c, tgt, wt, scratch)
        ctx.dims = (B, K, h, w, H, W, int(ignore_index))
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        lib = _abi.load()
        seg_c, tgt, wt, scratch = ctx.keep
        B, K, h, w, H, W, ign = ctx.dims
        dev = seg_c.device
        go = _grad_scalar(grad_out, dev)
        dseg = torch.empty_like(seg_c)
        with _on_device(dev):
            _abi.check(lib.pcl_seg_ce_bwd(seg_c.data_ptr(), tgt.data_ptr(), _abi.ptr(wt), B, K, h, w, H, W, ign,
                                          scratch.data_ptr(), go.data_ptr(), dseg.data_ptr(), _stream_ptr(dev)),
                       "pcl_seg_ce_bwd")
        ctx.keep = None
        return dseg, None, None, None


def upsample_cross_entropy(seg: torch.Tensor, target: torch.Tensor, weight: Optional[torch.Tensor] = None,
                           ignore_index: int = -1) -> torch.Tensor:
    """mean CE of bilinearly (align_corners=True) up-sampled logits against a full-resolution label map, fused:
    == F.cross_entropy(F.interpolate(seg, target.shape[1:], mode='bilinear', align_corners=True), target,
                       weight, ignore_index=ignore_index)  without the (B,K,Himg,Wimg) intermediate."""
    return _SegCeFn.apply(seg, target, weight, ignore_index)


def seg_ce_loss_and_grad(seg: torch.Tensor, target: torch.Tensor, weight: Optional[torch.Tensor] = None,
                         ignore_index: int = -1, grad_scale=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(loss, dseg) of upsample_cross_entropy in one tile pass (pcl_seg_ce_fwd_bwd), outside autograd, for tests and
    tools: loss is the forward's to the bit, dseg = grad_scale * d loss / d seg (grad_scale: None for 1, a float, or a
    device scalar read when the kernels run).  seg fp32, bf16 or fp16 (read as fp32); dseg comes back in seg's dtype.
    Every pixel ignored gives a NaN loss and a zero dseg.  A label grid smaller than seg raises PclError."""
    if seg.dim() != 4 or target.dim() != 3 or seg.shape[0] != target.shape[0]:
        raise ValueError(f"seg (B,K,h,w) and target (B,H,W) expected, got {tuple(seg.shape)} and {tuple(target.shape)}")
    lib = _abi.load()
    seg_c, tgt, wt, (B, K, h, w, H, W) = _seg_operands(seg.detach(), target, weight)
    dev = seg_c.device
    gs = None
    if grad_scale is not None:
        gs = _grad_scalar(grad_scale if torch.is_tensor(grad_scale) else torch.tensor(float(grad_scale)), dev)
    scratch = torch.empty(lib.pcl_seg_ce_fwd_bwd_scratch_floats(B, K, H, W), dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    dseg = torch.empty_like(seg_c)
    with _on_device(dev):
        _abi.check(lib.pcl_seg_ce_fwd_bwd(seg_c.data_ptr(), tgt.data_ptr(), _abi.ptr(wt), B, K, h, w, H, W,
                                          int(ignore_index), scratch.data_ptr(), _abi.ptr(gs), loss.data_ptr(),
                                          dseg.data_ptr(), _stream_ptr(dev)), "pcl_seg_ce_fwd_bwd")
    return loss, dseg.to(seg.dtype)


# ------------------------------------------------------------------------------------------------
# §8f row f5: fused bilinear up-sampling (align_corners=True) + RMI loss, sigmoid path
# (lib/loss/rmi_loss.py:200-402 via lib/loss/loss_helper.py:316-369)
# ------------------------------------------------------------------------------------------------
class _RmiFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seg, target, params):
        lib = _abi.load()
        seg_c, tgt, _, (B, K, h, w, H, W) = _seg_operands(seg, target)
        dev = seg_c.device
        scratch = _byte_scratch(lib.pcl_rmi_scratch_bytes(B, K, h, w, H, W, params[0], params[1], params[2]),
                                "pcl_rmi_scratch_bytes", dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with _on_device(dev):
            _abi.check(lib.pcl_rmi_fwd(seg_c.data_ptr(), tgt.data_ptr(), B, K, h, w, H, W, *params, scratch.data_ptr(),
                                       out.data_ptr(), _stream_ptr(dev)), "pcl_rmi_fwd")
        ctx.keep = (seg_c, tgt, scratch)
        ctx.dims = (B, K, h, w, H, W)
        ctx.params = params
        ctx.seg_dtype = seg.dtype
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        lib = _abi.load()
        seg_c, tgt, scratch = ctx.keep
        dev = seg_c.device
        go = _grad_scalar(grad_out, dev)
        dseg = torch.empty_like(seg_c)
        with _on_device(dev):
            _abi.check(lib.pcl_rmi_bwd(seg_c.data_ptr(), tgt.data_ptr(), *ctx.dims, *ctx.params, scratch.data_ptr(),
                                       go.data_ptr(), dseg.data_ptr(), _stream_ptr(dev)), "pcl_rmi_bwd")
        ctx.keep = None
        return dseg.to(ctx.seg_dtype), None, None


def upsample_rmi_loss(seg: torch.Tensor, target: torch.Tensor, *, num_classes: int, radius: int = 3, pool_way: int = 0,
                      pool_stride: int = 3, weight_lambda: float = 0.5, lambda_way: int = 1,
                      loss_weight: float = 1.0) -> torch.Tensor:
    """RMI loss (sigmoid path) of bilinearly (align_corners=True) up-sampled logits against a full-resolution label map,
    fused: == RMILoss(...)(F.interpolate(seg, target.shape[1:], mode='bilinear', align_corners=True), target) without
    the (B,K,Himg,Wimg) intermediates.  Labels < 0 count as 255; a pixel is valid when its label < num_classes.
    ``target`` is not modified (the reference rewrites it in place).  seg fp32, bf16 or fp16 (read as fp32); the
    gradient comes back in seg's dtype.  radius 1-4, pool_way 0 (max) or 1 (avg), pool_stride 1-4 are implemented;
    anything else, a label grid smaller than seg, or a pooled map smaller than the radius raises PclError."""
    if seg.dim() != 4 or target.dim() != 3 or seg.shape[0] != target.shape[0]:
        raise ValueError(f"seg (B,K,h,w) and target (B,H,W) expected, got {tuple(seg.shape)} and {tuple(target.shape)}")
    if seg.shape[1] != num_classes:
        raise ValueError(f"seg has {seg.shape[1]} channels, num_classes is {num_classes}")
    params = (int(radius), int(pool_way), int(pool_stride), float(weight_lambda), 1 if lambda_way else 0,
              float(loss_weight))
    return _RmiFn.apply(seg, target, params)


# ------------------------------------------------------------------------------------------------
# §8f row f6: fused bilinear up-sampling (align_corners=True) + Lovasz-softmax, only present classes
# (lib/loss/lovasz_loss.py:216-267 via FSCELOVASZLoss, lib/loss/loss_helper.py:77-124)
# ------------------------------------------------------------------------------------------------
class _LovaszFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seg, target, ignore_index):
        lib = _abi.load()
        seg_c, tgt, _, (B, K, h, w, H, W) = _seg_operands(seg, target)
        dev = seg_c.device
        scratch = _byte_scratch(lib.pcl_lovasz_scratch_bytes(B, K, h, w, H, W), "pcl_lovasz_scratch_bytes", dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        with _on_device(dev):
            _abi.check(lib.pcl_lovasz_fwd(seg_c.data_ptr(), tgt.data_ptr(), B, K, h, w, H, W, int(ignore_index),
                                          scratch.data_ptr(), out.data_ptr(), _stream_ptr(dev)), "pcl_lovasz_fwd")
        ctx.keep = (seg_c, tgt, scratch)
        ctx.dims = (B, K, h, w, H, W, int(ignore_index))
        ctx.seg_dtype = seg.dtype
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        lib = _abi.load()
        seg_c, tgt, scratch = ctx.keep
        dev = seg_c.device
        go = _grad_scalar(grad_out, dev)
        dseg = torch.empty_like(seg_c)
        with _on_device(dev):
            _abi.check(lib.pcl_lovasz_bwd(seg_c.data_ptr(), tgt.data_ptr(), *ctx.dims, scratch.data_ptr(),
                                          go.data_ptr(), dseg.data_ptr(), _stream_ptr(dev)), "pcl_lovasz_bwd")
        ctx.keep = None
        return dseg.to(ctx.seg_dtype), None, None


def upsample_lovasz_softmax(seg: torch.Tensor, target: torch.Tensor, ignore_index: int = -1) -> torch.Tensor:
    """Lovasz-softmax loss of bilinearly (align_corners=True) up-sampled logits against a full-resolution label map,
    fused: == lovasz_softmax_flat(*flatten_probas(softmax(F.interpolate(seg, target.shape[1:], mode='bilinear',
    align_corners=True), 1), target, ignore_index), only_present=True) without the (B,K,Himg,Wimg) intermediates or a
    host sync.  Pixels are pooled over the batch; labels outside [0, K) count as ignored; every pixel ignored gives 0
    with a zero gradient.  Equal errors are ordered by ascending pixel index (a stable sort), which fixes the per-pixel
    gradient where the reference leaves it unspecified.  seg fp32, bf16 or fp16 (read as fp32); the gradient comes back
    in seg's dtype; ``target`` is not modified.  A label grid smaller than seg, more than 256 classes or 2^31 label
    pixels raise PclError."""
    if seg.dim() != 4 or target.dim() != 3 or seg.shape[0] != target.shape[0]:
        raise ValueError(f"seg (B,K,h,w) and target (B,H,W) expected, got {tuple(seg.shape)} and {tuple(target.shape)}")
    return _LovaszFn.apply(seg, target, ignore_index)


# ------------------------------------------------------------------------------------------------
# §8f row f7: fused bilinear up-sampling (align_corners=True) + OHEM cross-entropy
# (FSOhemCELoss, lib/loss/loss_helper.py:215-261)
# ------------------------------------------------------------------------------------------------
_OHEM_REDUCTIONS = {"mean": 0, "elementwise_mean": 0, "sum": 1}


def _ohem_forward(seg, target, weight, ignore_index, thresh, min_kept, reduction):
    """Runs pcl_ohem_ce_fwd; returns (loss, the kept tensors, dims, scratch)."""
    lib = _abi.load()
    seg_c, tgt, wt, (B, K, h, w, H, W) = _seg_operands(seg, target, weight)
    dev = seg_c.device
    scratch = _byte_scratch(lib.pcl_ohem_ce_scratch_bytes(B, K, h, w, H, W), "pcl_ohem_ce_scratch_bytes", dev)
    out = torch.empty((), dtype=torch.float32, device=dev)
    dims = (B, K, h, w, H, W, int(ignore_index))
    with _on_device(dev):
        _abi.check(lib.pcl_ohem_ce_fwd(seg_c.data_ptr(), tgt.data_ptr(), _abi.ptr(wt), *dims, float(thresh),
                                       int(min_kept), reduction, scratch.data_ptr(), out.data_ptr(), _stream_ptr(dev)),
                   "pcl_ohem_ce_fwd")
    return out, (seg_c, tgt, wt, scratch), dims


class _OhemCeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seg, target, weight, ignore_index, thresh, min_kept, reduction):
        out, ctx.keep, ctx.dims = _ohem_forward(seg, target, weight, ignore_index, thresh, min_kept, reduction)
        ctx.seg_dtype = seg.dtype
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        lib = _abi.load()
        seg_c, tgt, wt, scratch = ctx.keep
        dev = seg_c.device
        go = _grad_scalar(grad_out, dev)
        dseg = torch.empty_like(seg_c)
        with _on_device(dev):
            _abi.check(lib.pcl_ohem_ce_bwd(seg_c.data_ptr(), tgt.data_ptr(), _abi.ptr(wt), *ctx.dims, scratch.data_ptr(),
                                           go.data_ptr(), dseg.data_ptr(), _stream_ptr(dev)), "pcl_ohem_ce_bwd")
        ctx.keep = None
        return dseg.to(ctx.seg_dtype), None, None, None, None, None, None


def _ohem_args(seg, target, reduction, min_kept):
    if seg.dim() != 4 or target.dim() != 3 or seg.shape[0] != target.shape[0]:
        raise ValueError(f"seg (B,K,h,w) and target (B,H,W) expected, got {tuple(seg.shape)} and {tuple(target.shape)}")
    if reduction not in _OHEM_REDUCTIONS:
        raise NotImplementedError(f"Reduction Error! OHEM CE reduction {reduction!r} (mean, elementwise_mean or sum)")
    return _OHEM_REDUCTIONS[reduction], max(1, int(min_kept))


def upsample_ohem_cross_entropy(seg: torch.Tensor, target: torch.Tensor, weight: Optional[torch.Tensor] = None,
                                ignore_index: int = -1, thresh: float = 0.9, min_kept: int = 100000,
                                reduction: str = "mean") -> torch.Tensor:
    """OHEM cross-entropy of bilinearly (align_corners=True) up-sampled logits against a full-resolution label map,
    fused: == FSOhemCELoss.forward(F.interpolate(seg, target.shape[1:], mode='bilinear', align_corners=True), target)
    without the (B,K,Himg,Wimg) intermediates, the sort or a host sync (the defaults of thresh and min_kept are the
    contrast configs' ohem_thresh and ohem_minkeep).  Over the counted pixels (label not
    ignore_index and inside [0, K)) of the whole batch, p_t is the softmax of the target class; the pixels with
    p_t < max(kth, thresh) are kept, kth the min(max(1, min_kept), n - 1)-th smallest p_t (0-based), thresh compared in
    fp32.  reduction 'mean' (or 'elementwise_mean') divides the weighted NLL sum by the kept count (not by the sum of the
    weights), 'sum' does not; anything else raises NotImplementedError.  No counted pixel gives 0 with a zero gradient;
    an empty selection gives NaN ('mean') or 0 ('sum') with a zero gradient.  seg fp32, bf16 or fp16 (read as fp32); the
    gradient comes back in seg's dtype; ``target`` is not modified.  A label grid smaller than seg, more than 256
    classes or 2^31 label pixels raise PclError."""
    red, mk = _ohem_args(seg, target, reduction, min_kept)
    return _OhemCeFn.apply(seg, target, weight, ignore_index, float(thresh), mk, red)


def ohem_selection(seg: torch.Tensor, target: torch.Tensor, weight: Optional[torch.Tensor] = None,
                   ignore_index: int = -1, thresh: float = 0.9, min_kept: int = 100000,
                   reduction: str = "mean") -> dict:
    """The forward of upsample_ohem_cross_entropy with what it decided, for tests and measurement: the loss, the
    threshold, which branch set it ("select": the exact select of the kth value ran; "threshold": fp32(thresh) decided
    without it), the counted pixels n, the selected count and the (B,Himg,Wimg) bool mask of the selected pixels (the
    stored p_t < threshold, exactly the pixels the backward reads as selected).  Synchronises with the device."""
    red, mk = _ohem_args(seg, target, reduction, min_kept)
    with torch.no_grad():
        out, keep, dims = _ohem_forward(seg, target, weight, ignore_index, float(thresh), mk, red)
    scratch = keep[3]
    B, H, W = dims[0], dims[4], dims[5]
    head = scratch[:28].cpu()
    f = head[:12].view(torch.float32)
    i = head[12:28].view(torch.int32)
    p = scratch[256:256 + 4 * B * H * W].view(torch.float32).view(B, H, W)
    thr = float(f[2])
    return {"loss": out, "threshold": thr, "branch": "select" if int(i[0]) else "threshold", "n": int(i[1]),
            "count": int(i[3]), "selected": p < thr, "p": p}
