"""The whole contrast criterion (ContrastCELoss, ContrastAuxCELoss, MemContrastCELoss with with_embed=True), forward and
backward, replayed as one CUDA graph.

GraphedContrastStep captures the contrast half.  This object captures the seg half into the same graph (the step's
first graph on several ranks), with the kernels the eager wrapper runs for the same criterion (the wrapper's
``seg_terms``), and sums the total loss in the graph with the wrapper's fp32 operations in its order.  The upstream
gradient of every term is a device scalar (grad_scale times the term's weight), so each seg CE runs its forward and
backward as one call (pcl_seg_ce_fwd_bwd); RMI, Lovasz and OHEM run their forward, then their backward.  bf16 / fp16
logits are copied into static fp32 buffers inside the graph and their gradients cast back, as the eager path does.

The object covers the with_embed=True phase only: during the warm-up epochs (with_embed=False) trainers keep calling
the eager criterion.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import _abi
from . import functional as _fn
from .graph_step import GraphedContrastStep, _canonical, _canonical_float, _cols_backward, _keep_cols
from .loss import ContrastAuxCELoss, ContrastCELoss


class _Term:
    """Static buffers and launch sequence of one seg term (loss.SegTerm) on the fp32 logits x."""

    def __init__(self, lib, term, x: torch.Tensor, target: torch.Tensor, grad_scale: float):
        self.lib, self.kind, self.head, self.coef = lib, term.kind, term.head, term.coef
        self.x, self.target = x, target
        dev = x.device
        B, K, h, w = x.shape
        H, W = target.shape[1], target.shape[2]
        self.dims = (B, K, h, w, H, W)
        mod = term.module
        self.weight = None
        if self.kind == "ce":
            self.weight, self.ignore = mod.weight, int(mod.ignore_index)
            self.one_call = H >= h and W >= w
            n = (lib.pcl_seg_ce_fwd_bwd_scratch_floats(B, K, H, W) if self.one_call else
                 lib.pcl_seg_ce_scratch_floats(B, H, W))
            self.scratch = torch.empty(n, dtype=torch.float32, device=dev)
        elif self.kind == "rmi":
            if K != mod.num_classes:
                raise _abi.PclError(f"seg has {K} channels, the RMI loss num_classes is {mod.num_classes}")
            self.params = (int(mod.rmi_radius), int(mod.rmi_pool_way), int(mod.rmi_pool_stride),
                           float(mod.weight_lambda), 1 if mod.lambda_way else 0, float(mod.loss_weight))
            self.scratch = _fn._byte_scratch(lib.pcl_rmi_scratch_bytes(*self.dims, *self.params[:3]),
                                             "pcl_rmi_scratch_bytes", dev)
        elif self.kind == "lovasz":
            self.ignore = int(mod.ignore_index)
            self.scratch = _fn._byte_scratch(lib.pcl_lovasz_scratch_bytes(*self.dims), "pcl_lovasz_scratch_bytes", dev)
        else:                                                       # ohem
            self.weight, self.ignore = mod.weight, int(mod.ignore_label)
            self.red, self.min_kept = _fn._ohem_args(x, target, mod.reduction, mod.min_kept)
            self.thresh = float(mod.thresh)
            self.scratch = _fn._byte_scratch(lib.pcl_ohem_ce_scratch_bytes(*self.dims), "pcl_ohem_ce_scratch_bytes", dev)
        if self.weight is not None:
            self.weight = self.weight.to(device=dev, dtype=torch.float32).contiguous().clone()
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        self.dseg = torch.zeros_like(x)
        self.gs = torch.empty(1, dtype=torch.float32, device=dev)
        self.set_grad_scale(grad_scale)

    def set_grad_scale(self, g: float) -> None:
        self.gs.fill_(float(g) * (1.0 if self.coef is None else float(self.coef)))

    def launch(self, stream: int) -> None:
        lib, x, t, sc = self.lib, self.x.data_ptr(), self.target.data_ptr(), self.scratch.data_ptr()
        loss, gs, dseg = self.loss.data_ptr(), self.gs.data_ptr(), self.dseg.data_ptr()
        if self.kind == "ce":
            a = (x, t, _abi.ptr(self.weight), *self.dims, self.ignore)
            if self.one_call:
                _abi.check(lib.pcl_seg_ce_fwd_bwd(*a, sc, gs, loss, dseg, stream), "pcl_seg_ce_fwd_bwd")
            else:
                _abi.check(lib.pcl_seg_ce_fwd(*a, sc, loss, stream), "pcl_seg_ce_fwd")
                _abi.check(lib.pcl_seg_ce_bwd(*a, sc, gs, dseg, stream), "pcl_seg_ce_bwd")
        elif self.kind == "rmi":
            _abi.check(lib.pcl_rmi_fwd(x, t, *self.dims, *self.params, sc, loss, stream), "pcl_rmi_fwd")
            _abi.check(lib.pcl_rmi_bwd(x, t, *self.dims, *self.params, sc, gs, dseg, stream), "pcl_rmi_bwd")
        elif self.kind == "lovasz":
            _abi.check(lib.pcl_lovasz_fwd(x, t, *self.dims, self.ignore, sc, loss, stream), "pcl_lovasz_fwd")
            _abi.check(lib.pcl_lovasz_bwd(x, t, *self.dims, self.ignore, sc, gs, dseg, stream), "pcl_lovasz_bwd")
        else:
            a = (x, t, _abi.ptr(self.weight), *self.dims, self.ignore)
            _abi.check(lib.pcl_ohem_ce_fwd(*a, self.thresh, self.min_kept, self.red, sc, loss, stream),
                       "pcl_ohem_ce_fwd")
            _abi.check(lib.pcl_ohem_ce_bwd(*a, sc, gs, dseg, stream), "pcl_ohem_ce_bwd")


class GraphedContrastCriterion:
    """loss and gradients of ``crit(preds, target, with_embed=True)`` for fixed tensors, as one CUDA-graph replay.

    >>> gc = GraphedContrastCriterion(crit, preds, target, grad_scale=1.0)
    >>> loss, grads = gc.replay()       # grads: {'seg', 'embed'[, 'seg_aux']}, static buffers, times grad_scale
    >>> gc = GraphedContrastCriterion(crit, preds, target, embed_grad="cols")
    >>> loss, grads = gc.replay()       # grads['embed'] = (cols, col_pix): the anchor columns (GraphedContrastStep)

    ``preds`` holds the tensors the graph reads in place on every replay (refill them, do not replace them): 'seg',
    'embed', and 'seg_aux' (ContrastAuxCELoss) or 'segment_queue' / 'pixel_queue' [/ 'bank_shadow']
    (MemContrastCELoss); ``target`` too.  ``enqueue`` (bank steps) is GraphedContrastStep's.  Only the with_embed=True
    phase is captured: during the warm-up epochs, call the eager criterion.  Raises PclError, before anything is
    captured or written, for a criterion whose seg loss runs partly in torch (contrast.fused_seg_ce off, a CE the kernels do not
    fuse, a custom seg_criterion), rng other than 'device', tensors that are not contiguous or of the wrong dtype, and a
    MemContrastCELoss without queues.  embed_grad="cols": the embedding's gradient as the contrast step's anchor
    columns (GraphedContrastStep(grad="cols")): no dense embedding gradient and no fill in the graph, and apply() hands
    the columns to a sparse_grad projection head; the seg heads' gradients stay dense."""

    def __init__(self, crit: ContrastCELoss, preds: Dict[str, torch.Tensor], target: torch.Tensor,
                 grad_scale: float = 1.0, enqueue: Optional[dict] = None, capture: bool = True,
                 embed_grad: str = "dense"):
        if not isinstance(crit, ContrastCELoss):
            raise _abi.PclError("crit must be a ContrastCELoss, ContrastAuxCELoss or MemContrastCELoss")
        cc = crit.contrast_criterion
        if cc.rng != "device" or cc.perm_fn is not None:
            raise _abi.PclError("a captured criterion draws its anchors on the device: contrast.rng must be 'device'")
        heads = ["seg"] + (["seg_aux"] if isinstance(crit, ContrastAuxCELoss) else [])
        for k in heads + ["embed"]:
            if k not in preds:
                raise _abi.PclError(f"preds[{k!r}] is required")
        _fn._require_cuda(preds["embed"], "embed")
        dev = preds["embed"].device
        embed = _canonical_float(preds["embed"].detach(), "embed", dev)
        xs = {k: _canonical_float(preds[k].detach(), k, dev) for k in heads}
        target = _canonical(target, torch.int64, "target", dev)
        queues = crit._queues(preds)
        if crit.with_memory and queues is None:
            raise _abi.PclError("MemContrastCELoss needs preds['segment_queue'] and preds['pixel_queue']")
        terms = crit.seg_terms(preds)
        if terms is None:
            raise _abi.PclError("the wrapper runs (part of) this seg criterion in torch (contrast.fused_seg_ce off, a CE "
                                "the kernels do not fuse, or a custom seg_criterion): it cannot be captured")
        lib = _abi.load()
        self.device, self.heads, self.target = dev, heads, target
        self.xs = xs
        self.loss_weight = crit.loss_weight
        # fp32 logits are read in place; half logits through a static fp32 copy made inside the graph (the eager path's
        # seg.to(float32))
        self.x32 = {k: x if x.dtype == torch.float32 else torch.empty(x.shape, dtype=torch.float32, device=dev)
                    for k, x in xs.items()}
        self.terms = [_Term(lib, t, self.x32[t.head], target, grad_scale) for t in terms]
        # static gradient outputs: a fp32 head with one term hands out that term's dseg
        self.grads, self._tmp = {}, {}
        for k, x in xs.items():
            mine = [t for t in self.terms if t.head == k]
            self.grads[k] = mine[0].dseg if (x.dtype == torch.float32 and len(mine) == 1) else torch.empty_like(x)
            if x.dtype != torch.float32 and len(mine) > 1:
                self._tmp[k] = torch.empty_like(x)
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        opts = cc.options()
        opts.num_classes = xs["seg"].shape[1]
        segq, pixq = queues if queues is not None else (None, None)
        self.step = GraphedContrastStep(embed, target, seg=xs["seg"], segment_queue=segq, pixel_queue=pixq,
                                        bank_shadow=preds.get("bank_shadow"), options=opts,
                                        grad_scale=float(grad_scale) * self.loss_weight, capture=False,
                                        enqueue=enqueue, prologue=self._seg_half, epilogue=self._total,
                                        grad=embed_grad)
        if capture:                            # the hooks read self.step: capture once it is set
            self.step._capture(2)

    # captured into the step's first graph
    def _seg_half(self, stream: int) -> None:
        for k, x in self.xs.items():
            if x.dtype != torch.float32:
                self.x32[k].copy_(x)
        for t in self.terms:
            t.launch(stream)
        for k, x in self.xs.items():           # several terms on one head: autograd's sum of their gradients, each
            d = [t.dseg for t in self.terms if t.head == k]     # cast to the head's dtype first
            if x.dtype == torch.float32:
                if len(d) > 1:
                    torch.add(d[0], d[1], out=self.grads[k])
            else:
                self.grads[k].copy_(d[0])
                if len(d) > 1:
                    self._tmp[k].copy_(d[1])
                    self.grads[k].add_(self._tmp[k])

    # captured into the step's last graph: the wrapper's  seg loss + loss_weight * contrast loss
    def _total(self, stream: int) -> None:
        seg = None
        for t in self.terms:
            v = t.loss if t.coef is None else t.coef * t.loss
            seg = v if seg is None else seg + v
        self.loss.copy_(seg + self.loss_weight * self.step.loss)

    def set_grad_scale(self, value: float) -> None:
        for t in self.terms:
            t.set_grad_scale(value)
        self.step.set_grad_scale(float(value) * self.loss_weight)

    def replay(self) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """One criterion step on the current stream: (loss, grads), static buffers overwritten by the next replay
        (grads['embed'] = (cols, col_pix) with embed_grad="cols")."""
        self.step.replay()
        return self.loss, dict(self.grads, embed=self.step.grad_out)

    def apply(self, preds: Dict[str, torch.Tensor]) -> torch.Tensor:
        """Autograd hand-off: replays the graph and returns the loss connected to preds' heads and embedding (the
        tensors the graph was captured on); its backward hands them the replay's gradients.  Valid when backward starts
        from gradient 1 (fold weights into grad_scale), as GraphedContrastStep.apply.  embed_grad="cols": the embedding
        receives its gradient as GraphedContrastStep.apply() gives it in column mode."""
        ins = [preds[k] for k in self.heads] + [preds["embed"]]
        for k, t in zip(self.heads + ["embed"], ins):
            mine = self.step.embed if k == "embed" else self.xs[k]
            if t.data_ptr() != mine.data_ptr():
                raise _abi.PclError(f"apply() must receive the tensors the criterion was captured on ({k})")
        return _GraphedCriterionFn.apply(self, *ins)


class _GraphedCriterionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gc: GraphedContrastCriterion, *ins):
        loss, _ = gc.replay()
        ctx.gc = gc
        if gc.step.cols is not None:
            _keep_cols(ctx, gc.step, ins[-1])
        return loss.view(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        torch._assert_async((grad_out == 1).all(),
                            "GraphedContrastCriterion.apply(): upstream gradient != 1; fold the factor into grad_scale")
        gc = ctx.gc
        step = gc.step
        g_embed = step.grad if step.cols is None else _cols_backward(ctx, step.embed.shape, step.embed.dtype)
        return (None,) + tuple(gc.grads[k] for k in gc.heads) + (g_embed,)
