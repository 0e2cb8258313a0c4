"""Public functional entry point of the hot path.

``bags_head_loss`` = fc_cls projection + Balanced-Group-Softmax loss with a fused
backward, i.e. reference ``head.fc_cls(x)`` followed by ``head.loss(cls_score, None,
labels, ...)`` (convfc_bbox_head.py:166 + gs_bbox_head_with0.py:147-171), as one
autograd node.  ``GSBBoxHeadWith0`` (head.py) is the module-level drop-in built on it.
"""
from __future__ import annotations

import itertools
from typing import Optional, Union

import torch

from . import ops
from .tables import GroupTables

_seed_counter = itertools.count(1)


def bags_head_loss(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], labels: torch.Tensor,
                   tables: Union[GroupTables, ops.DeviceTables], others_sample_ratio: float = 8.0,
                   compute_dtype: torch.dtype = torch.bfloat16, wmask: Optional[torch.Tensor] = None,
                   avg: Optional[torch.Tensor] = None, seed: Optional[int] = None,
                   return_logits: bool = False, grad_bucket=None):
    """losses[G] (fp32, one per bin, already divided by the per-bin avg_factor).

    x [N,K] and weight [C,K] may be fp32 or bf16; ``compute_dtype`` selects bf16 or TF32 tensor-core
    products.  Without ``wmask`` the "others" rows are sampled on the device (``seed`` fixes the draw);
    with ``wmask`` [G,N] uint8 (e.g. recorded from the reference's numpy sampler) it is used as is.
    ``grad_bucket`` (data-parallel training; ``dist.PeerGradBucket`` / ``dist.NcclGradBucket`` over [(C,K), (C,)]): the
    backward writes dW / db into the bucket, exchanges them over NVLink as soon as they are complete and computes dX
    meanwhile; ``weight.grad`` / ``bias.grad`` receive the mean over ranks.
    """
    dt = tables if isinstance(tables, ops.DeviceTables) else ops.DeviceTables.from_tables(tables, x.device)
    if wmask is None:
        if seed is None:
            seed = (torch.initial_seed() * 0x9E3779B97F4A7C15 + next(_seed_counter)) & 0xFFFFFFFFFFFFFFFF
        wmask, avg = ops.sample_others(labels, dt, others_sample_ratio, seed)
    elif avg is None:
        avg = ops.mask_avg(wmask)
    logits = None
    if return_logits:
        logits = torch.empty((x.shape[0], weight.shape[0]), dtype=torch.float32, device=x.device)
    loss = ops.GroupSoftmaxFunction.apply(x, weight, bias, labels, dt, wmask, avg, compute_dtype, logits, grad_bucket)
    return (loss, logits) if return_logits else loss


class GraphedHeadStep(object):
    """One training step of the hot path, captured once as a CUDA graph and replayed.

        sample "others" masks -> fc_cls + BAGS loss (GroupSoftmaxFunction) -> sum_g c_g * loss_g -> backward
        [-> gradient exchange]

    i.e. what ``head.fc_cls(x)``, ``head.loss(...)``, ``parse_losses`` and ``loss.backward()`` do per iteration in the
    reference (convfc_bbox_head.py:166, gs_bbox_head_with0.py:147-171, apis/train.py:17-34, dist_utils.py:53), with
    the same autograd Function as the eager API underneath -- the standard ``torch.cuda.graph`` whole-step capture.
    The per-step host cost drops from a few hundred microseconds of Python / autograd / allocator work to one graph
    launch, which is what a 43 us GPU step needs.

    Static tensors (filled / read by the caller between replays):
        ``x`` [N,K], ``labels`` [N] int64        inputs (e.g. the destination of the H2D copies)
        ``losses`` [G] fp32                      per-bin losses of the last replay
        ``grad_weight``, ``grad_bias``, ``grad_x``   gradients of the last replay (also ``weight.grad`` / ``bias.grad``)
    The sampler's seed advances on the device after every replay, so replays draw different "others" subsets.
    """

    def __init__(self, weight: torch.nn.Parameter, bias: Optional[torch.nn.Parameter],
                 tables: Union[GroupTables, ops.DeviceTables], n_rois: int, others_sample_ratio: float = 8.0,
                 compute_dtype: torch.dtype = torch.bfloat16, x_dtype: Optional[torch.dtype] = None,
                 loss_weights: Optional[torch.Tensor] = None, need_dx: bool = True, seed: Optional[int] = None,
                 exchange=None, stream: Optional[torch.cuda.Stream] = None, warmup: int = 2, grad_bucket=None):
        dev = weight.device
        if dev.type != 'cuda':
            raise ops.nat.BagsNativeError('GraphedHeadStep runs on an H100 GPU only (weight is on %s)' % dev)
        self.weight, self.bias = weight, bias
        self.dt = tables if isinstance(tables, ops.DeviceTables) else ops.DeviceTables.from_tables(tables, dev)
        self.ratio = float(others_sample_ratio)
        self.compute_dtype = compute_dtype
        self.loss_weights = None if loss_weights is None else loss_weights.to(dev, torch.float32)
        self.exchange = exchange
        # data-parallel: dW / db are written into this bucket (dist.PeerGradBucket / NcclGradBucket), exchanged as soon as
        # they are complete and while dX is computed; weight.grad / bias.grad become the bucket's views (mean over ranks)
        self.grad_bucket = grad_bucket
        self.seed = int(seed if seed is not None else
                        (torch.initial_seed() * 0x9E3779B97F4A7C15 + next(_seed_counter))) & 0xFFFFFFFFFFFFFFFF
        K = weight.shape[1]
        self.x = torch.zeros((n_rois, K), dtype=(x_dtype or weight.dtype), device=dev, requires_grad=need_dx)
        self.labels = torch.zeros((n_rois,), dtype=torch.int64, device=dev)
        self.seed_step = torch.zeros((1,), dtype=torch.int64, device=dev)
        self.stream = stream if stream is not None else torch.cuda.Stream(device=dev)
        self.stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(self.stream):
            for _ in range(max(int(warmup), 1)):       # also lets the library set up its per-stream state
                self._clear_grads()
                self._body()
            self.stream.synchronize()
            self._clear_grads()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.losses = self._body()
            self.seed_step.zero_()
        self.grad_weight = weight.grad
        self.grad_bias = None if bias is None else bias.grad
        self.grad_x = self.x.grad
        torch.cuda.current_stream(dev).wait_stream(self.stream)

    def _clear_grads(self):
        self.weight.grad = None
        if self.bias is not None:
            self.bias.grad = None
        self.x.grad = None

    def _body(self):
        wmask, avg = ops.sample_others(self.labels, self.dt, self.ratio, self.seed, seed_step=self.seed_step)
        losses = ops.GroupSoftmaxFunction.apply(self.x, self.weight, self.bias, self.labels, self.dt, wmask, avg,
                                                self.compute_dtype, None, self.grad_bucket)
        total = losses.sum() if self.loss_weights is None else (losses * self.loss_weights).sum()
        total.backward()
        if self.exchange is not None:
            self.exchange()
        # last node of the graph: never the stream predecessor of the sampler, which reads it before its PDL wait
        self.seed_step.add_(1)
        return losses.detach()

    def replay(self) -> torch.Tensor:
        """Launch the captured step on the current stream; returns the static ``losses`` tensor."""
        self.graph.replay()
        return self.losses

    def __call__(self, x: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None) -> torch.Tensor:
        if x is not None:
            with torch.no_grad():
                self.x.copy_(x, non_blocking=True)
        if labels is not None:
            self.labels.copy_(labels, non_blocking=True)
        return self.replay()


class _GraphedPair(object):
    """Static buffers + two CUDA graphs (forward: sampler + fused forward; backward: preparation + merged backward) for ONE RoI count."""

    def __init__(self, n: int, k: int, c: int, dt: ops.DeviceTables, ratio: float, seed: int, op_dtype: torch.dtype,
                 has_bias: bool, need_dx: bool, device):
        self.n = n
        self.x = torch.zeros((n, k), dtype=op_dtype, device=device)
        self.labels = torch.zeros((n,), dtype=torch.int64, device=device)
        self.w = torch.zeros((c, k), dtype=op_dtype, device=device)
        self.bias = torch.zeros((c,), dtype=torch.float32, device=device) if has_bias else None
        self.gout = torch.ones((dt.G,), dtype=torch.float32, device=device)
        self.seed_step = torch.zeros((1,), dtype=torch.int64, device=device)
        self.dW = torch.zeros((c, k), dtype=torch.float32, device=device)
        self.db = torch.zeros((c,), dtype=torch.float32, device=device) if has_bias else None
        self.dX = torch.zeros((n, k), dtype=op_dtype, device=device) if need_dx else None
        self.wscratch = ops.bwd_scratch(self.w)
        self.w_version = None
        self.b_version = None
        self.stream = torch.cuda.Stream(device=device)
        self.stream.wait_stream(torch.cuda.current_stream(device))

        def fwd():
            wmask, avg = ops.sample_others(self.labels, dt, ratio, seed, seed_step=self.seed_step)
            loss, _, _, dz, _ = ops.fused_fwd(self.x, self.w, self.bias, self.labels, dt, wmask, avg, clear=self.dW)
            return loss, dz

        def bwd(dz):
            ops.fused_bwd(dz, self.x, self.w, self.gout, dt, None, need_db=has_bias, need_dx=need_dx, dW=self.dW,
                          dX=self.dX, wscratch=self.wscratch, db=self.db, dw_prezeroed=True)

        with torch.cuda.stream(self.stream):
            for _ in range(2):
                loss, dz = fwd()
                bwd(dz)
            self.stream.synchronize()
            self.g_fwd, self.g_bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_fwd, stream=self.stream):
                self.loss, self.dz = fwd()
                self.seed_step.add_(1)
            with torch.cuda.graph(self.g_bwd, stream=self.stream, pool=self.g_fwd.pool()):
                bwd(self.dz)
            self.seed_step.zero_()
        torch.cuda.current_stream(device).wait_stream(self.stream)


class _GraphCachedFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weight, bias, labels, pair: _GraphedPair):
        with torch.no_grad():
            pair.x.copy_(x)
            pair.labels.copy_(labels)
            if pair.w_version != (id(weight), weight._version):     # the operand copy follows optimizer updates
                pair.w.copy_(weight)
                pair.w_version = (id(weight), weight._version)
            if bias is not None and pair.b_version != (id(bias), bias._version):
                pair.bias.copy_(bias)
                pair.b_version = (id(bias), bias._version)
        pair.g_fwd.replay()
        ctx.pair = pair
        ctx.dtypes = (x.dtype, weight.dtype, None if bias is None else bias.dtype)
        return pair.loss.clone()

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        pair = ctx.pair
        pair.gout.copy_(grad_loss)
        pair.g_bwd.replay()
        xd, wd, bd = ctx.dtypes
        # gradients leave as fresh tensors (a cast already is one): the static buffers are rewritten by the next replay, and
        # fresh tensors can be adopted by AccumulateGrad without another copy (measured: 165 vs 195 us per call when the
        # static buffers themselves were returned and autograd made its own copies)
        dX = None
        if pair.dX is not None and ctx.needs_input_grad[0]:
            dX = pair.dX.clone() if pair.dX.dtype == xd else pair.dX.to(xd)
        dW = None
        if ctx.needs_input_grad[1]:
            dW = pair.dW.clone() if pair.dW.dtype == wd else pair.dW.to(wd)
        db = None
        if pair.db is not None and ctx.needs_input_grad[2]:
            db = pair.db.clone() if pair.db.dtype == bd else pair.db.to(bd)
        return dX, dW, db, None, None


class GraphCachedHeadLoss(object):
    """``bags_head_loss`` for callers whose RoI count is data-dependent (every real detector: up to 512 sampled RoIs per
    image, in practice almost always exactly that -- ``RandomSampler`` fills up with negatives,
    mmdet/core/bbox/samplers/base_sampler.py:30-78) but who still want graph-replay host costs inside an ordinary
    autograd graph (x comes from the trunk, dX flows back into it).

    Per RoI count N it keeps static buffers and two CUDA graphs (sampler + fused forward; preparation + merged backward); a call with a
    cached N costs a few small copies and two graph launches instead of ~220 us of Python / allocator / launch work.  A
    new N runs the eager path the first ``capture_after`` times it is seen and is captured after that; at most
    ``max_graphs`` counts stay cached (least recently used first out).  The "others" sampler's seed advances on the device
    with every replay."""

    def __init__(self, tables: Union[GroupTables, ops.DeviceTables], others_sample_ratio: float = 8.0,
                 compute_dtype: torch.dtype = torch.bfloat16, seed: Optional[int] = None, max_graphs: int = 4,
                 capture_after: int = 2, need_dx: bool = True):
        self.tables = tables
        self.ratio = float(others_sample_ratio)
        self.compute_dtype = compute_dtype
        self.seed = int(seed if seed is not None else
                        (torch.initial_seed() * 0x9E3779B97F4A7C15 + next(_seed_counter))) & 0xFFFFFFFFFFFFFFFF
        self.max_graphs, self.capture_after, self.need_dx = int(max_graphs), int(capture_after), bool(need_dx)
        self._pairs = {}      # N -> _GraphedPair, insertion order = recency
        self._seen = {}
        self._dt = None
        self.stats = {'replays': 0, 'eager': 0, 'captures': 0}

    def __call__(self, x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], labels: torch.Tensor):
        dev = x.device
        if self._dt is None:
            self._dt = self.tables if isinstance(self.tables, ops.DeviceTables) else \
                ops.DeviceTables.from_tables(self.tables, dev)
        n = int(x.shape[0])
        pair = self._pairs.pop(n, None)
        if pair is None:
            seen = self._seen.get(n, 0) + 1
            self._seen[n] = seen
            if n == 0 or seen <= self.capture_after or torch.cuda.is_current_stream_capturing():
                self.stats['eager'] += 1
                return bags_head_loss(x, weight, bias, labels, self._dt, self.ratio, compute_dtype=self.compute_dtype)
            op_dtype = torch.bfloat16 if self.compute_dtype == torch.bfloat16 else torch.float32
            pair = _GraphedPair(n, int(x.shape[1]), int(weight.shape[0]), self._dt, self.ratio,
                                (self.seed + 0x9E3779B97F4A7C15 * n) & 0xFFFFFFFFFFFFFFFF, op_dtype, bias is not None,
                                self.need_dx, dev)
            self.stats['captures'] += 1
            while len(self._pairs) >= self.max_graphs:
                self._pairs.pop(next(iter(self._pairs)))
        self._pairs[n] = pair                                   # most recently used last
        self.stats['replays'] += 1
        return _GraphCachedFunction.apply(x, weight, bias, labels, pair)
