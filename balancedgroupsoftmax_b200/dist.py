"""Data-parallel gradient exchange for the head over NVLink: one peer-memory kernel (PeerGradBucket), or NCCL.

Restates mmdet/core/utils/dist_utils.py:9-58 (``_allreduce_coalesced`` /
``allreduce_grads``): flatten all trainable grads by dtype into one bucket,
all-reduce, divide by world size, copy back.  Differences that keep the result
identical but remove passes: NCCL's native AVG op replaces the separate ``div_``,
and callers that allocate their grads as views of one flat bucket
(``flat_grad_bucket``) skip the flatten / copy-back entirely.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import OrderedDict
from typing import Iterable, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch._utils import _flatten_dense_tensors, _unflatten_dense_tensors


def _avg_op():
    return dist.ReduceOp.AVG if dist.get_backend() == 'nccl' else None


def allreduce_flat_(flat: torch.Tensor, async_op: bool = False):
    """In-place mean over ranks of one flat bucket."""
    op = _avg_op()
    if op is not None:
        return dist.all_reduce(flat, op=op, async_op=async_op)
    work = dist.all_reduce(flat, async_op=async_op)   # gloo has no AVG
    if async_op:
        work.wait()
    flat.div_(dist.get_world_size())
    return None


_peer_buckets = {}   # (device index, numel) -> PeerGradBucket | None (None: tried, unavailable)


def _peer_bucket_for(numel: int, device) -> Optional['PeerGradBucket']:
    """Cached peer-memory staging bucket for fp32 gradient sets of `numel` elements (None -> use NCCL)."""
    if os.environ.get('BAGS_ALLREDUCE', 'peer') == 'nccl' or not PeerGradBucket.available():
        return None
    key = (torch.device(device).index, int(numel))
    if key not in _peer_buckets:
        try:
            b = PeerGradBucket([(int(numel),)], device)
            _peer_buckets[key] = b if b.self_test() else None
        except Exception:
            _peer_buckets[key] = None
    return _peer_buckets[key]


def allreduce_grads(params: Iterable[torch.nn.Parameter], coalesce: bool = True) -> None:
    """Mean of the gradients over ranks (mmdet/core/utils/dist_utils.py:31-41).  fp32 CUDA gradients travel through
    the NVLink peer-memory kernel when it is available (flatten into the symmetric bucket -> bags_grad_allreduce ->
    copy back: the reference's flatten / all_reduce / div / unflatten with the collective replaced); anything else
    takes the reference's NCCL / gloo route."""
    grads = [p.grad.data for p in params if p.requires_grad and p.grad is not None]
    if not grads:
        return
    if coalesce:
        f32 = [g for g in grads if g.dtype == torch.float32 and g.is_cuda]
        if f32:
            bucket = _peer_bucket_for(sum(g.numel() for g in f32), f32[0].device)
            if bucket is not None:
                off = 0
                for g in f32:
                    bucket.flat[off:off + g.numel()].view_as(g).copy_(g)
                    off += g.numel()
                bucket.allreduce_()
                off = 0
                for g in f32:
                    g.copy_(bucket.flat[off:off + g.numel()].view_as(g))
                    off += g.numel()
                grads = [g for g in grads if not (g.dtype == torch.float32 and g.is_cuda)]
                if not grads:
                    return
    if not coalesce:
        for g in grads:
            allreduce_flat_(g)
        return
    buckets = OrderedDict()
    for g in grads:
        buckets.setdefault(g.type(), []).append(g)
    for bucket in buckets.values():
        if len(bucket) == 1 and bucket[0].is_contiguous():
            allreduce_flat_(bucket[0].view(-1))
            continue
        flat = _flatten_dense_tensors(bucket)
        allreduce_flat_(flat)
        for g, synced in zip(bucket, _unflatten_dense_tensors(flat, bucket)):
            g.copy_(synced)


def flat_grad_bucket(shapes: List[Tuple[int, ...]], device, dtype=torch.float32):
    """One flat buffer + per-tensor views (write grads straight into the bucket)."""
    sizes = [int(torch.Size(s).numel()) for s in shapes]
    flat = torch.zeros(sum(sizes), device=device, dtype=dtype)
    views, off = [], 0
    for s, n in zip(shapes, sizes):
        views.append(flat[off:off + n].view(*s))
        off += n
    return flat, views


# ---------------------------------------------------------------------------------------------------
# NVLink peer-memory exchange (libbags_b200.so: bags_grad_allreduce) -- the NVSwitch path
# ---------------------------------------------------------------------------------------------------
class PeerGradBucket(object):
    """Flat fp32 gradient bucket in symmetric (peer-mapped) memory + its one-kernel all-reduce.

    The reference flattens the grads, calls ``dist.all_reduce`` (NCCL), divides by the world size and copies back
    (mmdet/core/utils/dist_utils.py:9-41).  Here the backward kernels write dW / db straight into ``views`` of a bucket
    that every rank has mapped through NVLink, and ``allreduce_()`` launches ``bags_grad_allreduce``: cross-rank
    barrier, two-shot reduction over the NVSwitch multicast mapping (``multimem.ld_reduce`` / ``multimem.st``) or,
    without multicast support, plain peer loads / stores, cross-rank barrier -- one stream-ordered kernel that is
    CUDA-graph capturable and needs no host synchronisation.

    Allocation / rendezvous go through ``torch.distributed._symmetric_memory`` (plumbing only).  ``available()``
    tells whether that works in this process group; callers fall back to ``allreduce_flat_`` (NCCL) otherwise.
    """

    def __init__(self, shapes: List[Tuple[int, ...]], device, group=None, mean: bool = True, max_blocks: int = 0):
        import torch.distributed._symmetric_memory as symm
        from . import _native
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.mean = mean
        self.max_blocks = int(max_blocks)
        sizes = [int(torch.Size(s).numel()) for s in shapes]
        self.numel = sum(sizes)
        self.count = (self.numel + 3) // 4 * 4                       # the kernel moves 16-byte vectors
        self.flag_off = (self.count * 4 + 255) // 256 * 256
        flag_bytes = int(_native.lib().bags_grad_allreduce_flag_bytes(self.world))
        total_floats = (self.flag_off + flag_bytes) // 4
        self.storage = symm.empty(total_floats, dtype=torch.float32, device=device)
        self.storage.zero_()                                         # data + flag words (flags must start at zero)
        torch.cuda.synchronize(device)
        self.handle = symm.rendezvous(self.storage, self.group)      # exchanges the handles, maps the peers
        dist.barrier(self.group)                                     # every rank's flags are zero before any kernel runs
        off = int(getattr(self.handle, 'offset', 0) or 0)
        self.peer_ptrs = [int(p) + off for p in self.handle.buffer_ptrs]
        if self.peer_ptrs[self.rank] != self.storage.data_ptr():
            raise RuntimeError('symmetric memory: local mapping %#x != tensor %#x' % (self.peer_ptrs[self.rank],
                                                                                      self.storage.data_ptr()))
        mc = int(getattr(self.handle, 'multicast_ptr', 0) or 0)
        self.mc_ptr = (mc + off) if mc else 0
        self._peer_arr = (C.c_void_p * self.world)(*self.peer_ptrs)
        self.flat = self.storage[:self.numel]
        self.views, o = [], 0
        for s, n in zip(shapes, sizes):
            self.views.append(self.flat[o:o + n].view(*s))
            o += n

    why_not = ''   # set by available(): the reason the peer path cannot be used

    @staticmethod
    def available() -> bool:
        """True when the process group runs NCCL on CUDA with more than one rank and symmetric memory is importable."""
        cls = PeerGradBucket
        try:
            if not (dist.is_available() and dist.is_initialized()):
                cls.why_not = 'torch.distributed is not initialised'
                return False
            if dist.get_world_size() < 2:
                cls.why_not = 'world size 1'
                return False
            if not torch.cuda.is_available():
                cls.why_not = 'no CUDA device'
                return False
            backend = str(dist.get_backend()).lower()
            if 'nccl' not in backend:
                cls.why_not = 'backend %r is not NCCL' % backend
                return False
            import torch.distributed._symmetric_memory as _symm  # noqa: F401
            cls.why_not = ''
            return True
        except Exception as ex:
            cls.why_not = repr(ex)
            return False

    def status(self) -> int:
        """0, or 1 after an exchange in which some rank never arrived (soft mode: the kernel gave up and the bucket is
        unusable; normal mode: the kernel trapped and every later CUDA call of this process fails)."""
        from . import _native
        word = (self.flag_off + int(_native.lib().bags_grad_allreduce_status_offset(self.world))) // 4
        return int(self.storage[word:word + 1].view(torch.int32).item())

    def self_test(self) -> bool:
        """One exchange of a known pattern, verified on every rank (collective: all ranks must call it)."""
        dev = self.storage.device
        # a rank-, position- and sign-dependent pattern (a constant fill cannot see a chunk-boundary or ordering bug);
        # small integers, so the sum over ranks is exact in fp32 and the expected value is known in closed form
        idx = torch.arange(self.numel, device=dev, dtype=torch.float32)
        pat = torch.remainder(idx, 61.0) - 30.0
        self.flat.copy_(pat * float(self.rank + 1) + float(self.rank))
        self.allreduce_(soft=True)
        torch.cuda.synchronize(dev)
        s1 = self.world * (self.world + 1) / 2.0
        s0 = self.world * (self.world - 1) / 2.0
        expect = pat * s1 + s0
        if self.mean:
            expect = expect / self.world
        ok = self.status() == 0 and bool(((self.flat - expect).abs() <= 1e-5 * expect.abs().clamp_min(1.0)).all().item())
        verdict = torch.tensor([1 if ok else 0], device=dev)
        dist.all_reduce(verdict, op=dist.ReduceOp.MIN, group=self.group)
        self.flat.zero_()
        torch.cuda.synchronize(dev)
        return bool(verdict.item())

    @property
    def transport(self) -> str:
        return 'nvls-multimem' if (self.mc_ptr and not os.environ.get('BAGS_AR_NO_MULTIMEM')) else 'peer-ldst'

    def allreduce_(self, stream: Optional[int] = None, soft: bool = False) -> None:
        """In place, on the current stream (or the given cudaStream_t): every rank ends with the mean (or sum).
        A rank that never arrives makes the kernel trap after BAGS_AR_TIMEOUT_MS (default 30 s): the process fails
        loudly instead of training on un-averaged gradients.  ``soft=True`` (the self test): only the status word is
        set, so that the caller can fall back to NCCL."""
        from . import _native
        if stream is None:
            stream = torch.cuda.current_stream(self.storage.device).cuda_stream
        scale = (1.0 / self.world) if self.mean else 1.0
        rc = _native.lib().bags_grad_allreduce(self._peer_arr, self.mc_ptr or None, self.flag_off, self.count,
                                               self.rank, self.world, scale, -1 if soft else self.max_blocks, stream)
        _native.check(rc, 'bags_grad_allreduce')


def _exchange_overlapped(self, side_stream=None):
    """Start this bucket's exchange on a side stream, ordered after everything launched so far on the current stream
    (i.e. after the kernel that completed the gradients), and return a ``join()`` that makes the current stream wait
    for it.  What is launched on the current stream between the two -- the dX contraction -- overlaps the exchange."""
    dev = self.flat.device
    cur = torch.cuda.current_stream(dev)
    if isinstance(self, PeerGradBucket) and self.max_blocks == 0:
        # An exchange that shares the GPU with the dX GEMM wants a SMALL grid: its blocks then live on the SMs the GEMM
        # leaves free instead of competing with GEMM CTAs for issue slots, but large enough to keep
        # this rank's slice in flight: one block per 2048 16-byte vectors of the slice, between 16 and 48.
        per_rank = (self.count // 4 + self.world - 1) // self.world
        self.max_blocks = max(16, min(48, (per_rank + 2047) // 2048))
    if side_stream is None:
        side_stream = getattr(self, '_side_stream', None)
        if side_stream is None:
            side_stream = self._side_stream = torch.cuda.Stream(device=dev)
    ev = torch.cuda.Event()
    ev.record(cur)
    side_stream.wait_event(ev)
    with torch.cuda.stream(side_stream):
        self.allreduce_()

    def join():
        cur.wait_stream(side_stream)
    return join


PeerGradBucket.exchange_overlapped = _exchange_overlapped


class NcclGradBucket(object):
    """The same interface over a plain flat bucket exchanged with NCCL / gloo (the reference's route), for process
    groups where the peer-memory path is unavailable."""

    def __init__(self, shapes: List[Tuple[int, ...]], device):
        self.flat, self.views = flat_grad_bucket(shapes, device)

    def allreduce_(self):
        allreduce_flat_(self.flat)

    def status(self) -> int:
        return 0

    exchange_overlapped = _exchange_overlapped


def make_grad_bucket(shapes: List[Tuple[int, ...]], device, prefer_peer: bool = True, max_blocks: int = 0):
    """(bucket_or_None, flat, views, allreduce_fn): the peer-memory bucket when it can be set up, else a plain bucket
    exchanged with NCCL (same results; the reference's path)."""
    if prefer_peer and PeerGradBucket.available() and os.environ.get('BAGS_ALLREDUCE', 'peer') != 'nccl':
        try:
            b = PeerGradBucket(shapes, device, max_blocks=max_blocks)
            if not b.mc_ptr and b.world > 4 and os.environ.get('BAGS_ALLREDUCE') != 'peer':
                # without an NVSwitch multicast object the kernel falls back to plain peer loads / stores, which read every
                # element from all ranks: fine at 2 ranks, slower than NCCL at 8
                import warnings
                warnings.warn('no multicast (NVLS) mapping at %d ranks: using NCCL all-reduce for the gradient bucket' % b.world)
            elif b.self_test():
                return b, b.flat, b.views, b.allreduce_
            else:
                import warnings
                warnings.warn('peer-memory gradient exchange failed its self test; using NCCL all-reduce')
        except Exception as ex:  # symmetric memory not usable on this system
            import warnings
            warnings.warn('peer-memory gradient bucket unavailable (%r); using NCCL all-reduce' % (ex,))
    elif prefer_peer and dist.is_initialized() and dist.get_rank() == 0 and PeerGradBucket.why_not:
        import warnings
        warnings.warn('peer-memory gradient bucket not used: %s' % PeerGradBucket.why_not)
    flat, views = flat_grad_bucket(shapes, device)
    return None, flat, views, (lambda: allreduce_flat_(flat))
