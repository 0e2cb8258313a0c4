"""The data-parallel gradient exchange: its one barrier protocol, and GroupSoftmaxFunction's backward with a bucket.

CPU: bags_api.cu compiled to PTX for sm_90a holds exactly two exchange kernels (multimem and peer transport), both on
the epoch protocol: relaxed store at the first barrier, release store at the second, relaxed polling with one acquire
load, and no compare-and-swap.

GPU (one H100):
  * bags_grad_allreduce at world = 1 on the peer path: the data becomes scale * data bit for bit, the status word stays
    0, and every launched block's epoch advances by two per call (one per barrier), on the default and a limited grid
    and under a CUDA-graph replay.  The soft mode runs first, so that a protocol mistake sets the status word instead
    of trapping.
  * GroupSoftmaxFunction with a stub bucket: dW + db go into the bucket views, the exchange starts once they are final,
    dX runs between the exchange and its join, and the gradients agree with the same call without a bucket.
"""
import ctypes as C
import inspect
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200 import _native as nat
from balancedgroupsoftmax_b200 import build as B
from balancedgroupsoftmax_b200.tables import synthetic_tables


def _ptx_entries(ptx):
    """{entry name: body} of every kernel in a PTX module."""
    heads = list(re.finditer(r'\.entry\s+(\w+)\s*\(', ptx))
    return {m.group(1): ptx[m.end():heads[i + 1].start() if i + 1 < len(heads) else len(ptx)]
            for i, m in enumerate(heads)}


def test_exchange_kernels_use_the_epoch_protocol_only():
    try:
        nvcc = B._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, 'bags_api.ptx')
        cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-ptx', '-o', out] + B.SOURCES
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert res.returncode == 0, res.stdout
        ptx = open(out).read()
    kernels = {name: body for name, body in _ptx_entries(ptx).items() if 'bags_grad_allreduce_kernel' in name}
    assert len(kernels) == 2, sorted(kernels)
    for name, body in kernels.items():
        assert not re.search(r'\batom\.[\w.]*\bcas\b', body), name
        for op in ('st.relaxed.sys.global.u32', 'st.release.sys.global.u32', 'ld.relaxed.sys.global.u32',
                   'ld.acquire.sys.global.u32'):
            assert op in body, (name, op)


@pytest.mark.gpu
def test_exchange_at_world_one():
    lib = nat.lib()
    status_off = lib.bags_grad_allreduce_status_offset(1)
    maxb = status_off // 8                    # [maxb][world = 1] slots and [maxb] epochs precede the status word
    vecs = maxb * 1024 + 3                    # more blocks than the grid limit allows at 256 threads x 4 vectors
    count = 4 * vecs
    flag_off = (count * 4 + 255) // 256 * 256
    buf = torch.zeros((flag_off + lib.bags_grad_allreduce_flag_bytes(1)) // 4, dtype=torch.float32, device='cuda')
    g = torch.Generator().manual_seed(7)
    buf[:count] = torch.randint(-512, 513, (count,), generator=g).float().cuda()   # exact under any power-of-2 scale
    buf[count:flag_off // 4] = 12345.0        # padding between the data and the flags: never touched
    flags = buf[flag_off // 4:].view(torch.int32)
    peers = (C.c_void_p * 1)(buf.data_ptr())
    expect = buf[:count].clone()
    expect_epoch = np.zeros(maxb, dtype=np.int64)

    def call(max_blocks, scale, stream):
        nat.check(lib.bags_grad_allreduce(peers, None, flag_off, count, 0, 1, scale, max_blocks, stream),
                  'bags_grad_allreduce')

    def check(blocks, scale, what):
        nonlocal expect
        torch.cuda.synchronize()
        expect = expect * scale
        expect_epoch[:blocks] += 2
        assert flags[status_off // 4].item() == 0, what
        assert torch.equal(buf[:count].view(torch.int32), expect.view(torch.int32)), what
        assert (buf[count:flag_off // 4] == 12345.0).all().item(), what
        epochs = flags[maxb:2 * maxb].cpu().numpy()
        slots = flags[:maxb].cpu().numpy()    # slot[b][0]: the last epoch block b published to itself
        assert (epochs == expect_epoch).all(), (what, epochs)
        assert (slots == expect_epoch).all(), (what, slots)

    stream = torch.cuda.current_stream().cuda_stream
    call(-1, 0.5, stream)                     # soft mode, default grid: a missed barrier only sets the status word
    check(maxb, 0.5, 'soft mode')
    for max_blocks, blocks in ((0, maxb), (16, 16)):
        for scale in (0.5, 2.0):
            call(max_blocks, scale, stream)
            check(blocks, scale, 'max_blocks=%d scale=%g' % (max_blocks, scale))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        call(16, 0.5, side.cuda_stream)
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    check(16, 0.5, 'graph replay')


class _StubBucket(object):
    """What GroupSoftmaxFunction uses of a gradient bucket: ``views`` of one flat fp32 tensor and
    ``exchange_overlapped()``, which here records when it was called and what the views held at that point of the
    stream."""

    def __init__(self, C, K, log):
        self.flat = torch.zeros(C * K + C, dtype=torch.float32, device='cuda')
        self.views = [self.flat[:C * K].view(C, K), self.flat[C * K:]]
        self.log = log
        self.at_exchange = None

    def exchange_overlapped(self):
        self.log.append('exchange')
        self.at_exchange = [v.clone() for v in self.views]

        def join():
            self.log.append('join')
        return join


TOL = {torch.float32: 1e-3, torch.bfloat16: 5e-3}   # gradients, as in test_gpu_parity.py


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.gpu
@pytest.mark.parametrize('x_grad', [True, False], ids=['dx', 'no_dx'])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_group_softmax_backward_with_bucket(monkeypatch, mode, x_grad):
    from balancedgroupsoftmax_b200 import ops
    t = synthetic_tables(1231, seed=0)
    dt = ops.DeviceTables.from_tables(t, 'cuda')
    C, K, N = t.num_logits, 256, 512
    g = torch.Generator().manual_seed(5)
    x0 = torch.relu(torch.randn(N, K, generator=g)).cuda().to(mode)
    W0 = (torch.randn(C, K, generator=g) * 0.05).cuda()
    b0 = (torch.randn(C, generator=g) * 0.1).cuda()
    labels = torch.zeros(N, dtype=torch.int64)
    labels[:N // 4] = torch.randint(1, t.num_classes, (N // 4,), generator=g)
    labels = labels.cuda()
    wmask, avg = ops.sample_others(labels, dt, 8.0, 1234)
    gout = torch.linspace(0.5, 2.0, t.num_bins, device='cuda')

    log = []
    fused_bwd = ops.fused_bwd
    sig = inspect.signature(fused_bwd)

    def spy(*args, **kwargs):
        a = sig.bind(*args, **kwargs)
        a.apply_defaults()
        log.append(('bwd', a.arguments['need_dw'], a.arguments['need_db'], a.arguments['need_dx']))
        return fused_bwd(*args, **kwargs)
    monkeypatch.setattr(ops, 'fused_bwd', spy)

    def run(bucket):
        x = x0.clone().requires_grad_(x_grad)
        W = W0.clone().requires_grad_(True)
        b = b0.clone().requires_grad_(True)
        loss = ops.GroupSoftmaxFunction.apply(x, W, b, labels, dt, wmask, avg, mode, None, bucket)
        grads = torch.autograd.grad((loss * gout).sum(), [x, W, b] if x_grad else [W, b])
        log.append('returned')
        torch.cuda.synchronize()
        return grads if x_grad else (None,) + grads

    ref = run(None)
    assert log == [('bwd', True, True, x_grad), 'returned']
    del log[:]
    bucket = _StubBucket(C, K, log)
    got = run(bucket)
    # dW + db, then the exchange, then dX (only when x needs it), joined before the backward returns
    assert log == [('bwd', True, True, False), 'exchange'] + [('bwd', False, False, True)] * x_grad + ['join', 'returned']
    assert got[1].data_ptr() == bucket.views[0].data_ptr() and got[2].data_ptr() == bucket.views[1].data_ptr()
    assert torch.equal(bucket.at_exchange[0], got[1]) and torch.equal(bucket.at_exchange[1], got[2])
    assert (got[0] is None) == (not x_grad)
    for name, a, r in zip(('dX', 'dW', 'db'), got, ref):
        if r is not None:
            assert a.dtype == r.dtype and _rel(a.float(), r.float()) <= TOL[mode], (name, _rel(a.float(), r.float()))
