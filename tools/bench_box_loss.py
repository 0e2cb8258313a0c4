"""Time the class-specific box term -- fc_reg + gather + SmoothL1 'mean', forward and backward -- by the default route
(fc_reg GEMM into [N, 4 * 1231] fp32, boolean-mask gather with its host sync, SmoothL1 in torch, GEMM backward) against
the fused route (bags_box_fwd + bags_box_bwd), eager and CUDA-graph replayed, at N = 4096 and 1024 RoIs, K = 1024,
1231 classes, 25 % positives; then a whole GSBBoxHeadWith0 training step (forward, loss, backward) with
fuse_bbox_loss off and on, in alternating runs; then the fused kernels' bytes over their time against 3.35 TB/s
(the H100 SXM data sheet's HBM3 bandwidth).  Both routes' outputs are compared at every timed size before any number
is printed.  Prints the card name, power limit and SM clock, then one JSON line.  Needs a GPU:

    python tools/bench_box_loss.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from balancedgroupsoftmax_b200 import ops  # noqa: E402
from balancedgroupsoftmax_b200.losses import SmoothL1Loss  # noqa: E402

C, K = 1231, 1024
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def inputs(N, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(N, K, generator=g)).to(torch.bfloat16)
    W = torch.randn(4 * C, K, generator=g) * 0.001
    b = torch.zeros(4 * C)
    labels = torch.zeros(N, dtype=torch.int64)
    labels[:N // 4] = torch.randint(1, C, (N // 4,), generator=g)
    targets = torch.randn(N, 4, generator=g) * 0.1
    weights = torch.zeros(N, 4)
    weights[:N // 4] = 1.
    return [t.cuda() for t in (x, W, b, labels, targets, weights)]


def default_route(x, W, b, labels, targets, weights, loss_fn):
    """NativeFcClsHead._fc_reg + BBoxHead._bbox_loss as they run with fuse_bbox_loss off."""
    pred = ops.LinearActFunction.apply(x, W, b, False, torch.bfloat16, torch.float32)
    pos = labels > 0
    p = pred.view(pred.size(0), -1, 4)[pos, labels[pos]]
    return loss_fn(p, targets[pos], weights[pos], avg_factor=targets.size(0))


def fused_route(x, W, b, labels, targets, weights, loss_fn):
    return ops.SmoothL1BoxFunction.apply(x, W, b, labels, targets, weights, 1.0, float(targets.size(0)))[0]


def run(route, args):
    x, W, b = (t.detach().requires_grad_(True) for t in args[:3])
    loss = route(x, W, b, *args[3:], SmoothL1Loss(beta=1.0))
    loss.backward()
    return loss.detach(), W.grad, b.grad, x.grad


def timed(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def close(a, b, rel):
    a, b = a.double(), b.double()
    return (a - b).abs().max().item() <= rel * b.abs().max().item() + 1e-9


def graphed_fused(args):
    x, W, b, labels, targets, weights = args
    gout = torch.ones(1, device='cuda')

    def step():
        loss, g, index, _ = ops.box_fwd(x, W, b, labels, targets, weights, 1.0, float(x.shape[0]))
        return ops.box_bwd(g, gout, x, W, labels, index)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            step()
    torch.cuda.current_stream().wait_stream(s)
    return graph.replay


REPS = 20


def graphed(call):
    """A CUDA graph of REPS back-to-back launches of ``call`` (kernel time without the host's launch cost)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(REPS):
                call()
    torch.cuda.current_stream().wait_stream(s)
    return graph.replay


def kernel_bytes(args):
    """Bytes the fused kernels must move, from shapes: forward reads the positive x rows, the W rows (and bias) of the
    classes present, labels, targets and weights, and writes g; backward reads labels, g, the positive x rows and the
    W rows of the classes present, and writes dW, db and dX in full."""
    x, W, b, labels, targets, weights = args
    N = x.shape[0]
    pos = (labels > 0) & (labels < C)
    P = int(pos.sum())
    present = int(torch.unique(labels[pos]).numel())
    xb = P * K * x.element_size()
    wb = present * 4 * K * 4 + present * 4 * 4
    fwd = xb + wb + N * 8 + 2 * N * 16 + N * 16
    bwd = N * 8 + N * 16 + xb + wb + 4 * C * K * 4 + 4 * C * 4 + N * K * x.element_size()
    return fwd, bwd


def head_step_times(iters, rounds=5):
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    tables = synthetic_tables()
    N = 4096
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(N, 256, 7, 7, generator=g).cuda()
    labels = torch.zeros(N, dtype=torch.int64)
    labels[:N // 4] = torch.randint(1, C, (N // 4,), generator=g)
    labels = labels.cuda()
    lw = torch.ones(N, device='cuda')
    bt = torch.randn(N, 4, device='cuda') * 0.1
    bw = torch.zeros(N, 4, device='cuda')
    bw[:N // 4] = 1.
    heads = {}
    for fuse in (False, True):
        torch.manual_seed(0)
        h = GSBBoxHeadWith0(num_fcs=2, in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=C,
                            gs_config=dict(tables=tables, others_sample_ratio=8.0, num_bins=tables.num_bins,
                                           fuse_bbox_loss=fuse,
                                           loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
        h.init_weights()
        heads[fuse] = h.cuda().train()

    def step(h):
        cls_score, bbox_pred = h(feats)
        losses = h.loss(cls_score, bbox_pred, labels, lw, bt, bw)
        sum(v for k, v in losses.items() if k != 'acc').backward()
        return losses['loss_bbox'].detach()
    lb = {f: step(h) for f, h in heads.items()}
    assert close(lb[True], lb[False], 1e-2), (lb[True].item(), lb[False].item())
    out = {False: [], True: []}
    for _ in range(rounds):
        for fuse in (False, True):
            out[fuse].append(timed(lambda: step(heads[fuse]), iters))
    return {'off_ms': out[False], 'on_ms': out[True]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--head-iters', type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_box_loss needs a GPU')
    print('card (name, power limit, SM clock, max SM clock):', card())
    result = {'metric': 'box_loss_fwd_bwd_ms', 'card': card()}
    for N in (4096, 1024):
        args = inputs(N)
        want = run(default_route, args)
        got = run(fused_route, args)
        for name, a_, b_ in zip(('loss', 'dW', 'db', 'dX'), got, want):
            assert close(a_, b_, 2e-2), (N, name)
        replay = graphed_fused(args)
        default_ms = timed(lambda: run(default_route, args), a.iters)
        fused_ms = timed(lambda: run(fused_route, args), a.iters)
        graph_ms = timed(replay, a.iters)
        x, W, b, labels, targets, weights = args
        _, g, index, _ = ops.box_fwd(x, W, b, labels, targets, weights, 1.0, float(N))
        fwd_ms = timed(graphed(lambda: ops.box_fwd(x, W, b, labels, targets, weights, 1.0, float(N))), a.iters) / REPS
        bwd_ms = timed(graphed(lambda: ops.box_bwd(g, None, x, W, labels, index)), a.iters) / REPS
        fb, bb = kernel_bytes(args)
        result['N%d' % N] = {
            'default_eager_ms': round(default_ms, 4), 'fused_eager_ms': round(fused_ms, 4),
            'fused_graph_ms': round(graph_ms, 4), 'speedup_eager': round(default_ms / fused_ms, 2),
            'box_fwd_us': round(fwd_ms * 1e3, 2), 'box_bwd_us': round(bwd_ms * 1e3, 2),
            'box_fwd_GBps': round(fb / (fwd_ms * 1e-3) / 1e9, 1), 'box_bwd_GBps': round(bb / (bwd_ms * 1e-3) / 1e9, 1),
            'box_fwd_hbm_frac': round(fb / (fwd_ms * 1e-3) / HBM_BYTES_PER_S, 3),
            'box_bwd_hbm_frac': round(bb / (bwd_ms * 1e-3) / HBM_BYTES_PER_S, 3),
        }
    result['head_step_N4096'] = {k: [round(v, 4) for v in vs] for k, vs in head_step_times(a.head_iters).items()}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
