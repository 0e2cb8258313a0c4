"""Time the class-specific mask term -- conv_logits + mask_cross_entropy, forward and backward -- by the reference route
(1x1 conv into [P, 1231, 28, 28] fp32 logits, channel gather, BCE with logits 'mean', autograd) against the fused route
(bags_mask_fwd + bags_mask_bwd), eager and CUDA-graph replayed, at P = 256 and 1024 RoIs, Cin = 256, 28 x 28, 1231
classes, y in fp32 and bf16, and at P = 256 with skewed labels (10 classes; a class-agnostic head), where the
backward sums many RoIs per class; the peak allocated memory of both routes; the fused kernels' bytes over their time against
3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth); then a whole FCNMaskHead training step (forward, loss, backward)
on each route, in alternating runs.  Both routes' outputs are compared at every timed configuration before anything
is timed or printed.  Prints the card name, power limit and SM clock, then one JSON line.  Needs a GPU:

    python tools/bench_mask_loss.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from balancedgroupsoftmax_b200 import _native as nat  # noqa: E402
from balancedgroupsoftmax_b200 import ops  # noqa: E402
from balancedgroupsoftmax_b200.losses import mask_cross_entropy  # noqa: E402

C, CIN, H, W = 1231, 256, 28, 28
HBM_BYTES_PER_S = 3.35e12
REPS = 10


def card():
    """Name, power limit, SM clock and max SM clock, from a read-only nvidia-smi query ('unknown' without one)."""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    except OSError:
        return 'unknown'
    lines = q.stdout.strip().splitlines()
    return lines[0] if q.returncode == 0 and lines else 'unknown'


def inputs(P, dtype, seed=0, classes=C, label_classes=None):
    """y, W, b, labels, targets; labels uniform over 1 .. label_classes (C - 1 by default: about one RoI per class)."""
    g = torch.Generator().manual_seed(seed)
    y = torch.relu(torch.randn(P, CIN, H, W, generator=g)).to(dtype)
    Wt = torch.randn(classes, CIN, 1, 1, generator=g) * (2.0 / CIN) ** 0.5
    b = torch.zeros(classes)
    labels = torch.randint(1, (label_classes or classes - 1) + 1, (P,), generator=g) if classes > 1 else \
        torch.zeros(P, dtype=torch.int64)
    t = (torch.rand(P, H, W, generator=g) > 0.5).float()
    return [v.cuda() for v in (y, Wt, b, labels, t)]


def reference_route(y, Wt, b, labels, t):
    """FCNMaskHead.conv_logits + mask_cross_entropy as the reference runs them (conv in y's dtype, loss in fp32)."""
    return mask_cross_entropy(F.conv2d(y, Wt.to(y.dtype), b.to(y.dtype)).float(), t, labels)


def fused_route(y, Wt, b, labels, t):
    return ops.MaskBCEFunction.apply(y, Wt, b, labels, t)


def run(route, args):
    y, Wt, b = (v.detach().requires_grad_(True) for v in args[:3])
    loss = route(y, Wt, b, *args[3:])
    loss.sum().backward()
    return loss.detach(), Wt.grad, b.grad, y.grad


def timed(fn, iters):
    for _ in range(5):
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


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def graphed(call, reps=REPS):
    """A CUDA graph of ``reps`` back-to-back launches of ``call`` (kernel time without the host's launch cost)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(reps):
                call()
    torch.cuda.current_stream().wait_stream(s)
    return graph.replay


def kernel_bytes(args):
    """Bytes the fused kernels must move, from shapes: forward reads y once, the W rows of the labels, labels and
    targets, and writes g and the per-tile sums; backward reads g, the sums and the W rows, and writes dY, dW and db
    in full."""
    y, Wt, b, labels, t = args
    P = y.shape[0]
    tiles = (H * W + nat.MASK_TILE - 1) // nat.MASK_TILE
    yb = y.numel() * y.element_size()
    rs = P * tiles * (CIN + 2) * 4
    wrows = P * CIN * 4
    fwd = yb + wrows + P * 8 + 2 * P * H * W * 4 + rs
    classes = Wt.shape[0]
    bwd = P * H * W * 4 + rs + wrows + yb + classes * CIN * 4 + classes * 4
    return fwd, bwd


def head_step_times(iters, rounds=5):
    from balancedgroupsoftmax_b200.mask_head import FCNMaskHead
    P = 256
    g = torch.Generator().manual_seed(1)
    x = torch.randn(P, 256, 14, 14, generator=g).cuda()
    t = (torch.rand(P, H, W, generator=g) > 0.5).float().cuda()
    labels = torch.randint(1, C, (P,), generator=g).cuda()
    torch.manual_seed(0)
    head = FCNMaskHead(num_convs=4, in_channels=256, conv_out_channels=256, num_classes=C)
    head.init_weights()
    head.cuda().train()

    def step(materialise):
        pred = head(x)
        if materialise:
            pred = pred.tensor()
        loss = head.loss(pred, t, labels)['loss_mask']
        loss.sum().backward()
        return loss.detach()
    a, b = step(False), step(True)
    assert close(a, b, 1e-3), (a.item(), b.item())
    out = {'reference_ms': [], 'fused_ms': []}
    for _ in range(rounds):
        out['reference_ms'].append(timed(lambda: step(True), iters))
        out['fused_ms'].append(timed(lambda: step(False), iters))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--head-iters', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mask_loss needs a GPU')
    # every configuration's two routes are compared before anything is timed or printed
    configs = [('P%d_%s' % (P, dn), P, dt, {}) for P in (256, 1024)
               for dt, dn in ((torch.bfloat16, 'bf16'), (torch.float32, 'fp32'))]
    # skewed labels: the backward's per-class sums over many RoIs of one class
    configs += [('P256_bf16_10classes', 256, torch.bfloat16, dict(label_classes=10)),
                ('P256_bf16_agnostic', 256, torch.bfloat16, dict(classes=1))]
    for key, P, dtype, kw in configs:
        args = inputs(P, dtype, **kw)
        want = run(reference_route, args)
        got = run(fused_route, args)
        for name, x_, y_ in zip(('loss', 'dW', 'db', 'dY'), got, want):
            assert close(x_, y_, 3e-2), (key, name)
        del args, want, got
    torch.cuda.empty_cache()
    result = {'metric': 'mask_loss_fwd_bwd_ms'}
    for key, P, dtype, kw in configs:
        args = inputs(P, dtype, **kw)
        ref_peak = peak_bytes(lambda: run(reference_route, args))
        fused_peak = peak_bytes(lambda: run(fused_route, args))
        ref_ms = timed(lambda: run(reference_route, args), a.iters)
        fused_ms = timed(lambda: run(fused_route, args), a.iters)
        y, Wt, b, labels, t = args
        gout = torch.ones(1, device='cuda')

        def step():
            loss, g, rsum, index = ops.mask_fwd(y, Wt, b, labels, t)
            return ops.mask_bwd(g, rsum, gout, Wt, labels, index, tuple(y.shape), y.dtype)
        graph_ms = timed(graphed(step, 1), a.iters)
        _, g, rsum, index = ops.mask_fwd(y, Wt, b, labels, t)
        fwd_ms = timed(graphed(lambda: ops.mask_fwd(y, Wt, b, labels, t)), a.iters) / REPS
        bwd_ms = timed(graphed(lambda: ops.mask_bwd(g, rsum, None, Wt, labels, index, tuple(y.shape), y.dtype)),
                       a.iters) / REPS
        fb, bb = kernel_bytes(args)
        result[key] = {
            'reference_eager_ms': round(ref_ms, 4), 'fused_eager_ms': round(fused_ms, 4),
            'fused_graph_ms': round(graph_ms, 4), 'speedup_eager': round(ref_ms / fused_ms, 2),
            'reference_peak_MB': round(ref_peak / 2 ** 20, 1), 'fused_peak_MB': round(fused_peak / 2 ** 20, 1),
            'mask_fwd_us': round(fwd_ms * 1e3, 2), 'mask_bwd_us': round(bwd_ms * 1e3, 2),
            'mask_fwd_hbm_frac': round(fb / (fwd_ms * 1e-3) / HBM_BYTES_PER_S, 3),
            'mask_bwd_hbm_frac': round(bb / (bwd_ms * 1e-3) / HBM_BYTES_PER_S, 3),
        }
        del args, y, g, rsum
        torch.cuda.empty_cache()
    result['fcn_head_step_P256'] = {k: [round(v, 3) for v in vs] for k, vs in head_step_times(a.head_iters).items()}
    result['card'] = card()
    print('card (name, power limit, SM clock, max SM clock):', result['card'])
    print(json.dumps(result))


if __name__ == '__main__':
    main()
