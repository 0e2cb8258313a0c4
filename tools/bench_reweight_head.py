#!/usr/bin/env python
"""Training step of the class-reweighted softmax head (ReweightBBoxHead) -- NOT the headline bench.py.

    python tools/bench_reweight_head.py [--rois 4096] [--in-features 1024] [--classes 1231] [--steps-per-graph 20]

Times, in bf16 operands on one GPU, with CUDA events around replays of a CUDA graph that holds many steps:
  fused        bags_ce_fwd (fc_cls + weighted softmax CE + top-1 accuracy, logits on chip, dW zeroed in the kernel)
               + bags_bwd (dW, db, and dX when the RoI features need a gradient)
  reference    the reference formulation (reweight_bbox_head.py): F.linear -> weighted F.cross_entropy -> accuracy
               -> autograd backward, through torch / cuBLAS
"with dX" is the whole-head configuration; "no dX" is a head-only ("transferred") config where only fc_cls trains.
Prints the GPU name and power limit beside one JSON line of results.  Refuses to run without a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _power_limit_w():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                              str(torch_device_index())], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                             text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def torch_device_index():
    import torch
    return torch.cuda.current_device()


def _time_graph(step, steps_per_graph, replays):
    """ms per step of ``step`` captured ``steps_per_graph`` times into one CUDA graph."""
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps_per_graph):
            step()
    for _ in range(3):
        graph.replay()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(replays):
        graph.replay()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / (replays * steps_per_graph)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rois', type=int, default=4096)
    ap.add_argument('--in-features', type=int, default=1024)
    ap.add_argument('--classes', type=int, default=1231)
    ap.add_argument('--steps-per-graph', type=int, default=20)
    ap.add_argument('--replays', type=int, default=30)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        print('bench_reweight_head: needs a CUDA GPU (H100); refusing to run without one', file=sys.stderr)
        return 2
    from balancedgroupsoftmax_b200 import ops
    from balancedgroupsoftmax_b200.losses import accuracy

    N, K, C = args.rois, args.in_features, args.classes
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(0)
    x = torch.relu(torch.randn(N, K, generator=g)).to(dev, torch.bfloat16)
    W32 = (torch.randn(C, K, generator=g) * 0.02).to(dev)
    b = torch.zeros(C, device=dev)
    labels = torch.zeros(N, dtype=torch.long)
    labels[: N // 4] = torch.randint(1, C, (N // 4,), generator=g)
    labels = labels.to(dev)
    cls_weight = (torch.rand(C, generator=g) * 4.9 + 0.1).to(dev)
    label_weights = torch.ones(N, device=dev)
    Wc = W32.to(torch.bfloat16)
    dt1 = ops._single_slice_tables(C, dev)
    dW = torch.empty(C, K, device=dev)
    acc = torch.empty(1, device=dev)

    def fused(need_dx):
        def step():
            w = cls_weight[labels]
            avg = (label_weights > 0).sum(dtype=torch.float32).clamp_min(1.0).reshape(1)
            _, _, dz, _ = ops.ce_fwd(x, Wc, b, labels, w, avg, want_acc=True, clear=dW, acc_out=acc)
            ops.fused_bwd(dz, x, Wc, None, dt1, None, need_dx=need_dx, dW=dW, dw_prezeroed=True)
        return step

    Wr = Wc.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True)

    def reference(need_dx):
        xr = x.clone().requires_grad_(need_dx)

        def step():
            Wr.grad = br.grad = xr.grad = None
            z = F.linear(xr, Wr, br.to(torch.bfloat16)).float()
            avg = (label_weights > 0).sum(dtype=torch.float32).clamp_min(1.0)
            loss = (F.cross_entropy(z, labels, reduction='none') * cls_weight[labels]).sum() / avg
            accuracy(z, labels)
            loss.backward()
        return step

    res = {}
    for name, mk in (('fused', fused), ('reference', reference)):
        for need_dx in (True, False):
            res['%s_%s_ms' % (name, 'dx' if need_dx else 'no_dx')] = round(
                _time_graph(mk(need_dx), args.steps_per_graph, args.replays), 4)
    for v in ('dx', 'no_dx'):
        res['speedup_' + v] = round(res['reference_%s_ms' % v] / res['fused_%s_ms' % v], 2)
    prop = torch.cuda.get_device_properties(dev)
    res.update(gpu=prop.name, power_limit_w=_power_limit_w(), rois=N, in_features=K, classes=C, dtype='bf16',
               steps_per_graph=args.steps_per_graph, replays=args.replays)
    print('GPU: %s, power limit %s W' % (prop.name, res['power_limit_w']))
    print(json.dumps(res))
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
