#!/usr/bin/env python
"""Head-only training step of the bfocal baseline (ReweightBBoxHead + sigmoid FocalLoss) -- NOT the headline bench.py.

    python tools/bench_focal_head.py [--rois 4096] [--in-features 1024] [--classes 1231] [--gamma 0.5] [--alpha 1]

configs/transferred/faster_rcnn_r50_fpn_1x_lvis_reweighthead_bfocal.py trains only fc_cls, so its step is
fc_cls -> loss -> dW, db (no dX).  Times, in bf16 operands on one GPU, with CUDA events around replays of a CUDA graph
that holds many steps:
  fused        bags_focal_fwd (fc_cls + the focal loss and its gradient per element + top-1 accuracy, logits on chip,
               dW zeroed in the kernel) + bags_bwd (dW, db)
  reference    the reference formulation: F.linear -> the focal-loss op restated in torch (one-hot targets, the op's
               analytic gradient) weighted by cls_weight[labels] / (N * 1231) -> accuracy -> autograd backward
Prints the GPU name and power limit beside one JSON line of results.  Refuses to run without a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_reweight_head import _power_limit_w, _time_graph  # noqa: E402


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rois', type=int, default=4096)
    ap.add_argument('--in-features', type=int, default=1024)
    ap.add_argument('--classes', type=int, default=1231)
    ap.add_argument('--gamma', type=float, default=0.5)
    ap.add_argument('--alpha', type=float, default=1.0)
    ap.add_argument('--steps-per-graph', type=int, default=20)
    ap.add_argument('--replays', type=int, default=30)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        print('bench_focal_head: needs a CUDA GPU (H100); refusing to run without one', file=sys.stderr)
        return 2
    from balancedgroupsoftmax_b200 import ops
    from balancedgroupsoftmax_b200 import losses as L

    N, K, C = args.rois, args.in_features, args.classes
    gamma, alpha = args.gamma, args.alpha
    norm = float(N * L.FOCAL_ONE_HOT_CLASSES)
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(0)
    x = torch.relu(torch.randn(N, K, generator=g)).to(dev, torch.bfloat16)
    W32 = (torch.randn(C, K, generator=g) * 0.02).to(dev)
    b = torch.zeros(C, device=dev)
    labels = torch.zeros(N, dtype=torch.long)
    labels[: N // 4] = torch.randint(1, C, (N // 4,), generator=g)
    labels = labels.to(dev)
    cls_weight = (torch.rand(C, generator=g) * 4.9 + 0.1).to(dev)
    Wc = W32.to(torch.bfloat16)
    dt1 = ops._single_slice_tables(C, dev)
    dW = torch.empty(C, K, device=dev)
    acc = torch.empty(1, device=dev)

    def fused():
        w = cls_weight[labels]
        t = L.focal_targets(labels, N)
        _, _, dz, _ = ops.focal_fwd(x, Wc, b, t, norm, gamma, alpha, labels=labels, weights=w, want_acc=True,
                                    clear=dW, acc_out=acc)
        ops.fused_bwd(dz, x, Wc, None, dt1, None, need_dx=False, dW=dW, dw_prezeroed=True)

    Wr = Wc.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True)

    def reference():
        Wr.grad = br.grad = None
        z = F.linear(x, Wr, br.to(torch.bfloat16)).float()
        t = F.one_hot(labels, num_classes=L.FOCAL_ONE_HOT_CLASSES).reshape(-1)[:N]
        el = L._SigmoidFocalOp.apply(z, t, gamma, alpha)
        loss = (el * cls_weight[labels].view(-1, 1)).sum() / norm
        L.accuracy(z, labels)
        loss.backward()

    res = {'fused_ms': round(_time_graph(fused, args.steps_per_graph, args.replays), 4),
           'reference_ms': round(_time_graph(reference, args.steps_per_graph, args.replays), 4)}
    res['speedup'] = round(res['reference_ms'] / res['fused_ms'], 2)
    prop = torch.cuda.get_device_properties(dev)
    res.update(gpu=prop.name, power_limit_w=_power_limit_w(), rois=N, in_features=K, classes=C, dtype='bf16',
               gamma=gamma, alpha=alpha, steps_per_graph=args.steps_per_graph, replays=args.replays)
    print('GPU: %s, power limit %s W' % (prop.name, res['power_limit_w']))
    print(json.dumps(res))
    return 0


if __name__ == '__main__':
    raise SystemExit(main())
