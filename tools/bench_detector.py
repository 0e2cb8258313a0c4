#!/usr/bin/env python
"""Full-detector harness bench -- NOT the headline bench.py.

    python tools/bench_detector.py [--stages 1|3] [--imgs-per-gpu 2] [--steps 20] [--warmup 5]
    python -m torch.distributed.run --nproc-per-node N tools/bench_detector.py ...      (one rank per GPU)

Synthetic 1333x800 images -> frozen torchvision R50-FPN trunk + RPN + RoIAlign -> 512 sampled RoIs / image ->
BAGS head(s) forward + loss + backward -> mean of the head gradients over ranks -> SGD step on the head.
Reports images/s (whole job) and the share of a step spent in the head (CUDA events around the head's part), one JSON
line on rank 0.
--config faster|cascade|htc selects BASELINE.json configs[2..4]' head-call shapes: 2 img x 512 RoIs x 1 head, 2 x 512 x 3
heads, 1 x 512 x 3 heads (the HTC config's mask branch and X-101 trunk are not part of the harness: R50-FPN stands in).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default=None, choices=['faster', 'cascade', 'htc'])
    ap.add_argument('--stages', type=int, default=1, choices=[1, 3])
    ap.add_argument('--imgs-per-gpu', type=int, default=2)
    ap.add_argument('--height', type=int, default=800)
    ap.add_argument('--width', type=int, default=1333)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--dtype', default='bf16', choices=['bf16', 'fp32'])
    ap.add_argument('--no-amp', dest='amp', action='store_false', help='shared FCs / fc_reg in fp32 instead of bf16 autocast')
    args = ap.parse_args()
    if args.config is not None:
        args.stages, args.imgs_per_gpu = {'faster': (1, 2), 'cascade': (3, 2), 'htc': (3, 1)}[args.config]

    import torch
    import torch.distributed as dist
    from balancedgroupsoftmax_b200.dist import allreduce_grads
    from balancedgroupsoftmax_b200.harness import BagsDetectorHarness, synthetic_batch
    from balancedgroupsoftmax_b200.tables import synthetic_tables

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if not torch.cuda.is_available():
        raise SystemExit('bench_detector.py needs an H100 GPU (the BAGS head has no CPU fallback)')
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    tables = synthetic_tables(1231, seed=0)
    weights = (1.0,) if args.stages == 1 else (1.0, 0.5, 0.25)
    model = BagsDetectorHarness(tables, num_stages=args.stages, stage_loss_weights=weights, compute_dtype=args.dtype, amp=args.amp,
                                min_size=args.height, max_size=args.width).to(dev)
    model.train()
    params = model.head_parameters()
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9, weight_decay=1e-4)
    g = torch.Generator().manual_seed(100 + rank)
    batches = [synthetic_batch(args.imgs_per_gpu, args.height, args.width, device=dev, generator=g) for _ in range(4)]

    head_ms = []

    def step(i, timed=False):
        imgs, gb, gl = batches[i % len(batches)]
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        feats, proposals, sizes, scales = model.trunk(imgs)
        gbs = [b * s for b, s in zip(gb, scales)]
        e[0].record()
        opt.zero_grad(set_to_none=True)
        losses = {}
        rois = proposals
        for si, head in enumerate(model.heads):
            x, sampling, boxes = model.head_inputs(feats, rois, gbs, gl, sizes, si)
            cls_score, bbox_pred = model.run_head(head, x)
            targets = head.get_target(sampling, gbs, gl, model.rcnn_cfg)
            for k, v in head.loss(cls_score, bbox_pred, *targets).items():
                losses['s%d.%s' % (si, k)] = v * weights[si]
            if si + 1 < len(model.heads):
                with torch.no_grad():
                    br = torch.cat([torch.cat([b.new_full((b.size(0), 1), j), b], 1) for j, b in enumerate(boxes)], 0)
                    metas = [dict(img_shape=(int(s[0]), int(s[1]), 3)) for s in sizes]
                    rois = head.refine_bboxes(br, targets[0], bbox_pred.detach().float(), [s.pos_is_gt for s in sampling], metas)
        total = sum(losses.values())
        total.backward()
        if world > 1:
            allreduce_grads(params)
        opt.step()
        e[1].record()
        if timed:
            head_ms.append(e)
        return total

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    last = None
    for i in range(args.steps):
        last = step(i, timed=True)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.steps
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    head = sum(a.elapsed_time(b) for a, b in head_ms) / len(head_ms)
    if rank == 0:
        print(json.dumps({
            'metric': 'images/s, synthetic %dx%d, frozen R50-FPN trunk + %d BAGS head stage(s), fwd+bwd+exchange+SGD on the head'
                      % (args.width, args.height, args.stages),
            'value': world * args.imgs_per_gpu / (ms * 1e-3), 'unit': 'img/s', 'n_gpus': world, 'ms_per_step': ms,
            'head_ms_per_step': head, 'head_share': head / ms, 'steps': args.steps, 'warmup': args.warmup,
            'dtype': args.dtype, 'amp_trunk_fcs': bool(args.amp), 'data': 'synthetic', 'loss': float(last.detach().float().item()),
            'config': {'name': args.config, 'imgs_per_gpu': args.imgs_per_gpu, 'rois_per_image': 512, 'stages': args.stages,
                       'trunk': 'torchvision fasterrcnn_resnet50_fpn (frozen, random init)'}}), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == '__main__':
    sys.exit(main())
