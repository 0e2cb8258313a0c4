"""Time the RPN's training targets, native against the reference's route, alternated in one run:

    native     ops.anchor_targets as RPNHead.loss calls it: every image in a memset and four launches, no host sync
    reference  anchor_target as the reference runs it (tests/anchor_target_oracle.py, torch ops as the reference
               runs them): per image the [G, N] IoU matrix on the GPU at <= 50 gts and on the CPU above, the per-gt
               loop of MaxIoUAssigner's step 4 with its host syncs, and RandomSampler's np.random.shuffle

at 2 images padded to 800 x 1344, 5 levels, 3 anchors per location (268,569 anchors per image) and the configs'
rpn train cfg, for 3, 15, 50, 100 and 300 gts per image.  Once per shape, both routes run with num >= the anchor
count and pos_fraction 1, where the sample takes every positive and negative, and their targets are compared
bit for bit (``assign_equal``).  Milliseconds per call from CUDA events over ``--reps`` calls after a warm-up,
median of ``--rounds`` rounds; the card's name and power limit are printed with them.

    python tools/bench_anchor_target.py [--reps 5] [--rounds 3] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

from balancedgroupsoftmax_b200 import ops  # noqa: E402
from balancedgroupsoftmax_b200.rpn_head import AnchorGenerator  # noqa: E402

STRIDES = [4, 8, 16, 32, 64]
GTS = [3, 15, 50, 100, 300]
CFG = dict(assigner=dict(type='MaxIoUAssigner', pos_iou_thr=0.7, neg_iou_thr=0.3, min_pos_iou=0.3, ignore_iof_thr=-1),
           sampler=dict(type='RandomSampler', num=256, pos_fraction=0.5, neg_pos_ub=-1, add_gt_as_proposals=False),
           allowed_border=0, pos_weight=-1)
METAS = [dict(img_shape=(800, 1333, 3), pad_shape=(800, 1344, 3)),
         dict(img_shape=(750, 1344, 3), pad_shape=(800, 1344, 3))]


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out or 'unknown'


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _gts(n, gen):
    out = []
    for m in METAS:
        h, w = m['img_shape'][:2]
        x1, y1 = torch.rand(n, generator=gen) * (w - 8), torch.rand(n, generator=gen) * (h - 8)
        bw, bh = 4 + torch.rand(n, generator=gen) * 396, 4 + torch.rand(n, generator=gen) * 396
        out.append(torch.stack([x1, y1, (x1 + bw).clamp(max=w - 1), (y1 + bh).clamp(max=h - 1)], 1).round().cuda())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_anchor_target needs a GPU'
    import anchor_target_oracle as O
    name, power = _gpu_info()
    print('GPU: %s, power limit %s' % (name, power))
    base = [AnchorGenerator(s, [8], [0.5, 1.0, 2.0]).base_anchors for s in STRIDES]
    sizes = [((800 + s - 1) // s, (1344 + s - 1) // s) for s in STRIDES]
    N = sum(h * w * 3 for h, w in sizes)
    gen = torch.Generator().manual_seed(0)
    zero, one = (0., 0., 0., 0.), (1., 1., 1., 1.)
    results = {}
    for n in GTS:
        gts = _gts(n, gen)

        def native(cfg=CFG, seed=[0]):
            seed[0] += 1
            a, s = cfg['assigner'], cfg['sampler']
            return ops.anchor_targets(sizes, base, STRIDES, [m['img_shape'] for m in METAS],
                                      [m['pad_shape'] for m in METAS], gts, a['pos_iou_thr'], a['neg_iou_thr'],
                                      a['min_pos_iou'], True, cfg['allowed_border'], s['num'], s['pos_fraction'],
                                      s['neg_pos_ub'], cfg['pos_weight'], zero, one, seed=seed[0])

        def reference(cfg=CFG):
            return O.anchor_target(base, sizes, STRIDES, gts, METAS, zero, one, cfg, O.numpy_shuffle, 'cuda')

        all_cfg = dict(CFG, sampler=dict(CFG['sampler'], num=N, pos_fraction=1.0))
        got, (want, counts) = native(all_cfg), reference(all_cfg)
        same = all(torch.equal(torch.nan_to_num(a), torch.nan_to_num(b)) for a, b in zip(got[:4], want)) and \
            got[4].tolist()[:2] == list(counts)
        times = {}
        for _ in range(args.rounds):
            for which, fn in (('native', native), ('reference', reference)):
                times.setdefault(which, []).append(_events(fn, args.reps))
        med = {k: float(np.median(v)) for k, v in times.items()}
        key = '2x800x1344_%dgts' % n
        results[key] = dict(assign_equal=same, ms=med, speedup=med['reference'] / med['native'],
                            reference_route='cpu' if n > 50 else 'cuda')
        print('%-22s assign_equal=%s  native %.3f ms  reference (%s) %.2f ms  speed-up %.0fx'
              % (key, same, med['native'], results[key]['reference_route'], med['reference'],
                 med['reference'] / med['native']))
    print(json.dumps(dict(gpu=name, power_limit=power, results=results)))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=name, power_limit=power, results=results), f, indent=1)


if __name__ == '__main__':
    main()
