"""Time RPN proposal generation, native against the reference's loop, alternated in one run:

    native     ops.rpn_proposals: every image and level in four launches, no host sync (the counts are read once
               afterwards, as RPNHead.get_bboxes does)
    reference  the reference's per-image, per-level loop of RPNHead.get_bboxes_single (tests/rpn_oracle.py, torch ops
               as the reference runs them) on the reference's own NMS op built into oracle/_ref/, which copies its
               suppression matrix to the host and scans it on the CPU

at the training shape (2 images padded to 800 x 1344, 5 levels, nms_pre = nms_post = max_num = 2000, nms_thr 0.7) and
the test shape (1 image, 1000), on logits whose sigmoids are distinct, so that the two routes' proposals are compared
bit for bit (``equal``).  Milliseconds per call from CUDA events over ``--reps`` calls after a warm-up, median
of ``--rounds`` rounds; the card's name and power limit are printed with them.

    python tools/bench_rpn_proposals.py [--reps 20] [--rounds 5] [--json out.json]
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
SHAPES = {
    'train_2x800x1344_2000': dict(B=2, cfg=dict(nms_pre=2000, nms_post=2000, max_num=2000, nms_thr=0.7,
                                                 min_bbox_size=0)),
    'test_1x800x1344_1000': dict(B=1, cfg=dict(nms_pre=1000, nms_post=1000, max_num=1000, nms_thr=0.7,
                                                min_bbox_size=0)),
}


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out or 'unknown'


def _distinct_logits(sizes, B, gen):
    """[B, 3, H, W] logits per level, a permutation of evenly spaced values in [-4, 4] whose sigmoids are distinct in
    fp32: no tie decides the result, so the two routes must agree bit for bit."""
    total = B * 3 * sum(h * w for h, w in sizes)
    vals = torch.linspace(-4.0, 4.0, total, dtype=torch.float64).float()[torch.randperm(total, generator=gen)]
    assert torch.unique(vals.sigmoid()).numel() == total
    out, o = [], 0
    for h, w in sizes:
        out.append(vals[o:o + B * 3 * h * w].view(B, 3, h, w).cuda())
        o += B * 3 * h * w
    return out


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_rpn_proposals needs a GPU'
    import rpn_oracle as O
    from oracle import ref_nms as REF
    name, power = _gpu_info()
    print('GPU: %s, power limit %s' % (name, power))
    gens = [AnchorGenerator(s, [8], [0.5, 1.0, 2.0]) for s in STRIDES]
    base = [g.base_anchors for g in gens]
    sizes = [((800 + s - 1) // s, (1344 + s - 1) // s) for s in STRIDES]
    gen = torch.Generator().manual_seed(0)
    results = {}
    for shape, spec in SHAPES.items():
        B, cfg = spec['B'], spec['cfg']
        logits = _distinct_logits(sizes, B, gen)
        deltas = [(torch.randn(B, 12, h, w, generator=gen) * 0.5).cuda() for h, w in sizes]
        shapes = [(800, 1333 - 50 * b) for b in range(B)]

        def native():
            out, counts = ops.rpn_proposals(logits, deltas, base, STRIDES, shapes, cfg['nms_pre'], cfg['nms_post'],
                                            cfg['max_num'], cfg['nms_thr'], cfg['min_bbox_size'])
            c = counts.tolist()
            return [out[b, :c[b]] for b in range(B)]

        def reference():
            return O.get_bboxes(logits, deltas, base, STRIDES, shapes, cfg, REF.nms_wrapper_op)

        same = all(torch.equal(a, b) for a, b in zip(native(), reference()))
        times = {}
        for _ in range(args.rounds):
            for which, fn in (('native', native), ('reference', reference)):
                times.setdefault(which, []).append(_events(fn, args.reps))
        med = {k: float(np.median(v)) for k, v in times.items()}
        results[shape] = dict(equal=same, ms=med, speedup=med['reference'] / med['native'])
        print('%-24s equal=%s  native %.3f ms  reference %.3f ms  speed-up %.1fx'
              % (shape, same, med['native'], med['reference'], med['reference'] / med['native']))
    print(json.dumps(dict(gpu=name, power_limit=power, results=results)))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=name, power_limit=power, results=results), f, indent=1)


if __name__ == '__main__':
    main()
